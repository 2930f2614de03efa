"""CPU: the BGZF member walk (kmcb200_bgzf_scan) against a Python header walk, both host readers of gzip files against zlib, the
reference's size rules for gzip input, and the stored reference results pinned to their regenerated inputs."""
import hashlib
import json
import os
import zlib

import numpy as np
import pytest

import kmc_b200
from kmc_b200 import reads
from gzip_testlib import BGZF_EOF, GZIP_CASES, GZIP_GOLDEN, bgzf, bgzf_member, case_text, gz_variants, gzip_single, inflate_all, \
    py_bgzf_scan, write
from test_fastx_model import fasta_text, fastq_text

FQ = fastq_text(4041, 3000, max_len=150)


def _scan(raw, cap, max_members=None):
    c, t, m = kmc_b200.bgzf_scan(raw, cap, max_members)
    return c, t, [tuple(int(x) for x in r) for r in m]


@pytest.mark.parametrize("seed", [None, 1, 2])
def test_scan_matches_the_header_walk_over_capacity_and_partial_members(seed):
    raw = bgzf(FQ, seed=seed)
    want = py_bgzf_scan(raw, 1 << 40)
    assert sum(m[3] for m in want[2]) == len(FQ) and want[0] == len(raw)      # the EOF member is taken too
    ends = sorted({m[0] + m[2] for m in want[2]})
    for cut in [0, 3, 11, 17, 18, 19, len(raw) // 3, ends[0] - 1, ends[0], ends[0] + 1, len(raw) - len(BGZF_EOF), len(raw) - 1, len(raw)]:
        for cap in [0, 1, 65279, 65280, 65281, 200_000, 1 << 40]:
            assert _scan(raw[:cut], cap) == py_bgzf_scan(raw[:cut], cap), (cut, cap)
    assert _scan(raw, 1 << 40, max_members=2) == py_bgzf_scan(raw, 1 << 40, max_members=2)


def test_scan_offsets_are_the_exclusive_sum_of_isize():
    c, t, m = kmc_b200.bgzf_scan(bgzf(FQ, seed=7), 1 << 40)
    assert np.array_equal(m["out_off"], np.concatenate([[0], np.cumsum(m["isize"].astype(np.uint64))[:-1]]))
    assert np.array_equal(m["in_off"][1:], (m["in_off"] + m["in_bytes"])[:-1]) and t == len(FQ)


@pytest.mark.parametrize("raw", [gzip_single(FQ), b"@r1\nACGT\n+\nIIII\n", bytes(bgzf_member(b"x" * 70000, deflated=zlib.compress(b"x", 9)[2:-4]))],
                         ids=["plain_gzip", "text", "isize_over_64k"])
def test_scan_rejects_a_first_member_that_is_not_bgzf(raw):
    assert py_bgzf_scan(raw, 1 << 40) is None
    with pytest.raises(kmc_b200.KmcB200Error) as e:
        kmc_b200.bgzf_scan(raw, 1 << 40)
    assert e.value.code == kmc_b200.ERR_INVALID


def test_scan_stops_before_a_member_that_is_not_bgzf():
    raw = bgzf(FQ[:100_000], eof=False) + gzip_single(FQ[100_000:])
    c, t, m = kmc_b200.bgzf_scan(raw, 1 << 40)
    assert t == 100_000 and raw[c:c + 2] == b"\x1f\x8b" and (c, t, [tuple(int(x) for x in r) for r in m]) == py_bgzf_scan(raw, 1 << 40)


@pytest.mark.parametrize("text", [FQ, fasta_text(4042, 500, max_len=900), b""], ids=["fastq", "fasta", "empty"])
def test_host_reader_gives_the_plain_text(tmp_path, text):
    for name, data in gz_variants(text).items():
        assert reads.read_text(write(str(tmp_path / (name + ".gz")), data)) == text, name
    assert reads.read_text(write(str(tmp_path / "plain"), text)) == text


@pytest.mark.parametrize("kind", ["single", "concat"])
@pytest.mark.parametrize("chunk", [1 << 17, 1 << 18])
def test_chunk_reader_zlib_mode_gives_the_plain_text(tmp_path, monkeypatch, kind, chunk):
    """_RawChunks over a plain gzip file (zlib on the reader thread, no GPU): the chunks with the carried rests are the text."""
    monkeypatch.setattr(reads, "_pinned", lambda n: (None, np.empty(n, dtype=np.uint8)))
    path = write(str(tmp_path / "x.gz"), gz_variants(FQ)[kind])
    got, cut = [], 0
    with reads._RawChunks(path, chunk) as chunks:
        for c, final in chunks:
            used = len(c) if final else len(c) - 1000                   # carry a rest, as an unfinished record would be
            got.append(bytes(c[:used]))
            chunks.consumed(used)
            cut += 1
    assert b"".join(got) == FQ and cut > 2


def test_truncated_and_corrupt_gzip_are_errors(tmp_path):
    data = gzip_single(FQ)
    with pytest.raises(kmc_b200.KmcB200Error, match="truncated"):
        reads.read_text(write(str(tmp_path / "t.gz"), data[:len(data) // 2]))
    bad = bytearray(data)
    bad[-8] ^= 1
    with pytest.raises(kmc_b200.KmcB200Error, match="gzip input"):
        reads.read_text(write(str(tmp_path / "c.gz"), bytes(bad)))


def test_size_rules_count_gzip_as_the_reference_does(tmp_path):
    """binary_reader.h:378-386: (uint64)(3.2 * size) for gzip; kmc.h:1002 max(2^28, predicted / 100); kmc.h:1118-1121 s by predicted size."""
    gz = write(str(tmp_path / "a.fq.gz"), gzip_single(FQ))
    plain = write(str(tmp_path / "b.fq"), FQ)
    size = os.path.getsize(gz)
    assert reads.predicted_size([gz]) == int(3.2 * size) and reads.predicted_size([gz, plain]) == int(3.2 * size) + len(FQ)
    assert reads.is_gzip(gz) and not reads.is_gzip(plain)
    # a file of 1.6e10 bytes (sparse) predicts 5.12e10 >= 5e10 as gzip (s = 11), not as text (s = 7)
    big = str(tmp_path / "big.gz")
    with open(big, "wb") as f:
        f.write(b"\x1f\x8b")
        f.truncate(16 * 10 ** 9)
    assert reads.predicted_size([big]) == 51_200_000_000 and reads.estimate_s([big]) == 11
    with open(big, "r+b") as f:
        f.write(b"@r")
    assert reads.estimate_s([big]) == 7


def test_reference_inputs_are_the_stored_texts():
    """The stored reference results belong to these texts: the cases regenerate them from their seeds."""
    golden = json.load(open(GZIP_GOLDEN))
    assert sorted(golden) == sorted(GZIP_CASES)
    for name, (kind, k, opts, _) in GZIP_CASES.items():
        assert golden[name]["text_md5"] == hashlib.md5(case_text(kind)).hexdigest(), name
        assert golden[name]["k"] == k and golden[name]["options"] == opts
        assert inflate_all(bgzf(case_text(kind))) == case_text(kind)
