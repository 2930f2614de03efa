"""CPU: the BGZF member walk (kmcb200_bgzf_scan) against a Python header walk, both host readers of gzip files against zlib, the
reference's size rules for gzip input, the stored reference results pinned to their regenerated inputs, and the DEFLATE writer and zlib
oracle the GPU inflate tests stand on: every valid stream the writer makes decodes under zlib to the text its tokens spell, every
malformed one is refused by zlib for the reason that maps to the kernel's expected error, and the differential streams' verdicts."""
import hashlib
import json
import os
import zlib

import numpy as np
import pytest

import kmc_b200
from kmc_b200 import reads
from gzip_testlib import BGZF_EOF, BGZF_MAX_DATA, DIFF_BASES, DIFF_SEEDS, GZ_ERRORS, GZIP_CASES, GZIP_GOLDEN, ZLIB_TO_KERNEL, Dynamic, Fixed, Stored, \
    bgzf, bgzf_member, blocks_text, case_text, deflate, differential_streams, gz_variants, gzip_single, huffman_lengths, inflate_all, \
    malformed_streams, py_bgzf_scan, rle_lengths, shape_blocks, shape_streams, write, zlib_inflate
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


# ----------------------------------------------------------------------------- the DEFLATE writer and the zlib oracle
SHAPES = shape_streams()


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_writer_shape_decodes_under_zlib_to_its_tokens_text(name):
    """The text is spelled from the tokens, not taken from zlib; zlib ends the stream on its last byte with no bytes left over."""
    data, text = SHAPES[name]
    d = zlib.decompressobj(-15)
    assert d.decompress(data) == text and d.eof and d.unused_data == b"" and d.unconsumed_tail == b"", zlib.ZLIB_RUNTIME_VERSION
    assert len(text) <= 65536


def test_writer_shapes_have_the_features_they_are_named_for():
    blocks = {k: b for k, (b, _) in shape_blocks().items()}

    def crossing(b, sym):
        lit, dist, hlit, _ = b.code_lengths()
        at = 0
        for s in rle_lengths(lit + dist, hlit, b.rle):
            n = 1 if isinstance(s, int) else s[1]
            if not isinstance(s, int) and s[0] == sym and at < hlit < at + n:
                return True
            at += n
        return False

    assert crossing(blocks["repeat16_across_trees"][0], 16) and crossing(blocks["zero_run_across_trees"][0], 18)
    assert blocks["zero_run_across_trees"][0].code_lengths()[2:] == (286, 30)
    assert max(blocks["repeat16_across_trees"][0].code_lengths()[1]) == 9
    assert [b.code_lengths()[1] for b in blocks["single_1bit_distance_code"]] == [[1], [0] * 9 + [1]]
    assert blocks["single_1bit_end_of_block"][0].code_lengths()[0] == [0] * 256 + [1]
    assert [b.code_lengths()[1:] for b in blocks["literal_only_empty_distance_tree"]] == [([0], 257, 1), ([0] * 30, 257, 30)]
    assert blocks["hlit_257_hdist_1"][0].code_lengths()[2:] == (257, 1)
    assert blocks["hlit_hdist_above_need"][0].code_lengths()[2:] == (286, 30)
    assert [b.hclen for b in blocks["hclen_5_to_19"]] == list(range(5, 20))
    lit, dist, _, _ = blocks["distance_codes_9_to_15_bits"][0].code_lengths()
    used = {t.dsym for t in blocks["distance_codes_9_to_15_bits"][0].tokens if not isinstance(t, int)}
    assert set(range(8, 16)) <= used and max(dist) == 15
    lit = blocks["literal_codes_10_and_11_bits"][0].code_lengths()[0]
    toks = blocks["literal_codes_10_and_11_bits"][0].tokens
    syms = {t if isinstance(t, int) else t.lsym for t in toks}
    assert {lit[s] for s in syms} == {8, 10, 11} and lit[256] == 10
    lay = []
    deflate(blocks["mixed_blocks_stored_every_phase"], layout=lay)
    phases = [s % 8 for (s, _, _), b in zip(lay, blocks["mixed_blocks_stored_every_phase"]) if isinstance(b, Stored)]
    assert sorted(phases) == list(range(8))
    assert {type(b) for b in blocks["mixed_blocks_stored_every_phase"]} == {Stored, Fixed, Dynamic}
    assert len(deflate(blocks["stored_largest"])) == 65510
    assert sum(1 for b in blocks["length_258_as_284_31"] for t in b.tokens if not isinstance(t, (int, tuple)) and (t.lsym, t.lextra) == (284, 31)) > 50


def test_writer_gives_the_former_fixed_block_bytes():
    """The fixed blocks of the distance_32768 and overlap_lengths members are the bytes the former fixed-block writer gave."""
    rng = np.random.default_rng(5052)
    rand = bytes(rng.integers(0, 256, 32768, dtype=np.uint8))
    a = deflate([Fixed(list(rand) + [(258, 32768)] * 126 + [(130, 32768)] * 2)])
    b = deflate([Fixed([97, 98] + [(n, 2) for n in [3, 31, 32, 33, 258, 258, 183]])])
    assert hashlib.sha256(a).hexdigest() == "8bb971c420e26697ed8d30e2e1aa8ae4a0b6559e4ebdde38c8a207e93f45891f"
    assert b.hex() == "4b4c0242029010240847e1281ca21000"
    assert deflate([Fixed([97, (3, 2)])]).hex() == "4b044200" and deflate([Fixed([97, 286])]).hex() == "4b1c0300"


def test_writer_stored_lengths_0_to_65535_at_every_bit_phase():
    data = bytes(range(256)) * 256
    for n in [0, 1, 65535]:
        for phase in range(8):
            blocks = [Fixed([200] * phase + [65]), Stored(data[:n]), Stored(b"")]
            lay = []
            raw = deflate(blocks, seed=phase, layout=lay)
            assert lay[1][0] % 8 == (phase + 3 + 8 + 7) % 8 and zlib_inflate(raw, 1 << 17) == ("ok", blocks_text(blocks))


def test_huffman_lengths_are_complete_and_limited():
    rng = np.random.default_rng(8)
    for limit in [7, 9, 12, 15]:
        for n in [2, 3, 19, 30, 286]:
            if n > 1 << limit:
                continue
            freq = [int(x) for x in (2.0 ** rng.integers(0, 30, n)).astype(np.int64)]
            lens = huffman_lengths(freq, limit)
            assert max(lens) <= limit and sum(2.0 ** -x for x in lens) == 1.0, (limit, n)
            assert all(lens[i] <= lens[j] for i in range(n) for j in range(n) if freq[i] > freq[j])
    assert huffman_lengths([0, 5, 0], 15) == [0, 1, 0] and huffman_lengths([0, 0], 15) == [0, 0]


MALFORMED = malformed_streams()


@pytest.mark.parametrize("name", sorted(MALFORMED))
def test_malformed_stream_is_refused_by_zlib_for_the_mapped_reason(name):
    data, text, error = MALFORMED[name]
    verdict, detail = zlib_inflate(data)
    reason = detail if verdict == "error" else verdict
    assert ZLIB_TO_KERNEL.get(reason) == error, (verdict, detail, zlib.ZLIB_RUNTIME_VERSION)
    assert error in GZ_ERRORS and len(text) <= 65536 and len(data) >= 2                 # a BGZF member holds at least 2 bytes of data


def test_every_mapped_zlib_reason_has_a_malformed_case():
    got = set()
    for data, _, _ in MALFORMED.values():
        verdict, detail = zlib_inflate(data)
        got.add(detail if verdict == "error" else verdict)
    assert got == set(ZLIB_TO_KERNEL)


@pytest.mark.parametrize("seed", DIFF_SEEDS)
def test_differential_streams_zlib_verdicts(seed):
    """Every generated stream is valid and decodes to its blocks' text; its mutations give zlib verdicts of every kind, a few hundred
    accepted and a few hundred refused per seed, every accepted text within a BGZF member."""
    streams = differential_streams(seed)
    assert len(streams) == 3 * DIFF_BASES
    verdicts = {"ok": 0, "error": 0, "unfinished": 0, "trailing": 0, "oversize": 0}
    for i, (data, text) in enumerate(streams):
        assert 2 <= len(data) <= BGZF_MAX_DATA, (seed, i)                               # each fits a BGZF member
        verdict, out = zlib_inflate(data)
        if i % 3 == 0:
            assert (verdict, out) == ("ok", text), (seed, i, zlib.ZLIB_RUNTIME_VERSION)
        verdicts[verdict] += 1
    assert verdicts["ok"] >= 300 and verdicts["error"] + verdicts["unfinished"] + verdicts["trailing"] >= 300, verdicts
    assert min(verdicts["error"], verdicts["unfinished"], verdicts["trailing"]) >= 50 and verdicts["oversize"] == 0, verdicts
    assert differential_streams(seed)[:30] == streams[:30]
