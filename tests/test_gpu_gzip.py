"""GPU: BGZF members inflated on the GPU equal zlib byte for byte over levels, strategies, member sizes, long matches and flushes; malformed
members are errors that hand on no text; and gzip inputs (BGZF, plain, concatenated, mixed) give the databases, -e files and totals of the
same text uncompressed, which are the reference's (tests/golden/gzip_reference.json), on both parse modes and through the command line."""
import hashlib
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import kmc_b200
from kmc_b200 import reads
from gzip_testlib import BGZF_EOF, GZIP_CASES, GZIP_GOLDEN, bgzf, bgzf_member, case_text, deflate_fixed, gz_variants, inflate_all, write
from test_fastx_model import fastq_text

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FQ = fastq_text(5051, 6000, max_len=150)
RNG = np.random.default_rng(5052)
RANDOM = bytes(RNG.integers(0, 256, 32768, dtype=np.uint8))
SKEW = bytes(RNG.choice(256, 60000, p=np.r_[[0.5 ** (i + 1) for i in range(255)], [0.5 ** 255]]).astype(np.uint8))


def _corpus():
    c = {"level%d" % lv: bgzf(FQ[:400_000], level=lv) for lv in range(10)}
    for name, st in [("fixed", zlib.Z_FIXED), ("huffman_only", zlib.Z_HUFFMAN_ONLY), ("rle", zlib.Z_RLE), ("filtered", zlib.Z_FILTERED)]:
        c[name] = bgzf(FQ[:300_000], strategy=st)
    c["mem_level1"] = bgzf(FQ[:200_000], mem_level=1, level=9)
    c["sizes_0_to_65536"] = b"".join(bgzf_member(FQ[:n]) for n in [0, 1, 2, 31, 32, 33, 255, 4096, 65279, 65280, 65535, 65536]) + BGZF_EOF
    c["random_sizes"] = bgzf(FQ, seed=11)
    c["poly_a"] = bgzf(b"A" * 65536, piece=65536) + bgzf(b"A" * 65536, piece=65536, level=1)
    c["distance_32768"] = bgzf_member(RANDOM * 2, deflated=deflate_fixed(list(RANDOM) + [(258, 32768)] * 126 + [(130, 32768)] * 2))
    c["overlap_lengths"] = bgzf_member(b"ab" * 400, deflated=deflate_fixed([97, 98] + [(n, 2) for n in [3, 31, 32, 33, 258, 258, 183]]))
    c["skewed_15_bit_codes"] = bgzf(SKEW, piece=65536)
    c["random_stored"] = bgzf(RANDOM[:30000] * 2, piece=60000, level=1)
    c["sync_flush"] = bgzf(FQ[:300_000], flush_every=1000)
    c["full_flush"] = bgzf(FQ[:300_000], flush_every=2500, flush_mode=zlib.Z_FULL_FLUSH)
    c["eof_only"] = BGZF_EOF
    return c


CORPUS = _corpus()


@pytest.fixture(scope="module")
def gz():
    g = kmc_b200.Gunzip(0, max_in_bytes=1 << 23, max_out_bytes=1 << 23)
    yield g
    g.close()


@pytest.mark.parametrize("name", sorted(CORPUS))
def test_inflate_equals_zlib(gz, name):
    raw = CORPUS[name]
    want = inflate_all(raw)
    out = np.zeros(len(want) + 1, dtype=np.uint8)
    before = gz.kernel_launches()
    consumed, n = gz.inflate(raw, out)
    assert (consumed, n) == (len(raw), len(want)) and out[:n].tobytes() == want
    assert gz.kernel_launches() == before + 1


def test_capacity_and_partial_member_cut_a_call(gz):
    raw = CORPUS["random_sizes"]
    want = inflate_all(raw)
    c, t, m = kmc_b200.bgzf_scan(raw, 1 << 40)
    mid = int(m["in_off"][len(m) // 2]) + 10                            # inside a member
    pieces, pos = [], 0
    for cut_in, cap in [(mid, 1 << 30), (len(raw), 150_000), (len(raw), 1 << 30)]:
        out = np.zeros(cap if cap < 1 << 30 else len(want), dtype=np.uint8)
        used, n = gz.inflate(raw[pos:cut_in], out)
        assert used > 0 and n <= out.size
        pieces.append(out[:n].tobytes())
        pos += used
    while pos < len(raw):
        out = np.zeros(len(want) + 1, dtype=np.uint8)
        used, n = gz.inflate(raw[pos:], out)
        pieces.append(out[:n].tobytes())
        pos += used
    assert b"".join(pieces) == want
    out = np.zeros(10, dtype=np.uint8)
    assert gz.inflate(raw, out) == (0, 0)                               # not one whole member fits


def test_device_twin_equals_zlib():
    import torch
    raw = CORPUS["random_sizes"] + CORPUS["level1"] + CORPUS["skewed_15_bit_codes"]
    want = inflate_all(raw)
    c, t, m = kmc_b200.bgzf_scan(raw, 1 << 40)
    g = kmc_b200.Gunzip(0, 1 << 20, 1 << 20)
    try:
        d_raw = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
        d_m = torch.from_numpy(m.view(np.uint8).copy()).cuda()
        d_text = torch.zeros(t, dtype=torch.uint8, device="cuda")
        d_err = torch.zeros(1, dtype=torch.int64, device="cuda")
        s = torch.cuda.current_stream()
        g.dev_inflate(d_m.data_ptr(), len(m), d_raw.data_ptr(), len(raw), d_text.data_ptr(), t, d_err.data_ptr(), s.cuda_stream)
        s.synchronize()
        assert int(d_err.item()) == -1 and d_text.cpu().numpy().tobytes() == want
        # a table entry that reaches past the buffers is the kernel's error, not a read or write outside them
        bad = m.copy()
        bad["out_off"][3] = t - 10
        d_m = torch.from_numpy(bad.view(np.uint8).copy()).cuda()
        g.dev_inflate(d_m.data_ptr(), len(m), d_raw.data_ptr(), len(raw), d_text.data_ptr(), t, d_err.data_ptr(), s.cuda_stream)
        s.synchronize()
        e = int(d_err.item()) & ((1 << 64) - 1)
        assert e >> 8 == 3 and e & 0xff == 1
    finally:
        g.close()


def _malformed():
    text = FQ[:20_000]
    good = bgzf_member(text)
    data = good[18:-8]
    crc = bytearray(good)
    crc[-8] ^= 1
    isize = bgzf_member(text[:-1], deflated=data)[:-4] + len(text[:-1]).to_bytes(4, "little")
    isize = isize[:-8] + zlib.crc32(text).to_bytes(4, "little") + isize[-4:]
    return {
        "crc": bytes(crc),
        "isize": isize,
        "distance_before_start": bgzf_member(b"aaaa", deflated=deflate_fixed([97, (3, 2)])),
        "invalid_code": bgzf_member(b"aaaa", deflated=deflate_fixed([97, 286])),
        "invalid_distance_code": bgzf_member(b"aaaa", deflated=deflate_fixed([97])[:-1] + b"\xff\xff"),
        "truncated": bgzf_member(text, deflated=data[:len(data) // 2]),
        "block_type_3": bgzf_member(b"", deflated=b"\x07\x00"),
        "stored_length": bgzf_member(b"ab", deflated=b"\x01\x02\x00\x00\x00ab"),
        "trailing_bytes": bgzf_member(text, deflated=data + b"\x00"),
    }


@pytest.mark.parametrize("name", sorted(_malformed()))
def test_malformed_member_is_an_error_and_hands_on_no_text(gz, name):
    raw = bgzf(FQ[:100_000]) [:-len(BGZF_EOF)] + _malformed()[name] + BGZF_EOF
    out = np.full(200_000, 7, dtype=np.uint8)
    with pytest.raises(kmc_b200.KmcB200Error) as e:
        gz.inflate(raw, out)
    assert e.value.code == kmc_b200.ERR_INVALID and "BGZF member 2 (byte %d" % (len(raw) - len(BGZF_EOF) - len(_malformed()[name])) in str(e.value)
    assert np.all(out == 7)
    used, n = gz.inflate(CORPUS["level6"], np.zeros(1 << 20, dtype=np.uint8))     # the handle is still good
    assert used == len(CORPUS["level6"])


def test_non_bgzf_header_is_an_error(gz):
    with pytest.raises(kmc_b200.KmcB200Error) as e:
        gz.inflate(zlib.compress(FQ[:1000]), np.zeros(2000, dtype=np.uint8))
    assert e.value.code == kmc_b200.ERR_INVALID


# ----------------------------------------------------------------------------- reads -> databases
GOLDEN = json.load(open(GZIP_GOLDEN))


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def _run_case(name, path, out, parse, batch_bytes=1 << 26):
    kind, k, opts, kw = GZIP_CASES[name]
    if "-e" in opts:
        reads.write_histogram(out + ".txt", reads.estimate_histogram([path], k, batch_bytes=batch_bytes, parse=parse))
        return {"histogram_md5": md5(out + ".txt")}
    res = reads.count_reads([path], out, k, 9, None, batch_bytes=batch_bytes, parse=parse, **kw)
    return {"kmc_pre_md5": md5(out + ".kmc_pre"), "kmc_suf_md5": md5(out + ".kmc_suf"), "unique_kmers": res["n_unique"]}


def _expected(name):
    g = GOLDEN[name]
    return {key: g[key] for key in ("histogram_md5", "kmc_pre_md5", "kmc_suf_md5", "unique_kmers") if key in g}


@pytest.mark.parametrize("parse", ["gpu", "host"])
@pytest.mark.parametrize("name", sorted(GZIP_CASES))
def test_bgzf_input_gives_the_reference_files(tmp_path, name, parse):
    text = case_text(GZIP_CASES[name][0])
    path = write(str(tmp_path / "in.gz"), bgzf(text))
    assert _run_case(name, path, str(tmp_path / "db"), parse) == _expected(name)


@pytest.mark.parametrize("batch_bytes", [1 << 20, 1 << 26])
@pytest.mark.parametrize("kind", ["bgzf", "single", "concat", "mixed"])
def test_every_gzip_layout_gives_the_plain_files(tmp_path, kind, batch_bytes):
    for name in ["fq_k31", "fm_k31", "fq_k13_small"]:
        text = case_text(GZIP_CASES[name][0])
        path = write(str(tmp_path / ("in_%s.gz" % name)), gz_variants(text)[kind])
        assert _run_case(name, path, str(tmp_path / name), "gpu", batch_bytes) == _expected(name), name


def test_gpu_reader_inflates_bgzf_on_the_gpu(tmp_path, monkeypatch):
    """The BGZF path runs the inflate kernel: every piece of a multi-chunk file comes from Gunzip calls, and no zlib is used."""
    calls = []
    real = kmc_b200.Gunzip.inflate
    monkeypatch.setattr(kmc_b200.Gunzip, "inflate", lambda self, raw, out: calls.append(1) or real(self, raw, out))
    monkeypatch.setattr(reads, "_zlib_members", None)
    text = case_text("fq")
    path = write(str(tmp_path / "in.gz"), bgzf(text))
    with reads._RawChunks(path, (1 << 20) - 1) as chunks:
        got = []
        for c, final in chunks:
            got.append(bytes(c))
            chunks.consumed(len(c))
    assert b"".join(got) == text and len(calls) >= len(text) // (1 << 19)


def test_command_line_takes_gz(tmp_path):
    text = case_text("fq")
    plain = write(str(tmp_path / "r.fq"), text)
    gzp = write(str(tmp_path / "r.fq.gz"), bgzf(text))
    env = dict(os.environ, PYTHONPATH=ROOT)
    for path, out in [(plain, "p"), (gzp, "g")]:
        subprocess.run([sys.executable, "-m", "kmc_b200.reads", "--gpu-parse", "-k31", path, str(tmp_path / out)], check=True, env=env,
                       stdout=subprocess.DEVNULL)
    for ext in (".kmc_pre", ".kmc_suf"):
        assert md5(str(tmp_path / ("p" + ext))) == md5(str(tmp_path / ("g" + ext)))


def test_gunzip_returns_its_memory():
    import torch

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info(0)[0]

    def cycle():
        g = kmc_b200.Gunzip(0, 1 << 24, 1 << 24)
        g.inflate(CORPUS["level6"], np.zeros(1 << 20, dtype=np.uint8))
        g.close()

    cycle()
    before = free()
    cycle()
    assert before - free() <= 8 << 20
