"""GPU: BGZF members inflated on the GPU equal zlib byte for byte over levels, strategies, member sizes, long matches and flushes, and over
the legal stream shapes zlib never writes; malformed members are errors for the right reason that hand on no text, one case per validation
rule, and the first bad member of a call is the one named; seeded random streams and their mutations get zlib's verdict; and gzip inputs (BGZF, plain, concatenated, mixed) give the databases, -e files and totals of the
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
from gzip_testlib import BGZF_EOF, DIFF_SEEDS, GZ_ERRORS, GZIP_CASES, GZIP_GOLDEN, ZLIB_TO_KERNEL, Fixed, bgzf, bgzf_member, case_text, deflate, \
    differential_streams, gz_variants, inflate_all, malformed_streams, shape_streams, write, zlib_inflate
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
    c["distance_32768"] = bgzf_member(RANDOM * 2, deflated=deflate([Fixed(list(RANDOM) + [(258, 32768)] * 126 + [(130, 32768)] * 2)]))
    c["overlap_lengths"] = bgzf_member(b"ab" * 400, deflated=deflate([Fixed([97, 98] + [(n, 2) for n in [3, 31, 32, 33, 258, 258, 183]])]))
    c["skewed_15_bit_codes"] = bgzf(SKEW, piece=65536)
    c["random_stored"] = bgzf(RANDOM[:30000] * 2, piece=60000, level=1)
    c["sync_flush"] = bgzf(FQ[:300_000], flush_every=1000)
    c["full_flush"] = bgzf(FQ[:300_000], flush_every=2500, flush_mode=zlib.Z_FULL_FLUSH)
    c["eof_only"] = BGZF_EOF
    for name, (data, text) in shape_streams().items():                 # legal shapes zlib's deflate never writes
        c["shape_" + name] = bgzf_member(text, deflated=data) + BGZF_EOF
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
    """name -> (member, the kernel's error): a zlib member's CRC, ISIZE, half its data and a byte after it, and the deflate streams of
    gzip_testlib.malformed_streams, one per validation rule, each framed with the CRC32 and length of a text of at most 64 KiB."""
    text = FQ[:20_000]
    good = bgzf_member(text)
    data = good[18:-8]
    crc = bytearray(good)
    crc[-8] ^= 1
    isize = bgzf_member(text[:-1], deflated=data)[:-4] + len(text[:-1]).to_bytes(4, "little")
    isize = isize[:-8] + zlib.crc32(text).to_bytes(4, "little") + isize[-4:]
    m = {
        "crc": (bytes(crc), "crc"),
        "isize": (isize, "output"),
        "isize_above_text": (bgzf_member(text + b"x", deflated=data), "isize"),
        "truncated": (bgzf_member(text, deflated=data[:len(data) // 2]), "truncated"),
        "trailing_bytes": (bgzf_member(text, deflated=data + b"\x00"), "trailing"),
    }
    for name, (d, t, err) in malformed_streams().items():
        m[name] = (bgzf_member(t, deflated=d), err)
    return m


MALFORMED = _malformed()


def _reason(err):
    return ": " + GZ_ERRORS[err][1]


@pytest.mark.parametrize("name", sorted(MALFORMED))
def test_malformed_member_is_an_error_and_hands_on_no_text(gz, name):
    member, err = MALFORMED[name]
    raw = bgzf(FQ[:100_000]) [:-len(BGZF_EOF)] + member + BGZF_EOF
    out = np.full(200_000, 7, dtype=np.uint8)
    with pytest.raises(kmc_b200.KmcB200Error) as e:
        gz.inflate(raw, out)
    msg = str(e.value)
    assert e.value.code == kmc_b200.ERR_INVALID and "BGZF member 2 (byte %d of the input)" % (len(raw) - len(BGZF_EOF) - len(member)) in msg
    assert msg.endswith(_reason(err)), msg
    assert np.all(out == 7)
    used, n = gz.inflate(CORPUS["level6"], np.zeros(1 << 20, dtype=np.uint8))     # the handle is still good
    assert used == len(CORPUS["level6"])


def test_the_first_bad_member_is_named(gz):
    """Bad members at 7 and 3 with different errors: the call names member 3 and its reason, and the device twin's error word is
    3 << 8 | member 3's code (the lower code of member 7 does not win)."""
    import torch
    members = [bgzf_member(FQ[i * 3000:(i + 1) * 3000]) for i in range(10)]
    members[3], err3 = MALFORMED["no_end_of_block"]
    members[7], err7 = MALFORMED["block_type_3"]
    assert GZ_ERRORS[err7][0] < GZ_ERRORS[err3][0]
    raw = b"".join(members)
    out = np.full(40_000, 7, dtype=np.uint8)
    with pytest.raises(kmc_b200.KmcB200Error) as e:
        gz.inflate(raw, out)
    assert "BGZF member 3 (byte %d " % len(b"".join(members[:3])) in str(e.value) and str(e.value).endswith(_reason(err3)), str(e.value)
    assert np.all(out == 7)
    c, t, m = kmc_b200.bgzf_scan(raw, 1 << 40)
    assert len(m) == 10
    d_raw = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
    d_m = torch.from_numpy(m.view(np.uint8).copy()).cuda()
    d_text = torch.zeros(max(t, 1), dtype=torch.uint8, device="cuda")
    d_err = torch.zeros(1, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    gz.dev_inflate(d_m.data_ptr(), len(m), d_raw.data_ptr(), len(raw), d_text.data_ptr(), t, d_err.data_ptr(), s.cuda_stream)
    s.synchronize()
    assert int(d_err.item()) & ((1 << 64) - 1) == 3 << 8 | GZ_ERRORS[err3][0]


@pytest.mark.parametrize("seed", DIFF_SEEDS)
def test_random_streams_get_zlibs_verdict(seed):
    """Seeded random block sequences and their mutations (tests/gzip_testlib.differential_streams): a stream zlib accepts with no bytes
    left over inflates to zlib's text, all such members in one call; a stream zlib refuses, leaves unfinished or finds bytes after is an
    error of its own call, for the reason ZLIB_TO_KERNEL maps zlib's to, and hands on no text.  A refused member's trailer is well formed
    with ISIZE 65536, so the kernel never stops at the ISIZE bound or reaches the CRC32 / ISIZE check before the deflate data's error.  A
    failure names the seed and stream: differential_streams(seed)[i] replays it on the CPU."""
    g = kmc_b200.Gunzip(0, max_in_bytes=1 << 24, max_out_bytes=1 << 25)
    try:
        where = "seed %d, zlib %s" % (seed, zlib.ZLIB_RUNTIME_VERSION)
        good, good_text, bad = [], [], []
        for i, (data, text) in enumerate(differential_streams(seed)):
            verdict, out = zlib_inflate(data)
            if verdict == "ok":
                good.append((i, bgzf_member(out, deflated=data)))
                good_text.append(out)
            elif verdict != "oversize":
                member = bgzf_member(text, deflated=data)
                bad.append((i, member[:-4] + (65536).to_bytes(4, "little"), ZLIB_TO_KERNEL[out if verdict == "error" else verdict]))
        raw = b"".join(m for _, m in good)
        want = b"".join(good_text)
        out = np.zeros(len(want) + 1, dtype=np.uint8)
        try:
            used, n = g.inflate(raw, out)
        except kmc_b200.KmcB200Error as e:
            k = int(str(e).split("BGZF member ")[1].split(" ")[0])
            raise AssertionError("%s: stream %d accepted by zlib is refused: %s" % (where, good[k][0], e))
        assert (used, n) == (len(raw), len(want)), where
        if out[:n].tobytes() != want:
            at = 0
            for (i, _), t in zip(good, good_text):
                assert out[at:at + len(t)].tobytes() == t, "%s: stream %d inflates to other text than zlib's" % (where, i)
                at += len(t)
        wrong = []
        for i, member, err in bad:
            out = np.full(65536, 7, dtype=np.uint8)
            try:
                g.inflate(member, out)
            except kmc_b200.KmcB200Error as e:
                assert e.code == kmc_b200.ERR_INVALID and np.all(out == 7), "%s: stream %d: %s" % (where, i, e)
                if not str(e).endswith(_reason(err)):
                    wrong.append("stream %d: %s, zlib's reason maps to %r" % (i, str(e).split(": ")[-1], err))
                continue
            raise AssertionError("%s: stream %d, which zlib refuses (%s), is accepted: %s" % (where, i, err, member.hex()))
        assert not wrong, "%s: %d refused streams with another reason than zlib's, the first: %s" % (where, len(wrong), "; ".join(wrong[:5]))
        print("%s: %d streams accepted (%d text bytes compared in one call of %d members), %d refused" % (where, len(good), len(want),
                                                                                                              len(good), len(bad)))
        assert len(good) >= 300 and len(bad) >= 300
    finally:
        g.close()


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
