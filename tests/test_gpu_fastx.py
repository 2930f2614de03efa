"""GPU: the reads-text parser on the H100 (kmcb200_fastx_* / kmc_b200.FastxParser, kmcb200_split_fastx, kmcb200_sigstats_add_fastx,
count_reads(parse="gpu")).  Every case is compared with the numpy model of tests/test_fastx_model.py (parse_chunk) or with
kmc_b200.reads.sequences_to_batch, and the databases with the host path's and the reference's."""
import os

import numpy as np
import pytest

from stage1_testlib import STAGE1_CASES, STAGE1_GOLDEN, case_reads, make_reads, random_map, write_fastq_reads
from test_fastx_model import (CORPUS, FASTA, FASTQ, TOO_LONG, fasta_text, fastq_text, longest_record, parse_chunk, parse_in_chunks,
                              random_cuts, records_of, special_cuts)

pytestmark = pytest.mark.gpu


def parser(fmt, max_chunk=1 << 22):
    import kmc_b200
    return kmc_b200.FastxParser(fmt, max_chunk_bytes=max_chunk)


def big_fastq(n_bytes, seed=3):
    """> n_bytes of FASTQ, full-Phred qualities: a tiled block of fastq_text, so it is cheap to make."""
    block = fastq_text(seed, 4000, max_len=250)
    return block * (n_bytes // len(block) + 1)


# ----------------------------------------------------------------------------- parse parity
@pytest.mark.parametrize("name,data,fmt", CORPUS, ids=[c[0] for c in CORPUS])
def test_parse_whole_chunk_equals_model(name, data, fmt):
    from kmc_b200.reads import sequences_to_batch
    p = parser(fmt)
    seq, c = p.parse(data, True)
    want, wc = parse_chunk(data, fmt, True)
    assert c == wc == len(data)
    assert seq.tobytes() == want.tobytes() == sequences_to_batch(data).tobytes()
    p.close()


@pytest.mark.parametrize("name,data,fmt", CORPUS, ids=[c[0] for c in CORPUS])
def test_parse_in_chunks_equals_model(name, data, fmt):
    from kmc_b200.reads import sequences_to_batch
    p = parser(fmt)
    gpu = lambda raw, f, final: p.parse(raw, final)
    want = sequences_to_batch(data).tobytes()
    got, starts = parse_in_chunks(data, fmt, special_cuts(data, fmt), gpu)
    assert got.tobytes() == want
    assert starts == parse_in_chunks(data, fmt, special_cuts(data, fmt))[1]
    rng = np.random.default_rng(len(data))
    longest = longest_record(data, fmt)
    for trial in range(6):
        lo = 1 if trial % 2 else longest + 1
        cuts = random_cuts(rng, len(data), lo, lo + int(rng.integers(1, 3 * longest + 2)))
        got, starts = parse_in_chunks(data, fmt, cuts, gpu)
        assert got.tobytes() == want
        assert starts == parse_in_chunks(data, fmt, cuts)[1]
    p.close()


@pytest.mark.parametrize("name,data,fmt", CORPUS[:8], ids=[c[0] for c in CORPUS[:8]])
def test_consumed_limit_and_records_equal_model(name, data, fmt):
    import torch
    p = parser(fmt)
    rng = np.random.default_rng(99 + len(data))
    dev = torch.device("cuda:0")
    d_raw = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(dev)
    d_seq = torch.zeros(len(data) + 1, dtype=torch.uint8, device=dev)
    d_res = torch.zeros(4, dtype=torch.int64, device=dev)
    for limit in [None, 1, len(data) - 1] + [int(x) for x in rng.integers(1, len(data), 12)]:
        for final in (True, False):
            end = len(data) if final else int(rng.integers(len(data) // 2, len(data)))
            raw = data[:end]
            try:
                want, wc = parse_chunk(raw, fmt, final, limit)
            except Exception as e:  # noqa: BLE001
                assert TOO_LONG in str(e)
                continue
            seq, c = p.parse(raw, final, limit)
            assert (c, seq.tobytes()) == (wc, want.tobytes()), (limit, final, end)
            p.dev_parse(d_raw.data_ptr(), end, final, limit, d_seq.data_ptr(), d_seq.numel(), d_res.data_ptr(), None)
            torch.cuda.synchronize()
            res = d_res.cpu().numpy()
            assert list(res) == [wc, want.size, records_of(raw, fmt, wc), 0], (limit, final, end)
            assert d_seq[:want.size].cpu().numpy().tobytes() == want.tobytes()
    p.close()


def test_errors_and_capacity_leave_the_output_untouched():
    import torch
    import kmc_b200
    data = fastq_text(21, 50)
    p = parser(FASTQ, max_chunk=4096)
    first = int(np.flatnonzero(np.frombuffer(data, np.uint8) == 10)[3]) + 1
    out = np.full(first + 8, 0xAB, dtype=np.uint8)
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        p.parse(data[:first - 1], False, out=out)
    assert ei.value.code == kmc_b200.ERR_INVALID and TOO_LONG in str(ei.value)
    assert (out == 0xAB).all()
    want, _ = parse_chunk(data[:first], FASTQ, True)
    short = np.full(want.size - 1, 0xAB, dtype=np.uint8)
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        p.parse(data[:first], True, out=short)
    assert ei.value.code == kmc_b200.ERR_CAPACITY and (short == 0xAB).all()
    exact = np.empty(want.size, dtype=np.uint8)
    assert p.parse(data[:first], True, out=exact)[0].tobytes() == want.tobytes()
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        p.parse(data[:4097], True)                                          # over max_chunk_bytes
    assert ei.value.code == kmc_b200.ERR_INVALID
    dev = torch.device("cuda:0")
    d_raw = torch.frombuffer(bytearray(data[:first - 1]), dtype=torch.uint8).to(dev)
    d_seq = torch.full((first,), 0xAB, dtype=torch.uint8, device=dev)
    d_res = torch.zeros(4, dtype=torch.int64, device=dev)
    p.dev_parse(d_raw.data_ptr(), first - 1, False, None, d_seq.data_ptr(), d_seq.numel(), d_res.data_ptr(), None)
    torch.cuda.synchronize()
    assert list(d_res.cpu().numpy()) == [0, 0, 0, 1] and bool((d_seq == 0xAB).all())
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        p.dev_parse(d_raw.data_ptr(), first - 1, False, None, d_seq.data_ptr(), first - 1, d_res.data_ptr(), None)   # capacity < bytes + 1
    assert ei.value.code == kmc_b200.ERR_INVALID
    for kw in (dict(fmt=3), dict(max_chunk=0), dict(max_chunk=(1 << 31) + 1)):
        a = dict(fmt=FASTQ, max_chunk=1 << 20)
        a.update(kw)
        with pytest.raises(kmc_b200.KmcB200Error) as ei:
            parser(a["fmt"], a["max_chunk"])
        assert ei.value.code == kmc_b200.ERR_INVALID
    p.close()


def test_launches_per_call_do_not_depend_on_size_and_a_large_chunk():
    """9 launches for 1 KB and for 256 MB; a chunk of more than 2^28 bytes parses like sequences_to_batch."""
    from kmc_b200.reads import sequences_to_batch
    big = big_fastq((1 << 28) + (1 << 20))
    p = parser(FASTQ, max_chunk=len(big))
    counts = []
    for raw in (big[:1000], big[:256_000_000], big):
        b = p.kernel_launches()
        seq, c = p.parse(raw, raw is big)
        counts.append(p.kernel_launches() - b)
    assert counts == [9, 9, 9]
    assert c == len(big) and len(big) > 1 << 28
    assert seq.tobytes() == sequences_to_batch(big).tobytes()
    p.close()


# ----------------------------------------------------------------------------- device twin into dev_split / dev_sigstats_add
def test_dev_parse_feeds_dev_split_and_dev_sigstats_add():
    import torch
    import kmc_b200
    from kmc_b200.reads import sequences_to_batch
    k, m, nb = 31, 9, 64
    data = fastq_text(31, 2000, max_len=250)
    batch = sequences_to_batch(data)
    sig_map = random_map(31, m, nb)
    p = parser(FASTQ)
    sp = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=len(data) + 1)
    st = kmc_b200.SignatureStats(k, m, max_batch_bytes=len(data) + 1)
    want_out, want_packs, want_frags = [x.copy() if hasattr(x, "copy") else x for x in sp.split_raw(batch)]
    st.add(batch)
    want_counts = st.read()
    st.reset()
    dev = torch.device("cuda:0")
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        d_raw = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(dev)
        d_seq = torch.empty(len(data) + 1, dtype=torch.uint8, device=dev)
        d_res = torch.zeros(4, dtype=torch.int64, device=dev)
        p.dev_parse(d_raw.data_ptr(), len(data), True, None, d_seq.data_ptr(), d_seq.numel(), d_res.data_ptr(), s.cuda_stream)
    s.synchronize()
    n = int(d_res[1])
    assert n == batch.size and int(d_res[0]) == len(data) and int(d_res[2]) == 2000
    assert d_seq[:n].cpu().numpy().tobytes() == batch.tobytes()
    d_out = torch.empty(want_out.size + 64, dtype=torch.uint8, device=dev)
    d_packs = torch.empty(want_packs.size + 8, dtype=torch.int64, device=dev)
    d_frags = torch.zeros(nb * 5, dtype=torch.int64, device=dev)
    d_sres = torch.zeros(8, dtype=torch.int64, device=dev)
    with torch.cuda.stream(s):
        sp.dev_split(d_seq.data_ptr(), n, d_out.data_ptr(), d_out.numel(), d_packs.data_ptr(), d_packs.numel(), d_frags.data_ptr(), d_sres.data_ptr(),
                     s.cuda_stream)
        st.dev_add(d_seq.data_ptr(), n, s.cuda_stream)
    s.synchronize()
    assert int(d_sres[2]) == 0 and int(d_sres[0]) == want_out.size
    assert d_out[:want_out.size].cpu().numpy().tobytes() == want_out.tobytes()
    assert np.array_equal(d_packs[:want_packs.size].cpu().numpy().view(np.uint64), want_packs)
    assert np.array_equal(st.read(), want_counts)
    for x in (p, sp, st):
        x.close()


# ----------------------------------------------------------------------------- the _fastx entry points
def split_tuple(out, packs, frags):
    fr = np.array([[f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs] for f in frags], dtype=np.uint64)
    return out.tobytes(), packs.tobytes(), fr.tobytes()


@pytest.mark.parametrize("k", [17, 31, 55, 128])
@pytest.mark.parametrize("m", [5, 9, 11])
def test_split_fastx_equals_split_raw_of_sequences_to_batch(k, m):
    import kmc_b200
    from kmc_b200.reads import sequences_to_batch
    nb = 128
    sig_map = random_map(k * 7 + m, m, nb)
    texts = [(fastq_text(k + m, 600, max_len=250, crlf=bool(k % 2)), FASTQ), (fasta_text(k * m, 200, max_len=600), FASTA)]
    for data, fmt in texts:
        p = parser(fmt)
        sp = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=len(data) + 1)
        ref = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=len(data) + 1)
        launches = sp.kernel_launches()
        out, packs, frags, c, nseq = sp.split_fastx(p, data, True)
        batch = sequences_to_batch(data)
        assert c == len(data) and nseq == batch.size
        assert split_tuple(out, packs, frags) == split_tuple(*ref.split_raw(batch))
        assert sp.kernel_launches() - launches == ref.kernel_launches()      # the parse's launches are the parser's
        whole = [out[f.byte_off:f.byte_off + f.bytes].tobytes() for f in frags]   # out is the splitter's buffer: copy before the next call
        # chunked: the concatenation of each bin's fragments is the one-batch bin
        half = len(data) // 2
        out1, packs1, frags1, c1, _ = sp.split_fastx(p, data[:half], False)
        b1 = [out1[f.byte_off:f.byte_off + f.bytes].tobytes() for f in frags1]
        out2, packs2, frags2, c2, _ = sp.split_fastx(p, data[c1:], True)
        assert c1 + c2 == len(data)
        assert [b1[b] + out2[f.byte_off:f.byte_off + f.bytes].tobytes() for b, f in enumerate(frags2)] == whole
        for x in (p, sp, ref):
            x.close()


def test_add_fastx_equals_add_and_limit():
    import kmc_b200
    from kmc_b200.reads import _record_end, sequences_to_batch
    k, m = 31, 9
    data = fastq_text(41, 1500, max_len=250)
    p = parser(FASTQ)
    st = kmc_b200.SignatureStats(k, m, max_batch_bytes=len(data) + 1)
    ref = kmc_b200.SignatureStats(k, m, max_batch_bytes=len(data) + 1)
    assert st.add_fastx(p, data, True) == len(data)
    ref.add(sequences_to_batch(data))
    assert np.array_equal(st.read(), ref.read())
    st.reset()
    ref.reset()
    limit = len(data) // 3
    c = st.add_fastx(p, data, True, limit)
    assert c == _record_end(data, limit - 1)
    ref.add(sequences_to_batch(data[:c]))
    assert np.array_equal(st.read(), ref.read())
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        st.add_fastx(p, data[:10], False)
    assert ei.value.code == kmc_b200.ERR_INVALID and TOO_LONG in str(ei.value)
    for x in (p, st, ref):
        x.close()


def test_splitter_without_fastx_keeps_its_launch_count():
    import kmc_b200
    from kmc_b200.reads import sequences_to_batch
    data = fastq_text(51, 300)
    batch = sequences_to_batch(data)
    sig_map = random_map(5, 7, 32)
    a = kmc_b200.Splitter(31, 7, sig_map, 32, max_batch_bytes=len(data) + 1)
    b = kmc_b200.Splitter(31, 7, sig_map, 32, max_batch_bytes=len(data) + 1)
    p = parser(FASTQ)
    a.split_raw(batch)                                                  # the first calls also size the host output buffers
    b.split_fastx(p, data, True)
    assert a.kernel_launches() == b.kernel_launches() > 0
    n = a.kernel_launches()
    a.split_raw(batch)
    b.split_fastx(p, data, True)
    assert a.kernel_launches() - n == b.kernel_launches() - n > 0       # the parse's 9 launches are counted on the parser
    for x in (a, b, p):
        x.close()


# ----------------------------------------------------------------------------- count_reads(parse="gpu")
def _golden_case(case):
    import json
    return json.load(open(STAGE1_GOLDEN))["cases"][case]


@pytest.mark.parametrize("case", sorted(STAGE1_CASES))
@pytest.mark.parametrize("with_map", [False, True])
def test_count_reads_gpu_parse_matches_stored_reference_database(tmp_path, case, with_map):
    from kmc_b200.reads import count_reads
    from kmc_testlib import digest
    from stage1_testlib import load_map
    c = _golden_case(case)
    h = c["header"]
    fq = str(tmp_path / "reads.fq")
    write_fastq_reads(fq, case_reads(case))
    out = str(tmp_path / "db")
    sig_map = load_map(case) if with_map else None
    res = count_reads([fq], out, h["k"], h["sig_len"], sig_map, h["p"], h["cmin"], h["cmax"], c["counter_max"], h["both"], batch_bytes=1 << 20,
                      n_bins=len(c["bins"]), parse="gpu")
    assert {ext: digest(open(out + ext, "rb").read()) for ext in (".kmc_pre", ".kmc_suf")} == c["files"]
    assert res["n_kmers"] == c["total_kmers"] == res["n_total"]
    assert res["n_super_kmers"] == c["total_super_kmers"]


def test_cli_gpu_parse(tmp_path):
    import subprocess
    import sys
    from kmc_testlib import digest
    case = "k55_p9_ndense_b"
    c = _golden_case(case)
    h = c["header"]
    fq = str(tmp_path / "reads.fq")
    write_fastq_reads(fq, case_reads(case))
    out = str(tmp_path / "db")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run([sys.executable, "-m", "kmc_b200.reads", "--gpu-parse", "--batch-bytes", str(1 << 18), "-n64", "-k%d" % h["k"], "-p%d" % h["sig_len"],
                    "--lut-prefix-len", str(h["p"]), "--ci", str(h["cmin"]), "--cs", str(c["counter_max"]), "-b", fq, out], check=True, cwd=root,
                   capture_output=True)
    assert {ext: digest(open(out + ext, "rb").read()) for ext in (".kmc_pre", ".kmc_suf")} == c["files"]


def _both(paths, tmp, **kw):
    from kmc_b200.reads import count_reads
    res, files = {}, {}
    for parse in ("host", "gpu"):
        out = os.path.join(tmp, parse)
        r = count_reads(paths, out, 31, 9, None, 7, 2, 10 ** 9, 255, True, parse=parse, **kw)
        res[parse] = {key: r[key] for key in ("n_unique", "n_cutoff_min", "n_cutoff_max", "n_total", "n_super_kmers", "n_kmers", "n_bases")}
        files[parse] = [open(out + ext, "rb").read() for ext in (".kmc_pre", ".kmc_suf")]
    assert res["host"] == res["gpu"]
    assert files["host"] == files["gpu"]
    return res["gpu"]


def test_host_and_gpu_parse_agree_on_several_files_and_a_small_sample(tmp_path, monkeypatch):
    from kmc_b200 import reads
    tmp = str(tmp_path)
    texts = [fastq_text(61, 3000, max_len=250), fastq_text(62, 2000, max_len=250, crlf=True, final_newline=False), fasta_text(63, 800, max_len=2000),
             b"", fasta_text(64, 300, max_len=600, final_newline=False)]
    paths = []
    for i, t in enumerate(texts):
        paths.append(os.path.join(tmp, "in%d.txt" % i))
        open(paths[-1], "wb").write(t)
    r = _both(paths, tmp, batch_bytes=1 << 16)                          # many chunks per file
    assert r["n_kmers"] > 0
    monkeypatch.setattr(reads, "STATS_SAMPLE_BYTES", len(texts[0]) + 12345)   # the sample ends inside the second file
    _both(paths, tmp, batch_bytes=1 << 16)
    monkeypatch.setattr(reads, "STATS_SAMPLE_BYTES", 5000)                    # ... inside the first file's first chunk
    _both(paths, tmp, batch_bytes=1 << 16)


@pytest.mark.parametrize("crlf", [False, True])
def test_gpu_parse_matches_reference_cli(tmp_path, crlf):
    """Where the reference CLI is built: full-Phred FASTQ (and CRLF) through kmc_ref -sr1 and through count_reads(parse="gpu")."""
    from kmc_b200.reads import count_reads
    from test_gpu_kmc_files import KMC_REF, count, md5
    if not os.path.exists(KMC_REF):
        pytest.skip("oracle/_ref/kmc_ref not built")
    tmp = str(tmp_path)
    reads = make_reads(71, "short", 20000, 150, genome_len=300_000)
    rng = np.random.default_rng(72)
    eol = b"\r\n" if crlf else b"\n"
    fq = os.path.join(tmp, "reads.fq")
    with open(fq, "wb") as f:
        for i, r in enumerate(reads):
            q = np.arange(33, 75, dtype=np.uint8)[rng.integers(0, 42, len(r))].tobytes()
            f.write(b"@r%d" % i + eol + r + eol + b"+" + eol + q + eol)
    k, p = 31, 9
    ref_db, st = count(KMC_REF, tmp, "ref", fq, k, ("-p%d" % p, "-ci2", "-sr1"))
    from stage1_testlib import kmc_pre_bins
    h = kmc_pre_bins(ref_db + ".kmc_pre", ref_db + ".kmc_suf")[0]
    out = os.path.join(tmp, "gpu")
    count_reads([fq], out, k, p, None, h["p"], h["cmin"], h["cmax"], 255, True, batch_bytes=1 << 21, parse="gpu")
    assert md5(out + ".kmc_suf") == md5(ref_db + ".kmc_suf")
    assert md5(out + ".kmc_pre") == md5(ref_db + ".kmc_pre")
