"""Histogram estimation on the GPU (kmcb200_estimator_*, kmc_b200.HistogramEstimator, kmc_b200.reads.estimate_histogram and
count_reads(lut_prefix_len=None, opt_out_size=...)) against the stored reference results (tests/golden/estimate_reference.json) and the
oracle (oracle/estimate_oracle.c), which test_oracle_estimate.py pins to the reference with no GPU."""
import os

import numpy as np
import pytest

import estimate_testlib as et
import kmc_b200
from kmc_b200 import ERR_INVALID, FASTQ, FastxParser, HistogramEstimator, KmcB200Error
from kmc_b200.reads import count_reads, main as reads_main

pytestmark = pytest.mark.gpu
GOLDEN = et.load_golden()


def _counters_equal_oracle(est, batch, k, s):
    got = et.SparseCounters.from_dense(est.read().reshape(-1))
    want = et.SparseCounters(et.oracle_increments(batch, k, s))
    assert np.array_equal(got.index, want.index) and np.array_equal(got.value, want.value), "k=%d s=%d: counters differ" % (k, s)
    return want


@pytest.fixture(scope="module")
def small_batch():
    return et.case_batch({"gen": {"kind": "reads", "seed": 901, "n_reads": 300, "read_len": [50, 600], "lower_frac": 0.05, "n_frac": 0.01}})


@pytest.mark.parametrize("case", [c for c in GOLDEN["cli"] + GOLDEN["harness"] if c["md5"]], ids=lambda c: c["name"])
def test_stored_cases(case):
    batch = et.case_batch(case)
    est = HistogramEstimator(case["k"], case["s"], max_batch_bytes=max(len(batch), 1))
    est.add(batch)
    hist = est.histogram()
    assert est.kernel_launches() == (2 if batch else 1)
    assert et.md5(et.hist_text(hist)) == case["md5"]
    est.close()


def test_value_histograms_equal_the_oracle_at_every_k(small_batch):
    for k in range(1, 257):
        est = HistogramEstimator(k, 7, max_batch_bytes=len(small_batch))
        est.add(small_batch)
        assert np.array_equal(est.histogram(), et.oracle_histogram(small_batch, k, 7)), "k=%d" % k
        est.close()


# every k mod 31 and k mod 33 class the rotations of R^k depend on near the window sizes, and both ends of the k range
FULL_KS = [1, 2, 5, 13, 21, 30, 31, 32, 33, 34, 62, 63, 64, 65, 66, 96, 99, 127, 128, 129, 200, 255, 256]


@pytest.mark.parametrize("s", [7, 11])
@pytest.mark.parametrize("k", FULL_KS)
def test_full_counters_equal_the_oracle(small_batch, k, s):
    est = HistogramEstimator(k, s, max_batch_bytes=len(small_batch))
    est.add(small_batch)
    want = _counters_equal_oracle(est, small_batch, k, s)
    assert np.array_equal(est.histogram(), et.oracle_recursion(*want.value_histograms(), s))
    est.close()


def test_entry_points_agree(small_batch):
    import torch
    k, s = 31, 7
    a = HistogramEstimator(k, s, max_batch_bytes=len(small_batch))
    a.add(small_batch)
    want = a.read()
    # many batches, cut between records
    b = HistogramEstimator(k, s, max_batch_bytes=len(small_batch))
    cuts = [0] + [i + 1 for i in range(len(small_batch)) if small_batch[i] == 10][::37] + [len(small_batch)]
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        b.add(small_batch[lo:hi])
    assert np.array_equal(b.read(), want)
    # device batches on a torch stream
    b.reset()
    assert not b.read().any()
    d = torch.frombuffer(bytearray(small_batch), dtype=torch.uint8).cuda()
    st = torch.cuda.Stream()
    half = cuts[len(cuts) // 2]
    b.dev_add(d.data_ptr(), half, st.cuda_stream)
    b.dev_add(d.data_ptr() + half, len(small_batch) - half, st.cuda_stream)
    assert np.array_equal(b.read(), want)
    # raw FASTQ in chunks through the GPU parser
    reads = [r for r in small_batch.split(b"\n") if r]
    fq = et.fastq_text(reads)
    c = HistogramEstimator(k, s, max_batch_bytes=len(fq) + 1)
    p = FastxParser(FASTQ, max_chunk_bytes=len(fq))
    pos, recs = 0, 0
    while pos < len(fq):
        end = min(len(fq), pos + 20_000)
        pos += c.add_fastx(p, fq[pos:end], end == len(fq))
        recs += c.last_records
    assert recs == len(reads)
    assert np.array_equal(c.read(), want)
    assert np.array_equal(c.histogram(), a.histogram())
    for h in (a, b, c, p):
        h.close()


def test_long_read_crosses_tile_seams():
    read = et.make_reads(902, 1, 5_000_000, genome_len=6_000_000, n_frac=0.0)[0]
    batch = read + b"\n"
    for k, s in ((21, 7), (128, 7), (256, 11)):
        est = HistogramEstimator(k, s, max_batch_bytes=len(batch))
        est.add(batch)
        _counters_equal_oracle(est, batch, k, s)
        est.close()


def test_lower_case_and_separators(small_batch):
    upper = small_batch.upper()
    mixed = bytearray(small_batch.lower())
    mixed[::997] = b"x" * len(mixed[::997])                               # foreign bytes separate like N
    for k in (5, 31, 100):
        a = HistogramEstimator(k, 7, max_batch_bytes=len(upper))
        a.add(upper)
        b = HistogramEstimator(k, 7, max_batch_bytes=len(upper))
        b.add(small_batch.lower())
        assert np.array_equal(a.read(), b.read())
        b.reset()
        b.add(bytes(mixed))
        _counters_equal_oracle(b, bytes(mixed), k, 7)
        a.close()
        b.close()


def test_parameters_and_lifecycle():
    for kw in ({"kmer_len": 0}, {"kmer_len": 257}, {"s": 8}, {"s": 0}, {"max_batch_bytes": 0}, {"max_batch_bytes": (1 << 31) + 1}):
        args = dict(kmer_len=21, s=7, max_batch_bytes=1024)
        args.update(kw)
        with pytest.raises(KmcB200Error) as e:
            HistogramEstimator(**args)
        assert e.value.code == ERR_INVALID
    est = HistogramEstimator(21, 7, max_batch_bytes=16)
    with pytest.raises(KmcB200Error):
        est.add(b"A" * 17)
    assert list(est.histogram()) == [0, 0, 0]                           # no k-mers: max_occ 2, all zeros
    est.close()
    est.close()
    for _ in range(3):                                                  # 1 GiB each: destroyed handles give their memory back
        HistogramEstimator(21, 11, max_batch_bytes=1 << 20).close()


def _write(tmp_path, case):
    path = str(tmp_path / ("in." + case["format"]))
    with open(path, "wb") as f:
        f.write(et.case_text(case))
    return path


@pytest.mark.parametrize("case", [c for c in GOLDEN["cli"] if c["md5"] and c["name"].startswith(("long_k21", "long_k128", "max_occ"))],
                         ids=lambda c: c["name"])
def test_cli_histogram_file_equals_kmc_e(tmp_path, case):
    path = _write(tmp_path, case)
    for parse in ([], ["--gpu-parse", "--batch-bytes", str(1 << 20)]):
        out = str(tmp_path / "hist.txt")
        assert reads_main(["-e", "-k%d" % case["k"]] + parse + [path, out]) == 0
        assert et.md5(open(out, "rb").read()) == case["md5"]
    with pytest.raises(SystemExit):
        reads_main(["-e", "-b", "-k21", path, str(tmp_path / "x.txt")])


@pytest.mark.parametrize("case", GOLDEN["db"], ids=lambda c: c["name"])
@pytest.mark.parametrize("opt", [False, True])
@pytest.mark.parametrize("parse", ["host", "gpu"])
def test_count_reads_chooses_the_lut_prefix_len_as_kmc(tmp_path, case, opt, parse):
    path = _write(tmp_path, case)
    ci = int(next(a for a in case["args"] if a.startswith("-ci"))[3:])
    n_bins = int(next(a for a in case["args"] if a.startswith("-n"))[2:])
    out = str(tmp_path / "db")
    res = count_reads([path], out, case["k"], 9, None, None, cutoff_min=ci, n_bins=n_bins, parse=parse, opt_out_size=opt,
                      batch_bytes=1 << 22)
    assert res["n_reads"] == case["gen"]["n_reads"]
    want = case["opt" if opt else "default"]
    for ext in ("kmc_pre", "kmc_suf"):
        assert et.md5(open(out + "." + ext, "rb").read()) == want[ext], "%s %s: .%s differs (lp %d)" % (case["name"], opt, ext, res["lut_prefix_len"])
    if case["name"] == "lp_changes_k30":
        assert res["lut_prefix_len"] == (6 if opt else 2)


def test_opt_out_size_refused_where_kmc_refuses(tmp_path):
    case = GOLDEN["db"][0]
    path = _write(tmp_path, case)
    with pytest.raises(KmcB200Error):
        count_reads([path], str(tmp_path / "a"), 9, 9, None, None, opt_out_size=True)               # small-k path
    with pytest.raises(KmcB200Error):
        count_reads([path], str(tmp_path / "b"), 31, 9, None, None, both_strands=False, opt_out_size=True)
    with pytest.raises(SystemExit):
        reads_main(["-k31", "--opt-out-size", "--lut-prefix-len", "7", path, str(tmp_path / "c")])
