"""Histogram estimation on the GPU (kmcb200_estimator_*): hash kernel times, the counter scan, the host recursion, FASTQ -> `-e` file, and
count_reads(opt_out_size=True) against the same run without it.

    python scripts/estimate_bench.py --out DIR [--bases 1e9] [--reps 20]

Reports, into DIR/estimate_bench.json and one JSON line on stdout:
  * the hash kernel on one resident batch (split_bench.py's 150-bp reads, 2^28 - 1024 bytes, about 2.7e8 bases) at k in {21, 31, 55, 128}
    with s = 7 and s = 11: median of `reps` CUDA-event timings of kmcb200_dev_estimator_add;
  * the counter scan (estimate_hist_kernel, 1 GiB read) and the host recursion, from kmcb200_estimator_histogram timed with CUDA events and
    a host clock;
  * `bases` of 150-bp FASTQ -> histogram file with estimate_histogram(parse="gpu") at k = 31, and kmc_ref -e on the host's cores where
    oracle/_ref/kmc_ref exists;
  * count_reads(opt_out_size=True) and the same run without it (lut_prefix_len=None), on a tenth of those bases, k = 31;
  * the card's name and power limit, read in the same run.
Every resident result is checked against the oracle (oracle/estimate_oracle.c), the end-to-end file against kmc_ref -e's.  Scratch files go
to a temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from split_bench import gpu_info, synth_batch, write_fastq  # noqa: E402

KS = (21, 31, 55, 128)
KMC_REF = os.path.join(ROOT, "oracle", "_ref", "kmc_ref")


def cuda_time(fn, reps, before=None):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        if before:
            before()
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    return float(np.median(times)), times


def resident(batch, reps):
    import torch
    import kmc_b200
    import estimate_testlib as et
    d_seq = torch.from_numpy(batch).cuda()
    out = {}
    for s in (7, 11):
        for k in KS:
            est = kmc_b200.HistogramEstimator(k, s, max_batch_bytes=batch.size)
            run = lambda: est.dev_add(d_seq.data_ptr(), batch.size, None)
            run()
            torch.cuda.synchronize()
            hist = est.histogram()
            assert np.array_equal(hist, et.oracle_histogram(batch, k, s)), "k=%d s=%d: GPU estimate differs from the oracle" % (k, s)
            t, times = cuda_time(run, reps, est.reset)
            r = {"hash_s_median": t, "hash_s_all": times, "bases_per_s": batch.size / t, "max_occ": int(hist.size - 1)}
            if k == 31:
                t_hist, _ = cuda_time(lambda: est.histogram(), 5)
                h0 = time.perf_counter()
                est.histogram()
                r["histogram_call_s"] = time.perf_counter() - h0
                r["histogram_call_s_events"] = t_hist
            out["k%d_s%d" % (k, s)] = r
            est.close()
    return out


def scan_and_recursion(reps):
    """The counter scan alone (events around the histogram call minus nothing: the recursion at max_occ = 2 is negligible), and the
    recursion at max_occ = 65536, timed through the oracle-equal host code of kmcb200_estimator_histogram on a one-k-mer input."""
    import torch
    import kmc_b200
    import estimate_testlib as et
    est = kmc_b200.HistogramEstimator(21, 7, max_batch_bytes=1 << 20)
    t_scan, _ = cuda_time(lambda: est.histogram(), reps)
    case = next(c for c in et.load_golden()["cli"] if c["name"] == "max_occ_k21")
    batch = et.case_batch(case)
    est.close()
    est = kmc_b200.HistogramEstimator(21, 7, max_batch_bytes=len(batch))
    est.add(batch)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hist = est.histogram()
    t_rec = time.perf_counter() - t0
    assert et.md5(et.hist_text(hist)) == case["md5"], "max_occ case differs from the stored kmc -e file"
    est.close()
    return {"scan_1GiB_s_median": t_scan, "scan_bytes_per_s": 2 ** 30 / t_scan, "histogram_call_at_max_occ_65536_s": t_rec,
            "max_occ": int(hist.size - 1)}


def end_to_end(tmp, n_bases):
    from kmc_b200.reads import count_reads, estimate_histogram, write_histogram
    import estimate_testlib as et
    fq = os.path.join(tmp, "reads.fq")
    write_fastq(fq, synth_batch(11, n_bases, 150, genome_len=200_000_000), 150)
    out = {"bases": n_bases, "fastq_bytes": os.path.getsize(fq)}
    t0 = time.perf_counter()
    hist = estimate_histogram([fq], 31, parse="gpu", batch_bytes=1 << 28)
    out["gpu_e_s"] = time.perf_counter() - t0
    write_histogram(os.path.join(tmp, "gpu.txt"), hist)
    if os.path.exists(KMC_REF):
        t0 = time.perf_counter()
        subprocess.run([KMC_REF, "-k31", "-fq", "-e", "-t%d" % os.cpu_count(), fq, os.path.join(tmp, "ref.txt"), tmp], check=True,
                       stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        out["kmc_ref_e_s"] = time.perf_counter() - t0
        out["kmc_ref_threads"] = os.cpu_count()
        assert open(os.path.join(tmp, "ref.txt"), "rb").read() == open(os.path.join(tmp, "gpu.txt"), "rb").read(), "-e file differs from kmc_ref's"
        out["equal_to_kmc_ref"] = True
    small = os.path.join(tmp, "small.fq")
    write_fastq(small, synth_batch(12, n_bases // 10, 150, genome_len=50_000_000), 150)
    for opt in (False, True):
        t0 = time.perf_counter()
        r = count_reads([small], os.path.join(tmp, "db%d" % opt), 31, 9, None, None, parse="gpu", batch_bytes=1 << 28, opt_out_size=opt)
        out["count_reads_opt%d_s" % opt] = time.perf_counter() - t0
        out["count_reads_opt%d_lp" % opt] = r["lut_prefix_len"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bases", type=float, default=1e9)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info()}
    batch = synth_batch(10, (1 << 28) - 1024, 150)
    res["resident"] = resident(batch, a.reps)
    res["scan"] = scan_and_recursion(a.reps)
    with tempfile.TemporaryDirectory() as tmp:
        res["end_to_end"] = end_to_end(tmp, int(a.bases))
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "estimate_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
