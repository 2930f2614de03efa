"""Homopolymer compression on the GPU (`kmc -hc`, hc.cuh): the compaction alone on a resident batch, and reads -> database with and
without it.

    python scripts/hc_bench.py --out DIR [--bases 1e9] [--reps 30]

Reports, into DIR/hc_bench.json and one JSON line on stdout:
  * the compaction on one resident batch of 2^28 - 1024 bytes (about 2.7e8 bases), for split_bench.py's 150-bp reads and for long-read-like
    input (20 kb reads, homopolymer runs of geometric length, mean 2): the median of `reps` CUDA-event timings of a small-k add at k = 1
    with compression on minus the same with it off, and the three kernels' own times from torch.profiler in a separate pass; the bytes
    the compaction moves (the batch read twice, the kept bytes and the padding written) over that time, and their share of 3.35 TB/s;
  * `bases` of 150-bp FASTQ -> database (k = 31, the map chosen from the reads, parse="gpu") with and without homopolymer_compressed;
  * the card's name and power limit, read in the same run.
The compressed batch is checked against the numpy model (tests/hc_testlib.py) through the k = 1 counts.  Scratch files go to a temporary
directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from split_bench import gpu_info, synth_batch, write_fastq  # noqa: E402

HBM_BYTES_PER_S = 3.35e12                                              # H100 SXM data sheet
HC_KERNELS = ("hc_count_kernel", "split_scan_top_kernel", "hc_compact_kernel")


def long_read_batch(seed, n_bytes, read_len=20_000):
    """Reads of read_len bytes, '\\n' after each, made of runs of one base (no two neighbouring runs of the same base) of geometric
    length with mean 2."""
    rng = np.random.default_rng(seed)
    n_runs = n_bytes // 2 + 1024
    steps = rng.integers(1, 4, n_runs, dtype=np.uint8)
    bases = np.cumsum(steps, dtype=np.uint64) % 4
    seq = np.repeat(np.frombuffer(b"ACGT", dtype=np.uint8)[bases.astype(np.int64)], rng.geometric(0.5, n_runs))[:n_bytes]
    seq[read_len::read_len + 1] = 10
    seq[-1] = 10
    return seq


def cuda_time(fn, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    return float(np.median(times))


def compaction(batch, reps, tmp):
    import torch
    import kmc_b200
    from hc_testlib import homopolymer_compress
    d_seq = torch.from_numpy(batch).cuda()
    sk = kmc_b200.SmallKCounter(1, max_batch_bytes=batch.size)
    add = lambda: sk.dev_add(d_seq.data_ptr(), batch.size, None)
    add()
    t_off = cuda_time(add, reps)
    sk.set_homopolymer_compressed(True)
    sk.reset()
    add()
    kept = homopolymer_compress(batch)
    code = np.full(256, 4, dtype=np.uint8)
    code[np.frombuffer(b"ACGTacgt", np.uint8)] = [0, 1, 2, 3, 0, 1, 2, 3]
    per_base = np.bincount(code[kept], minlength=5)
    want = np.array([per_base[0] + per_base[3], per_base[1] + per_base[2], 0, 0], dtype=np.uint64)   # k = 1, canonical
    assert np.array_equal(sk.read(), want), "GPU compression differs from the model"
    t_on = cuda_time(add, reps)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            add()
        torch.cuda.synchronize()
    per = {n: 0.0 for n in HC_KERNELS}
    for e in prof.key_averages():
        for n in HC_KERNELS:
            if n in e.key:
                per[n] += e.device_time_total / 1e6 / reps
    sk.close()
    t_kernels = sum(per.values())
    moved = 2 * batch.size + batch.size                                # read twice; kept bytes + padding = the batch's length, written
    return {"bytes": int(batch.size), "kept": int(kept.size), "smallk_add_off_s": t_off, "smallk_add_on_s": t_on,
            "compaction_s_events": t_on - t_off, "kernel_s": per, "compaction_s_kernels": t_kernels, "bytes_moved": moved,
            "bytes_per_s": moved / t_kernels, "share_of_hbm_peak": moved / t_kernels / HBM_BYTES_PER_S}


def end_to_end(tmp, n_bases):
    from kmc_b200.reads import count_reads
    fq = os.path.join(tmp, "reads.fq")
    write_fastq(fq, synth_batch(11, n_bases, 150, genome_len=200_000_000), 150)
    out = {"bases": n_bases, "fastq_bytes": os.path.getsize(fq)}
    for hc in (False, True, False, True):
        t0 = time.perf_counter()
        r = count_reads([fq], os.path.join(tmp, "db%d" % hc), 31, 9, None, None, parse="gpu", batch_bytes=1 << 28, homopolymer_compressed=hc)
        out.setdefault("hc%d_s" % hc, []).append(time.perf_counter() - t0)
        out["hc%d_n_kmers" % hc] = r["n_kmers"]
        for key in ("stats_s", "split_s", "stage2_s", "read_s"):
            out.setdefault("hc%d_%s" % (hc, key), []).append(r[key])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bases", type=float, default=1e9)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info()}
    n = (1 << 28) - 1024
    with tempfile.TemporaryDirectory() as tmp:
        res["short_reads"] = compaction(synth_batch(10, n, 150)[:n], a.reps, tmp)
        res["long_reads"] = compaction(long_read_batch(12, n), a.reps, tmp)
        res["end_to_end"] = end_to_end(tmp, int(a.bases))
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "hc_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
