"""Stage 0 on the GPU: signature statistics (kmcb200_dev_sigstats_add) over one resident batch, next to split_signature_kernel alone.

    python scripts/sigstats_bench.py --out DIR [--bases 2.7e8] [--reps 20]

One batch of 150-bp reads (k = 31, p = 9) stays in HBM.  Reported, into DIR/sigstats_bench.json and one JSON line on stdout:
  * sigstats_kernel: median time of one kmcb200_dev_sigstats_add over the batch (CUDA events around each call), and bases/s;
  * split_signature_kernel: its time on the same batch, from torch.profiler (CUDA activity) over a profiled kmcb200_dev_split, since the
    split launches it as the first of its kernels; and sigstats_kernel's profiled time from the same kind of run;
  * the card's name, power limit and top SM clock, read in the same run.
Both kernels build the same windowed minimum per tile; the statistics then add runs into 4^p + 1 counters instead of writing a
signature word per position.  The counts are checked against a CPU count of a slice of the batch before anything is timed.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

K, P = 31, 9


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def profiled_ms(fn, key):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ms = [ev.device_time_total / 1e3 for ev in prof.events() if ev.device_type.name == "CUDA" and key in ev.name]
    return sum(ms) if ms else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bases", type=float, default=2.7e8)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    import torch
    import kmc_b200
    from split_bench import synth_batch
    from stage0_testlib import oracle_signature_stats
    from stage1_testlib import random_map
    res = {"gpu": gpu_info(), "k": K, "signature_len": P}
    batch = synth_batch(1, int(a.bases), 150)
    dev = torch.device("cuda:0")
    d_seq = torch.from_numpy(batch).to(dev)
    st = kmc_b200.SignatureStats(K, P, max_batch_bytes=batch.size)
    # correctness on a slice first (the CPU oracle is sequential)
    piece = batch[:151 * 20000]
    st.dev_add(d_seq.data_ptr(), piece.size, None)
    assert np.array_equal(st.read(), oracle_signature_stats(piece, K, P)), "GPU statistics differ from the oracle"
    st.reset()
    run = lambda: st.dev_add(d_seq.data_ptr(), batch.size, None)
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(a.reps):
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    t = float(np.median(times))
    counts = st.read()
    res["sigstats"] = {"bases": int(batch.size), "kmers_counted": int(counts.sum(dtype=np.uint64)), "ms_median": t, "ms_all": times,
                       "bases_per_s": batch.size / (t / 1e3), "profiled_kernel_ms": profiled_ms(run, "sigstats_kernel")}
    # split_signature_kernel alone, from a profiled split of the same batch (sizing run: no outputs, the kernel's work is the same)
    n_bins = 512
    sp = kmc_b200.Splitter(K, P, random_map(1, P, n_bins), n_bins, max_batch_bytes=batch.size)
    d_res = torch.zeros(8, dtype=torch.int64, device=dev)
    d_frags = torch.zeros(n_bins * 5, dtype=torch.int64, device=dev)
    split = lambda: sp.dev_split(d_seq.data_ptr(), batch.size, 0, 0, 0, 0, d_frags.data_ptr(), d_res.data_ptr(), None)
    for _ in range(2):
        split()
    torch.cuda.synchronize()
    sig_ms = [profiled_ms(split, "split_signature_kernel") for _ in range(3)]
    ref = float(np.median(sig_ms))
    res["split_signature_kernel"] = {"ms_profiled": sig_ms, "bases_per_s": batch.size / (ref / 1e3)}
    res["sigstats_over_split_signature"] = (res["sigstats"]["profiled_kernel_ms"] or t) / ref
    sp.close()
    st.close()
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "sigstats_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
