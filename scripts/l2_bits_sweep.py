"""Sweep of the second partition level's width (KMCB200_L2_BITS) over the bin sizes of bench.py's workload: device time of one whole
bin (kmcb200_dev_process_bin, CUDA events, median of REPS after WARM) and the medians of its level-2 and leaf intervals
(msd_count_L2, msd_partition_L2, leaf_count), with each width of --bits forced for each leaf kernel of --kernels (KMCB200_LEAF_KERNEL:
default = the library's rule, cta, hash) and with the default rule (choose_b2), for k = 31 over the 8 pool sizes and, unless
--no-k55, for k = 55 at 2^28 k-mers.  Every setting must give the same result words as the default.
Prints one JSON line.  Usage: python scripts/l2_bits_sweep.py [--reps N] [--bits 8,9,10] [--kernels default]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

WARM = 2


STAGES = ("msd_count_L2", "msd_partition_L2", "leaf_count")


def time_bin(kmc_b200, torch, k, b, bits, reps, kernel="default"):
    if bits:
        os.environ["KMCB200_L2_BITS"] = str(bits)
    else:
        os.environ.pop("KMCB200_L2_BITS", None)
    if kernel != "default":
        os.environ["KMCB200_LEAF_KERNEL"] = kernel
    ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(k, True, 2, 10 ** 9, 255, 7), device=0, n_slots=1)
    os.environ.pop("KMCB200_L2_BITS", None)
    os.environ.pop("KMCB200_LEAF_KERNEL", None)
    cap = ctx.out_capacity(b.n_rec) + 64
    d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device="cuda")
    d_bin[:b.size] = torch.from_numpy(b.data).cuda()
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device="cuda")
    d_res = torch.zeros(8, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()               # the inputs are written on torch's stream
    tstream = torch.cuda.Stream()          # a real stream: with stream 0 the library enqueues on its own, which these events would not see
    ms, stages = [], {nm: [] for nm in STAGES}
    for i in range(WARM + reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(tstream)
        ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, b.n_rec, b.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(), tstream.cuda_stream)
        e1.record(tstream)
        torch.cuda.synchronize()
        if i >= WARM:
            ms.append(e0.elapsed_time(e1))
            st = ctx.stage_times(0)
            iv = dict(zip(st["pass_names"], st["pass_ms"]))
            for nm in STAGES:
                stages[nm].append(iv.get(nm, 0.0))
    res = [int(x) for x in d_res.cpu().numpy()]
    ctx.close()
    del d_bin, d_out
    torch.cuda.empty_cache()
    return statistics.median(ms), {nm: statistics.median(v) for nm, v in stages.items()}, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--bits", default="8,9,10", help="forced widths, comma-separated")
    ap.add_argument("--kernels", default="default", help="leaf kernels (KMCB200_LEAF_KERNEL) to force each width with: default, cta, hash")
    ap.add_argument("--no-k55", action="store_true", help="leave out the k = 55 bin")
    args = ap.parse_args()
    widths = [int(x) for x in args.bits.split(",")]
    kernels = args.kernels.split(",")
    import torch
    import kmc_b200
    import bench
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    rows = []
    cases = [(31, n, 4000 + j) for j, n in enumerate(bench.pool_sizes(1))] + ([] if args.no_k55 else [(55, 1 << 28, 3000)])
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(min(32, os.cpu_count() or 8)) as ex:
        for k, n, seed in cases:
            b = bench.gen_bin(seed, k, n, ex)
            row = {"k": k, "n_rec": n}
            base_ms, base_st, base_res = time_bin(kmc_b200, torch, k, b, 0, args.reps)
            row["default_ms"] = base_ms
            row["default_stages"] = base_st
            for kernel in kernels:
                for bits in widths:
                    ms, st, res = time_bin(kmc_b200, torch, k, b, bits, args.reps, kernel)
                    assert res[:7] == base_res[:7], (k, n, bits, kernel, res, base_res)
                    name = "bits%d" % bits if kernel == "default" else "bits%d_%s" % (bits, kernel)
                    row[name + "_ms"] = ms
                    row[name + "_stages"] = st
            print(json.dumps(row), file=sys.stderr, flush=True)
            rows.append(row)
            del b
    print(json.dumps({"gpu": gpu, "reps": args.reps, "rows": rows}))


if __name__ == "__main__":
    main()
