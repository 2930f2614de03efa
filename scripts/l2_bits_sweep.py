"""Sweep of the second partition level's width (KMCB200_L2_BITS) over the bin sizes of bench.py's workload: device time of one whole
bin (kmcb200_dev_process_bin, CUDA events, median of REPS after WARM) with 8, 9 and 10 bits forced and with the default rule (choose_b2),
for k = 31 over the 8 pool sizes and for k = 55 at 2^28 k-mers.  Every setting must give the same result words as the default.
Prints one JSON line.  Usage: python scripts/l2_bits_sweep.py [--reps N]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

WARM = 2


def time_bin(kmc_b200, torch, k, b, bits, reps):
    if bits:
        os.environ["KMCB200_L2_BITS"] = str(bits)
    else:
        os.environ.pop("KMCB200_L2_BITS", None)
    ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(k, True, 2, 10 ** 9, 255, 7), device=0, n_slots=1)
    os.environ.pop("KMCB200_L2_BITS", None)
    cap = ctx.out_capacity(b.n_rec) + 64
    d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device="cuda")
    d_bin[:b.size] = torch.from_numpy(b.data).cuda()
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device="cuda")
    d_res = torch.zeros(8, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()               # the inputs are written on torch's stream
    tstream = torch.cuda.Stream()          # a real stream: with stream 0 the library enqueues on its own, which these events would not see
    ms = []
    for i in range(WARM + reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(tstream)
        ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, b.n_rec, b.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(), tstream.cuda_stream)
        e1.record(tstream)
        torch.cuda.synchronize()
        if i >= WARM:
            ms.append(e0.elapsed_time(e1))
    res = [int(x) for x in d_res.cpu().numpy()]
    ctx.close()
    del d_bin, d_out
    torch.cuda.empty_cache()
    return statistics.median(ms), res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import torch
    import kmc_b200
    import bench
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    rows = []
    cases = [(31, n, 4000 + j) for j, n in enumerate(bench.pool_sizes(1))] + [(55, 1 << 28, 3000)]
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(min(32, os.cpu_count() or 8)) as ex:
        for k, n, seed in cases:
            b = bench.gen_bin(seed, k, n, ex)
            row = {"k": k, "n_rec": n}
            base_ms, base_res = time_bin(kmc_b200, torch, k, b, 0, args.reps)
            row["default_ms"] = base_ms
            for bits in (8, 9, 10):
                ms, res = time_bin(kmc_b200, torch, k, b, bits, args.reps)
                assert res[:7] == base_res[:7], (k, n, bits, res, base_res)
                row["bits%d_ms" % bits] = ms
            rows.append(row)
            del b
    print(json.dumps({"gpu": gpu, "reps": args.reps, "rows": rows}))


if __name__ == "__main__":
    main()
