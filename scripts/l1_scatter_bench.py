"""Level 1 of a k=31 bin, two ways, on resident bins of bench.py's workload (same generator and seed family), in the library named by
KMCB200_LIB (default: the package's):
  new: index, whose pack walk counts the level-1 digit totals (`expand` interval of kmcb200_dev_process_bin), and the bucket bounds +
       the one expansion that writes every k-mer into its level-1 bucket (`expand_scatter_L1`), the bin path;
  old: index + expand_kernel<kExpandAll> (`expand` of kmcb200_dev_expand) and msd_partition_kernel (`msd_partition_L1` of
       kmcb200_dev_sort with hist_ready), the sequence kmcb200_dev_expand's callers still get.
Every interval is the median of REPS CUDA-event intervals.  The payload, the LUT and the 8 result words of the two paths are compared
(the old path counts with kmcb200_dev_count).  Algorithmic bytes: S = bin bytes, N = k-mers, 8-byte records:
  index + digit totals: S;  scatter: S + 8N;  old expand: S + 8N;  old partition: 16N.
Usage (GPU): python scripts/l1_scatter_bench.py [k-mers per bin, in Mi or as 2^x ...]"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

import kmc_b200
from bench import gen_bin

K, P, WARM, REPS = 31, 7, 2, 11
PEAK_GBS = 3350.0          # H100 SXM data sheet (HBM3)
MI = 1 << 20


def parse_size(s):
    return 1 << int(s[2:]) if s.startswith("2^") else int(s) * MI


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # (the power limit is then unknown: say so)
        q = "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)
    return q


def med(xs):
    return float(np.median(np.asarray(xs)))


def run_size(n_rec, seed):
    dev = torch.device("cuda", 0)
    with ThreadPoolExecutor(min(32, os.cpu_count() or 8)) as ex:
        b = gen_bin(seed, K, n_rec, ex)
    ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(K, True, 2, 10 ** 9, 255, P), device=0, n_slots=1)
    cap = ctx.out_capacity(n_rec) + 64
    d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device=dev)
    d_bin[:b.size] = torch.from_numpy(b.data).to(dev)
    outs = [torch.zeros(cap, dtype=torch.uint8, device=dev) for _ in range(2)]
    luts = [torch.zeros(ctx.lut_entries, dtype=torch.int64, device=dev) for _ in range(2)]
    ress = [torch.zeros(8, dtype=torch.int64, device=dev) for _ in range(2)]
    d_recs = torch.zeros(n_rec + 8, dtype=torch.int64, device=dev)
    d_tmp = torch.zeros(n_rec + 8, dtype=torch.int64, device=dev)
    d_eres = torch.zeros(8, dtype=torch.int64, device=dev)
    stream = torch.cuda.Stream(device=dev)
    st = stream.cuda_stream
    new_idx, new_sc, old_exp, old_part, launches = [], [], [], [], None
    with torch.cuda.stream(stream):
        for i in range(WARM + REPS):
            l0 = ctx.kernel_launches()
            ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, n_rec, b.pack_bytes, outs[0].data_ptr(), cap, luts[0].data_ptr(), ress[0].data_ptr(), st)
            launches = ctx.kernel_launches() - l0
            stream.synchronize()
            t = ctx.stage_times(0)
            iv = dict(zip(t["pass_names"], t["pass_ms"]))
            if i >= WARM:
                new_idx.append(t["expand_ms"])
                new_sc.append(iv["expand_scatter_L1"])
            ctx.dev_expand(0, d_bin.data_ptr(), b.size, n_rec, b.pack_bytes, d_recs.data_ptr(), d_eres.data_ptr(), st)
            where = ctx.dev_sort(0, d_recs.data_ptr(), d_tmp.data_ptr(), n_rec, hist_ready=True, stream=st)
            stream.synchronize()
            t = ctx.stage_times(0)
            iv = dict(zip(t["pass_names"], t["pass_ms"]))
            if i >= WARM:
                old_exp.append(t["expand_ms"])
                old_part.append(iv["msd_partition_L1"])
            srt = d_tmp if where == 1 else d_recs
            ctx.dev_count(0, srt.data_ptr(), n_rec, outs[1].data_ptr(), cap, luts[1].data_ptr(), ress[1].data_ptr(), st)
            stream.synchronize()
    r_new, r_old = [int(x) for x in ress[0].cpu()], [int(x) for x in ress[1].cpu()]
    nb = r_new[4] * ctx.out_rec_bytes
    same = (r_new == r_old and torch.equal(luts[0], luts[1]) and torch.equal(outs[0][:nb], outs[1][:nb]))
    ctx.close()
    S, N = b.size, n_rec
    rows = [("new index + totals", med(new_idx), S), ("new expand_scatter_L1", med(new_sc), S + 8 * N),
            ("old index + expand", med(old_exp), S + 8 * N), ("old msd_partition_L1", med(old_part), 16 * N)]
    print("n = %d k-mers (%.3g), S = %d bin bytes, %d launches per bin, lsd_fallback %d, results identical: %s, words %s"
          % (N, N, S, launches, r_new[7], same, r_new), flush=True)
    for name, ms, byt in rows:
        print("  %-24s %7.3f ms  %8.1f GB/s  %.2f of %.0f GB/s" % (name, ms, byt / (ms * 1e-3) / 1e9, byt / (ms * 1e-3) / 1e9 / PEAK_GBS, PEAK_GBS), flush=True)
    new_t, old_t = rows[0][1] + rows[1][1], rows[2][1] + rows[3][1]
    print("  level 1 in all: new %.3f ms, old %.3f ms (%.1f %%)" % (new_t, old_t, 100.0 * (new_t / old_t - 1.0)), flush=True)
    del d_bin, outs, luts, d_recs, d_tmp
    torch.cuda.empty_cache()
    return same and r_new[7] == 0


def main():
    print("card (name, power limit, max SM clock): %s" % card(), flush=True)
    print("library: %s" % kmc_b200.LIB_PATH, flush=True)
    sizes = [parse_size(s) for s in sys.argv[1:]] or [1 << 25, 1 << 26, 1 << 27, 112 * MI, 1 << 28]
    ok = True
    for j, n in enumerate(sizes):
        ok &= run_size(n, 4100 + j)
    print("all results identical" if ok else "RESULTS DIFFER", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
