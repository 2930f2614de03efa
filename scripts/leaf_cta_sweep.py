"""Leaf kernels of one-word records on resident 30x bins: leaf_hash_kernel (KMCB200_LEAF_KERNEL=hash) against leaf_hash_cta_kernel in each
KMCB200_LEAF_CTA shape (warps per CTA : log2 of the table's slots), alternating, with the result words checked against the first config.
Prints per config the step time and the leaf_count interval (CUDA events, mean of STEPS bins after WARM).
Usage (GPU box): [SWEEP_CONFIGS=hash,default,...] python scripts/leaf_cta_sweep.py [k-mers per bin in Mi ...]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import kmc_b200
from kmc_testlib import fast_bin

K, P, WARM, STEPS = 31, 7, 3, 10
CONFIGS = [("hash", {"KMCB200_LEAF_KERNEL": "hash"}), ("default", {}), ("cta 4:12", {"KMCB200_LEAF_KERNEL": "cta", "KMCB200_LEAF_CTA": "4:12"}),
           ("cta 4:10", {"KMCB200_LEAF_KERNEL": "cta", "KMCB200_LEAF_CTA": "4:10"}), ("cta L2=7", {"KMCB200_LEAF_KERNEL": "cta", "KMCB200_L2_BITS": "7"}),
           ("cta L2=6", {"KMCB200_LEAF_KERNEL": "cta", "KMCB200_L2_BITS": "6"})]
if os.environ.get("SWEEP_CONFIGS"):
    CONFIGS = [c for c in CONFIGS if c[0] in os.environ["SWEEP_CONFIGS"].split(",")]
dev = torch.device("cuda", 0)
print(torch.cuda.get_device_name(dev), flush=True)


def run(n_rec, d_bins, bins, env):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(K, True, 2, 10 ** 9, 255, P), device=0, n_slots=1)
    for k, v in saved.items():
        if v is None:
            del os.environ[k]
        else:
            os.environ[k] = v
    cap = ctx.out_capacity(n_rec) + 64
    d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device=dev)
    d_res = torch.zeros(8, dtype=torch.int64, device=dev)
    st = torch.cuda.Stream(device=dev)
    leaf_ms, res = [], None
    with torch.cuda.stream(st):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for i in range(WARM + STEPS):
            if i == WARM:
                e0.record(st)
            hb = bins[i % 2]
            ctx.dev_process_bin(0, d_bins[i % 2].data_ptr(), hb.size, n_rec, hb.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(), st.cuda_stream)
            if i >= WARM:
                st.synchronize()
                s = ctx.stage_times(0)
                leaf_ms.append(dict(zip(s.get("pass_names") or [], s["pass_ms"])).get("leaf_count", 0.0))
            if i == 0:
                st.synchronize()
                res = [int(x) for x in d_res.cpu().tolist()]
        e1.record(st)
        st.synchronize()
    ctx.close()
    # (the step time includes the synchronisations that read the stage intervals)
    return e0.elapsed_time(e1) / STEPS, sum(leaf_ms) / len(leaf_ms), res


for mi in [int(x) for x in sys.argv[1:]] or [32, 128, 256]:
    n_rec = mi << 20
    bins = [fast_bin(1000 + j, K, n_rec) for j in range(2)]
    d_bins = []
    for hb in bins:
        t = torch.zeros(hb.size + 64, dtype=torch.uint8, device=dev)
        t[:hb.size] = torch.from_numpy(hb.data).to(dev)
        d_bins.append(t)
    ref = None
    for rep in range(2):
        for name, env in CONFIGS:
            step, leaf, res = run(n_rec, d_bins, bins, env)
            ref = ref or res
            print("%d Mi %-9s rep %d: %.3f ms/bin  leaf_count %.3f ms  fallback=%d  same=%s" % (mi, name, rep, step, leaf, res[7], res == ref), flush=True)
    del d_bins
    torch.cuda.empty_cache()
