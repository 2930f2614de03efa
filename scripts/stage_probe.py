"""Development probe: per-stage / per-pass CUDA-event times of one resident bin (k=31, 2^26 k-mers by default)."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch, kmc_b200
from kmc_testlib import fast_bin

n_rec = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 26
k = int(sys.argv[2]) if len(sys.argv) > 2 else 31
p = {31: 7, 55: 7, 28: 4}.get(k, 7)
ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(k, True, 2, 10 ** 9, 255, p), device=0, n_slots=1)
seed = int(sys.argv[3]) if len(sys.argv) > 3 else 1
hb = fast_bin(seed, k, n_rec)
cap = ctx.out_capacity(n_rec) + 64
dev = torch.device("cuda", 0)
d_bin = torch.zeros(hb.size + 64, dtype=torch.uint8, device=dev); d_bin[:hb.size] = torch.from_numpy(hb.data).to(dev)
d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device=dev)
d_res = torch.zeros(8, dtype=torch.int64, device=dev)
st = torch.cuda.Stream(device=dev)
W = 8 * ctx.words
for it in range(5):
    ctx.dev_process_bin(0, d_bin.data_ptr(), hb.size, n_rec, hb.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(), st.cuda_stream)
    torch.cuda.synchronize()
    t = ctx.stage_times(0)
    tot = t["expand_ms"] + t["sort_ms"] + t["count_ms"]
    ps = t["pass_ms"]
    print("it%d total %.3f ms (%.2f G k-mers/s) expand %.3f sort %.3f count %.3f | pass avg %.3f ms = %.0f GB/s | %s" % (
        it, tot, n_rec / tot / 1e6, t["expand_ms"], t["sort_ms"], t["count_ms"], sum(ps) / len(ps), 2 * n_rec * W / (sum(ps) / len(ps)) / 1e6,
        " ".join("%s=%.3f" % (nm, x) for nm, x in zip(t["pass_names"], ps))))
print("result", d_res.cpu().numpy())
