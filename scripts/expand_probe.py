"""Development probe: time of the index + expand stage alone (kmcb200_dev_expand) for the library named by KMCB200_LIB."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch, kmc_b200
from kmc_testlib import fast_bin
n_rec = 1 << 26
dev = torch.device("cuda", 0)
hb = fast_bin(1000, 31, n_rec)
d_bin = torch.zeros(hb.size + 64, dtype=torch.uint8, device=dev); d_bin[:hb.size] = torch.from_numpy(hb.data).to(dev)
d_recs = torch.zeros(n_rec, dtype=torch.int64, device=dev)
d_res = torch.zeros(8, dtype=torch.int64, device=dev)
ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(31, True, 2, 10 ** 9, 255, 7), device=0, n_slots=1)
st = torch.cuda.Stream(device=dev); torch.cuda.set_stream(st)
for _ in range(3): ctx.dev_expand(0, d_bin.data_ptr(), hb.size, n_rec, hb.pack_bytes, d_recs.data_ptr(), d_res.data_ptr(), st.cuda_stream)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(20): ctx.dev_expand(0, d_bin.data_ptr(), hb.size, n_rec, hb.pack_bytes, d_recs.data_ptr(), d_res.data_ptr(), st.cuda_stream)
e1.record(); torch.cuda.synchronize()
print("%s: index + expand %.3f ms per bin, status %s, checksum %x" % (os.environ.get("KMCB200_LIB", "main"), e0.elapsed_time(e1) / 20, d_res.cpu().numpy()[[3, 6]].tolist(), int(d_recs.sum().item()) & 0xffffffffffff))
