"""Oversized bins on the hardware (SURVEY 8f N1): one bin of 2^LG k-mers (default 2^31 = 2.1e9 k-mers, 2.2 GB of super-k-mer bytes,
17 GB of records) through kmcb200_process_bin
  (a) in one shot - the block limit comes from the free HBM, so a GPU whose free HBM holds it sorts it as ONE bin (one expansion, no key blocks),
  (b) as key blocks of <= 2^(LG-2) k-mers (KMCB200_MAX_BLOCK_RECORDS): one counting expansion + one filtered expansion per block,
      asynchronous block loop, LUT / statistics accumulated on the device,
and checks that (b) is byte-identical to (a) and that both satisfy the size-independent properties (n_total, sum(LUT) = records,
strictly increasing k-mers, counters >= cutoff).  usage: big_bin_check.py [LG] [k]"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from concurrent.futures import ThreadPoolExecutor
import kmc_b200, bench

lg = int(sys.argv[1]) if len(sys.argv) > 1 else 31
K = int(sys.argv[2]) if len(sys.argv) > 2 else 31
P = 7


def properties(ctx, r, n_rec):
    assert r.n_total == n_rec, (r.n_total, n_rec)
    ob = ctx.out_rec_bytes
    n_emit = r.payload.size // ob
    assert int(r.lut.sum()) == n_emit == r.n_unique - r.n_cutoff_min - r.n_cutoff_max
    rec = r.payload.reshape(n_emit, ob)
    assert rec[:, -1].min() >= 2
    prefix = np.repeat(np.arange(ctx.lut_entries, dtype=np.uint64), r.lut.astype(np.int64))
    sb = ob - 1
    if sb <= 6:          # k = 31: the whole k-mer fits 64 bits
        suf = np.zeros(n_emit, dtype=np.uint64)
        for j in range(sb):
            suf = (suf << np.uint64(8)) | rec[:, j].astype(np.uint64)
        full = (prefix << np.uint64(8 * sb)) | suf
        assert np.all(full[1:] > full[:-1]), "emitted k-mers are not strictly increasing"
    return n_emit


def run(sk, env):
    for k_, v in env.items():
        os.environ[k_] = str(v)
    ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(K, True, 2, 10 ** 9, 255, P), device=0, n_slots=1)
    for k_ in env:
        del os.environ[k_]
    ts = []
    for it in range(2):
        t0 = time.perf_counter()
        r = ctx.process_bin(sk)
        ts.append(time.perf_counter() - t0)
    n_emit = properties(ctx, r, sk.n_rec)
    ctx.close()
    return r, n_emit, min(ts)


with ThreadPoolExecutor(32) as ex:
    sk = bench.gen_bin(4711, K, 1 << lg, ex)
print("bin: 2^%d k-mers, %.2f GB of super-k-mer bytes, %d packs" % (lg, sk.size / 1e9, sk.pack_bytes.size), flush=True)
a, na, ta = run(sk, {})
print("one shot   : %.1f ms host-to-host (pageable buffers) = %.3g k-mers/s, %d records" % (ta * 1e3, sk.n_rec / ta, na), flush=True)
for flow, blk in (("scatter", lg - 3), ("filter", lg - 2)):
    b, nb, tb = run(sk, {"KMCB200_MAX_BLOCK_RECORDS": 1 << blk, "KMCB200_KEY_BLOCKS": flow})
    same = na == nb and a.stats == b.stats and np.array_equal(a.lut, b.lut) and a.payload.tobytes() == b.payload.tobytes()
    print("key blocks, %-7s: %.1f ms (<= 2^%d k-mers per block) = %.3g k-mers/s, byte-identical to one shot: %s" % (flow, tb * 1e3, blk, sk.n_rec / tb, same), flush=True)
    assert same
