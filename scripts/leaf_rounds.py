"""How many table rounds each record of bench.py's pool needs (CPU only, no GPU): expands every pool bin (the seeded generator of bench.py,
--scale 1 by default), takes the leaves as the top 8 + b2 bits of the canonical k-mers (b2 as choose_b2 picks it) and applies the round
planning of the leaf kernels: a leaf of m records with d distinct k-mers per record is counted in 2^e0 rounds, e0 the least e with
m >> e <= fill * slots / d (e0 <= 8), every round reading the whole leaf.  A round whose distinct k-mers pass 7/8 of the slots is split
again (counted as one more read of its records; the even-split estimate).
Usage: python scripts/leaf_rounds.py [scale]"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench
from kmc_testlib import Oracle, Params

FILL = 0.62
TABLES = [("warp table, 1024 slots", 1024), ("CTA table, 4096 slots", 4096)]


def b2_for(n):
    lg = 0
    while (1 << lg) < (n + 1023) // 1024:
        lg += 1
    return min(max(lg - 8, 0), 8)


def reads_per_record(sizes, distinct, ratio, slots):
    round_recs = max(int(slots * FILL * 256) // max(int(ratio * 256), 8), 32)
    reads = 0
    rounds_hist = {}
    for m, d in zip(sizes, distinct):
        if m == 0:
            continue
        e0 = 0
        while (m >> e0) > round_recs and e0 < 8:
            e0 += 1
        r = 1 << e0
        extra = m if d / r > slots * 7 / 8 else 0          # the round overflows: split, its records read once more
        reads += m * r + extra
        key = r + (1 if extra else 0)
        rounds_hist[key] = rounds_hist.get(key, 0) + m
    return reads / sizes.sum(), rounds_hist


def main():
    scale = int(sys.argv[1]) if len(sys.argv) > 1 else 1
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    orc = Oracle()
    sizes = bench.pool_sizes(scale)
    tot = {name: 0.0 for name, _ in TABLES}
    w_all = 0
    print("| pool bin (k-mers) | bins of 512 | b2 | mean leaf | distinct / record | " + " | ".join("%s: reads per record (records by rounds)" % n for n, _ in TABLES) + " |")
    print("|---|---|---|---|---|" + "---|" * len(TABLES))
    for j, n in enumerate(sizes):
        b = bench.gen_bin(4000 + j, bench.K, n)
        recs = orc.expand(b, p)[:, 0]
        del b
        b2 = b2_for(n)
        shift = 62 - 8 - b2
        leaf = (recs >> np.uint64(shift)).astype(np.int64)
        m = np.bincount(leaf, minlength=1 << (8 + b2))
        u = np.unique(recs)
        del recs
        d = np.bincount((u >> np.uint64(shift)).astype(np.int64), minlength=1 << (8 + b2))
        ratio = u.size / n
        del u
        cells = []
        for name, slots in TABLES:
            rpr, hist = reads_per_record(m, d, ratio, slots)
            tot[name] += rpr * n * bench.POOL_COUNT[j]
            cells.append("%.2f (%s)" % (rpr, ", ".join("%d: %.0f %%" % (k, 100.0 * v / n) for k, v in sorted(hist.items()))))
        w_all += n * bench.POOL_COUNT[j]
        print("| %d | %d | %d | %d | %.3f | %s |" % (n, bench.POOL_COUNT[j], b2, n >> (8 + b2), ratio, " | ".join(cells)), flush=True)
    print("| workload (k-mer weighted) | 512 | | | | " + " | ".join("%.2f" % (tot[name] / w_all) for name, _ in TABLES) + " |")


if __name__ == "__main__":
    main()
