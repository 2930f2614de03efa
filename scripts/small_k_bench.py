"""Small k on the GPU (kmcb200_smallk_*): count times per k, finish + emit, and FASTQ -> KMC1 database.

    python scripts/small_k_bench.py --out DIR [--bases 1e9] [--reps 20]

Reports, into DIR/small_k_bench.json and one JSON line on stdout:
  * the count of one resident batch (split_bench.py's 150-bp reads, 2^28 - 1024 bytes, about 2.7e8 bases) for k in {5, 7, 9, 11, 12, 13}:
    median of `reps` CUDA-event timings of kmcb200_dev_smallk_add (k <= 7 takes the shared-memory kernel, k >= 8 the global one, so both
    sides of that choice are measured), with the sector traffic of the k >= 8 kernel's atomics (one 32-byte sector read and written per
    add, an upper bound: runs of equal values add once) for k = 12 and 13, whose counters do not fit in L2;
  * finish + emit at k = 13 (host clock around calls that end in a synchronisation, median of 5);
  * `bases` of 150-bp FASTQ -> database with count_reads_small_k(parse="gpu") at k = 13, and kmc_ref -k13 on the host's cores where
    oracle/_ref/kmc_ref exists;
  * the card's name and power limit, read in the same run.
The resident counts and finish + emit are checked against the numpy model (tests/test_small_k_model.py), the end-to-end database against
kmc_ref's files where kmc_ref exists.  Scratch files go to a temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from split_bench import gpu_info, synth_batch, write_fastq  # noqa: E402

HBM_PEAK = 3.35e12
KS = (5, 7, 9, 11, 12, 13)


def resident_counts(batch, reps):
    import torch
    import kmc_b200
    import test_small_k_model as M
    d_seq = torch.from_numpy(batch).cuda()
    out = {}
    for k in KS:
        sk = kmc_b200.SmallKCounter(k, max_batch_bytes=batch.size)
        run = lambda: sk.dev_add(d_seq.data_ptr(), batch.size, None)
        run()
        torch.cuda.synchronize()
        assert np.array_equal(sk.read(), M.counts(batch, k)), "k=%d: GPU counts differ from the model" % k
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(reps):
            sk.reset()
            torch.cuda.synchronize()
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        t = float(np.median(times))
        r = {"kernel": "shared" if k <= 7 else "global", "count_s_median": t, "count_s_all": times, "bases_per_s": batch.size / t}
        if k >= 12:
            kmers = int(M.kmer_values(batch, k).size)
            r["sector_bytes_upper_bound"] = kmers * 64
            r["sector_GB_per_s"] = kmers * 64 / t / 1e9
            r["share_of_hbm_peak"] = kmers * 64 / t / HBM_PEAK
        out[k] = r
        if k == 13:
            fin = []
            for _ in range(5):
                t0 = time.perf_counter()
                lp, cs, nbytes, stats = sk.finish(2, 10 ** 9, 255)
                recs, lut = sk.emit()
                fin.append(time.perf_counter() - t0)
            e_lp, e_cs, e_recs, e_lut, e_stats = M.finish(sk.read(), 13, 2, 10 ** 9, 255)
            assert (lp, stats) == (e_lp, e_stats) and np.array_equal(recs, e_recs) and np.array_equal(lut, e_lut), "finish / emit differ from the model"
            out["finish_emit_k13"] = {"seconds_median": float(np.median(fin)), "seconds_all": fin, "records": int(stats[0] - stats[1] - stats[2]),
                                      "suffix_bytes": nbytes, "lut_prefix_len": lp}
        sk.close()
    return out


def end_to_end(tmp, bases, batch_bytes):
    from kmc_b200.reads import count_reads_small_k
    batch = synth_batch(3, bases, 150)
    fq = os.path.join(tmp, "reads.fq")
    write_fastq(fq, batch, 150)
    del batch
    db = os.path.join(tmp, "gpu")
    t = time.perf_counter()
    r = count_reads_small_k([fq], db, 13, batch_bytes=batch_bytes, parse="gpu")
    r["seconds"] = time.perf_counter() - t
    r["kmers_per_s"] = r["n_total"] / r["seconds"]
    ref = os.path.join(ROOT, "oracle", "_ref", "kmc_ref")
    if os.path.exists(ref):
        wd = os.path.join(tmp, "wd")
        os.makedirs(wd, exist_ok=True)
        js = os.path.join(tmp, "ref.json")
        t = time.perf_counter()
        subprocess.run([ref, "-k13", "-ci2", "-m8", "-t%d" % (os.cpu_count() or 1), "-j" + js, fq, os.path.join(tmp, "ref"), wd], check=True,
                       capture_output=True)
        wall = time.perf_counter() - t
        st = json.load(open(js))
        same = all(open(db + e, "rb").read() == open(os.path.join(tmp, "ref") + e, "rb").read() for e in (".kmc_pre", ".kmc_suf"))
        r["reference_cli"] = {"threads": os.cpu_count(), "wall_s": wall, "total_kmers": st.get("Stats", {}).get("#Total no. of k-mers"),
                              "files_identical": same}
        assert same, "the GPU database differs from kmc_ref's"
    os.remove(fq)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bases", type=float, default=1e9, help="bases of the end-to-end FASTQ")
    ap.add_argument("--batch-bytes", type=int, default=1 << 28)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info(), "host_cores": os.cpu_count()}
    batch = synth_batch(1, a.batch_bytes - 1024, 150)
    res["bases"] = int(batch.size)
    res["resident_count"] = resident_counts(batch, a.reps)
    del batch
    with tempfile.TemporaryDirectory() as tmp:
        res["end_to_end_k13"] = end_to_end(tmp, int(a.bases), a.batch_bytes)
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "small_k_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
