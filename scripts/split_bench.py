"""Stage 1 on the GPU (kmcb200_dev_split / count_reads): split throughput, per-kernel times and reads -> database rates.

    python scripts/split_bench.py --out DIR [--bases 1e9] [--batch-bytes 268435456]

Reports, into DIR/split_bench.json and one JSON line on stdout:
  * the split of one resident batch (150-bp reads, k = 31, p = 9, 512 bins): bases/s and GB/s of algorithmic bytes (the batch read once +
    the bins written once) as a share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s).  The split is not a pure stream (a signature
    tile is re-read by the record passes, records are gathered and scattered), so this share is a lower bound of the traffic it moves;
  * kernel times of one split from torch.profiler (CUDA activity), by kernel name;
  * FASTQ -> .kmc_pre / .kmc_suf with kmc_b200.reads.count_reads (k-mers/s end to end, file reading and parsing included) for 150-bp and
    10-kb reads, and where oracle/_ref/kmc_ref exists, the reference CLI's 1st_stage time (-j) on the same FASTQ with the host's cores;
  * the card's name and power limit, read in the same run.
The signature map: per-signature k-mer counts of a 1 % sample (the stage-1 oracle with the identity map, what CSplitter::CalcStats counts),
grouped greedily onto 511 bins, the special signature in bin 511.  All scratch files go to a temporary directory.
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

HBM_PEAK = 3.35e12
K, P, N_BINS = 31, 9, 512


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def synth_batch(seed, n_bases, read_len, genome_len=50_000_000):
    """Reads of read_len sampled from a random genome, both strands, 1 % substitutions, '\\n' after each: one batch (uint8)."""
    rng = np.random.default_rng(seed)
    genome = rng.integers(0, 4, genome_len, dtype=np.uint8)
    n_reads = max(1, n_bases // read_len)
    out = np.empty(n_reads * (read_len + 1), dtype=np.uint8)
    letters = np.frombuffer(b"ACGT", dtype=np.uint8)
    chunk = max(1, (1 << 24) // read_len)
    for c0 in range(0, n_reads, chunk):
        c1 = min(n_reads, c0 + chunk)
        pos = rng.integers(0, genome_len - read_len, c1 - c0)
        idx = pos[:, None] + np.arange(read_len)[None, :]
        r = genome[idx]
        rc = rng.random(c1 - c0) < 0.5
        r[rc] = 3 - r[rc][:, ::-1]
        err = rng.random(r.shape) < 0.01
        r = np.where(err, (r + rng.integers(1, 4, r.shape)) % 4, r).astype(np.uint8)
        rows = out[c0 * (read_len + 1):c1 * (read_len + 1)].reshape(c1 - c0, read_len + 1)
        rows[:, :read_len] = letters[r]
        rows[:, read_len] = 10
    return out


def write_fastq(path, batch, read_len):
    rows = batch.reshape(-1, read_len + 1)
    n = rows.shape[0]
    with open(path, "wb") as f:
        chunk = max(1, (1 << 24) // read_len)
        qual = np.full(read_len + 1, ord("I"), dtype=np.uint8)
        qual[-1] = 10
        for c0 in range(0, n, chunk):
            c1 = min(n, c0 + chunk)
            rec = np.empty((c1 - c0, 4 + 2 * (read_len + 1)), dtype=np.uint8)
            rec[:, 0:2] = np.frombuffer(b"@\n", dtype=np.uint8)
            rec[:, 2:2 + read_len + 1] = rows[c0:c1]
            rec[:, 3 + read_len:5 + read_len] = np.frombuffer(b"+\n", dtype=np.uint8)
            rec[:, 5 + read_len:] = qual
            f.write(rec.tobytes())


def make_map(batch):
    from stage1_testlib import Stage1Oracle, greedy_map
    sample = batch[:max(1, batch.size // 100)]
    counts = Stage1Oracle().signature_counts(sample, K, P)
    return greedy_map(counts, N_BINS)


def resident_split(sig_map, batch, reps):
    import torch
    import kmc_b200
    dev = torch.device("cuda:0")
    sp = kmc_b200.Splitter(K, P, sig_map, N_BINS, max_batch_bytes=batch.size)
    d_seq = torch.from_numpy(batch).to(dev)
    d_res = torch.zeros(8, dtype=torch.int64, device=dev)
    d_frags = torch.zeros(N_BINS * 5, dtype=torch.int64, device=dev)
    # sizing run: no output capacity
    sp.dev_split(d_seq.data_ptr(), batch.size, 0, 0, 0, 0, d_frags.data_ptr(), d_res.data_ptr(), None)
    torch.cuda.synchronize()
    need_bytes, need_packs = int(d_res[0]), int(d_res[1])
    d_out = torch.empty(need_bytes + 64, dtype=torch.uint8, device=dev)
    d_packs = torch.empty(need_packs + 8, dtype=torch.int64, device=dev)
    run = lambda: sp.dev_split(d_seq.data_ptr(), batch.size, d_out.data_ptr(), d_out.numel(), d_packs.data_ptr(), d_packs.numel(), d_frags.data_ptr(),
                               d_res.data_ptr(), None)
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    assert int(d_res[2]) == 0
    launches = sp.kernel_launches()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    launches = (sp.kernel_launches() - launches) // reps
    # per-kernel times, in a separate profiled run
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and "split" in ev.name:
            name = ev.name.split("(")[0].replace("void ", "").replace("kmcb::", "")
            kern[name] = kern.get(name, 0.0) + ev.device_time_total / 1e3
    res = d_res.cpu().numpy()
    sp.close()
    t = float(np.median(times))
    algo = batch.size + need_bytes
    return {"bases": int(batch.size), "out_bytes": need_bytes, "packs": need_packs, "super_kmers": int(res[3]), "kmers": int(res[4]),
            "launches_per_split": int(launches), "split_s_median": t, "split_s_all": times, "bases_per_s": batch.size / t,
            "algorithmic_GB_per_s": algo / t / 1e9, "share_of_hbm_peak": algo / t / HBM_PEAK, "kernel_ms": kern}


def end_to_end(tmp, sig_map, bases, read_len, batch_bytes, seed):
    from kmc_b200.reads import count_reads
    batch = synth_batch(seed, bases, read_len)
    fq = os.path.join(tmp, "reads_%d.fq" % read_len)
    write_fastq(fq, batch, read_len)
    del batch
    t = time.perf_counter()
    with open(fq, "rb") as f:
        from kmc_b200.reads import sequences_to_batch
        parsed = sequences_to_batch(f.read()).size
    r_parse = time.perf_counter() - t
    t = time.perf_counter()
    r = count_reads([fq], os.path.join(tmp, "db_%d" % read_len), K, P, sig_map, 7, 2, 10 ** 9, 255, True, batch_bytes, n_bins=N_BINS)
    total = time.perf_counter() - t
    r.update({"read_len": read_len, "seconds": total, "kmers_per_s": r["n_kmers"] / total, "read_and_parse_s": r_parse, "parsed_bytes": parsed})
    ref = os.path.join(ROOT, "oracle", "_ref", "kmc_ref")
    if os.path.exists(ref):
        wd = os.path.join(tmp, "wd_%d" % read_len)
        os.makedirs(wd, exist_ok=True)
        js = os.path.join(tmp, "ref_%d.json" % read_len)
        t = time.perf_counter()
        subprocess.run([ref, "-k%d" % K, "-p%d" % P, "-ci2", "-t%d" % (os.cpu_count() or 1), "-j" + js, fq, os.path.join(tmp, "ref_%d" % read_len), wd],
                       check=True, capture_output=True)
        wall = time.perf_counter() - t
        st = json.load(open(js))
        r["reference_cli"] = {"threads": os.cpu_count(), "wall_s": wall, "first_stage_s": float(str(st["1st_stage"]).rstrip("s")),
                              "second_stage_s": float(str(st["2nd_stage"]).rstrip("s")),
                              "total_kmers": st.get("Stats", {}).get("#Total no. of k-mers")}
    os.remove(fq)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bases", type=float, default=1e9, help="bases per end-to-end read set")
    ap.add_argument("--batch-bytes", type=int, default=1 << 28)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info(), "host_cores": os.cpu_count(), "k": K, "signature_len": P, "n_bins": N_BINS}
    batch = synth_batch(1, a.batch_bytes - 1024, 150)
    sig_map = make_map(batch)
    res["resident_split_150bp"] = resident_split(sig_map, batch, a.reps)
    del batch
    with tempfile.TemporaryDirectory() as tmp:
        res["end_to_end"] = [end_to_end(tmp, sig_map, int(a.bases), rl, a.batch_bytes, 2 + rl) for rl in (150, 10_000)]
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "split_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
