"""Reads text -> batch on the GPU (kmc_b200.FastxParser) and count_reads with parse="host" / "gpu".

    python scripts/fastx_bench.py --out DIR [--bases 1e9] [--batch-bytes 268435456] [--reps 20]

Reports, into DIR/fastx_bench.json and one JSON line on stdout:
  * the resident parse of one 256 MiB raw chunk of 150-bp FASTQ and one of FASTA (60-column lines): CUDA events, median of --reps after
    warm-up; raw GB/s, and algorithmic bytes (the raw chunk read once + the batch written once) over the H100 SXM data-sheet HBM bandwidth
    (3.35 TB/s), which bounds it; per-kernel times from torch.profiler in a separate run;
  * the host-to-device copy rate of a pinned 256 MiB buffer (the copy each chunk of the GPU path pays);
  * FASTQ -> .kmc_pre / .kmc_suf with count_reads on split_bench.py's 150-bp and 10-kb read sets (its generators), parse="host" and
    parse="gpu" alternated, twice each, with the md5 of both outputs checked equal; the time reading (host: read(); gpu: waiting for the
    reader thread), the split phase (parse and split, copies included) and stage 2; and where oracle/_ref/kmc_ref exists, the reference
    CLI's wall time on the same file with the host's cores;
  * the card's name and power limit, read in the same run.
All scratch files go to a temporary directory.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from split_bench import HBM_PEAK, K, N_BINS, P, gpu_info, make_map, synth_batch, write_fastq  # noqa: E402


def fasta_of(batch, read_len, line=60):
    """The reads of a batch (read_len + '\\n' each) as FASTA records with 60-column lines."""
    rows = batch.reshape(-1, read_len + 1)[:, :read_len]
    parts = []
    for i in range(rows.shape[0]):
        r = rows[i].tobytes()
        parts.append(b">r%d\n" % i + b"\n".join(r[j:j + line] for j in range(0, read_len, line)) + b"\n")
    return b"".join(parts)


def resident_parse(raw, fmt, reps):
    import torch
    import kmc_b200
    dev = torch.device("cuda:0")
    p = kmc_b200.FastxParser(fmt, max_chunk_bytes=len(raw))
    d_raw = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(dev)
    d_seq = torch.empty(len(raw) + 1, dtype=torch.uint8, device=dev)
    d_res = torch.zeros(4, dtype=torch.int64, device=dev)
    run = lambda: p.dev_parse(d_raw.data_ptr(), len(raw), True, None, d_seq.data_ptr(), d_seq.numel(), d_res.data_ptr(), None)
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    launches = p.kernel_launches()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    launches = (p.kernel_launches() - launches) // reps
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and ("fastx" in ev.name or "split_scan" in ev.name):
            name = ev.name.split("(")[0].replace("void ", "").replace("kmcb::", "")
            kern[name] = kern.get(name, 0.0) + ev.device_time_total / 1e3
    res = d_res.cpu().numpy()
    from kmc_b200.reads import sequences_to_batch
    assert d_seq[:int(res[1])].cpu().numpy().tobytes() == sequences_to_batch(raw).tobytes(), "the GPU parse differs from sequences_to_batch"
    p.close()
    t = float(np.median(times))
    algo = len(raw) + int(res[1])
    return {"raw_bytes": len(raw), "seq_bytes": int(res[1]), "records": int(res[2]), "launches_per_parse": int(launches), "parse_s_median": t,
            "parse_s_all": times, "raw_GB_per_s": len(raw) / t / 1e9, "algorithmic_GB_per_s": algo / t / 1e9,
            "share_of_hbm_peak": algo / t / HBM_PEAK, "bound": "HBM bandwidth (raw read once + batch written once)", "kernel_ms": kern}


def h2d_rate(nbytes, reps=10):
    import torch
    src = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    return nbytes * reps / (time.perf_counter() - t) / 1e9


def md5(path):
    h = hashlib.md5()
    with open(path, "rb") as f:
        for block in iter(lambda: f.read(1 << 24), b""):
            h.update(block)
    return h.hexdigest()


def end_to_end(tmp, sig_map, bases, read_len, batch_bytes, seed):
    from kmc_b200.reads import count_reads
    batch = synth_batch(seed, bases, read_len)
    fq = os.path.join(tmp, "reads_%d.fq" % read_len)
    write_fastq(fq, batch, read_len)
    del batch
    runs = []
    digests = {}
    for rep in range(2):
        for parse in ("host", "gpu"):
            out = os.path.join(tmp, "db_%d_%s" % (read_len, parse))
            t = time.perf_counter()
            r = count_reads([fq], out, K, P, sig_map, 7, 2, 10 ** 9, 255, True, batch_bytes, n_bins=N_BINS, parse=parse)
            r.update({"parse": parse, "rep": rep, "seconds": time.perf_counter() - t})
            r["kmers_per_s"] = r["n_kmers"] / r["seconds"]
            runs.append(r)
            digests.setdefault(parse, set()).add((md5(out + ".kmc_pre"), md5(out + ".kmc_suf")))
    assert len(digests["host"]) == 1 and digests["host"] == digests["gpu"], "host and GPU parsing gave different databases"
    res = {"read_len": read_len, "raw_bytes": os.path.getsize(fq), "runs": runs, "same_md5": True}
    ref = os.path.join(ROOT, "oracle", "_ref", "kmc_ref")
    if os.path.exists(ref):
        wd = os.path.join(tmp, "wd_%d" % read_len)
        os.makedirs(wd, exist_ok=True)
        t = time.perf_counter()
        subprocess.run([ref, "-k%d" % K, "-p%d" % P, "-ci2", "-t%d" % (os.cpu_count() or 1), fq, os.path.join(tmp, "ref_%d" % read_len), wd],
                       check=True, capture_output=True)
        res["reference_cli"] = {"threads": os.cpu_count(), "wall_s": time.perf_counter() - t}
    os.remove(fq)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bases", type=float, default=1e9, help="bases per end-to-end read set")
    ap.add_argument("--batch-bytes", type=int, default=1 << 28)
    ap.add_argument("--chunk-bytes", type=int, default=1 << 28)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    from kmc_b200 import FASTA, FASTQ
    res = {"gpu": gpu_info(), "host_cores": os.cpu_count(), "k": K, "signature_len": P, "n_bins": N_BINS}
    batch = synth_batch(1, a.chunk_bytes // 2, 150)
    fq = os.path.join(tempfile.gettempdir(), "fastx_bench_%d.fq" % os.getpid())
    write_fastq(fq, batch, 150)
    raw = open(fq, "rb").read()[:a.chunk_bytes]
    os.remove(fq)
    raw = raw[:raw.rfind(b"\n@") + 1]
    res["resident_parse_fastq_150bp"] = resident_parse(raw, FASTQ, a.reps)
    fa = fasta_of(synth_batch(2, a.chunk_bytes // 2, 150), 150)
    fa = fa[:fa.rfind(b"\n>", 0, a.chunk_bytes) + 1]
    res["resident_parse_fasta_150bp"] = resident_parse(fa, FASTA, a.reps)
    res["h2d_pinned_GB_per_s"] = h2d_rate(a.chunk_bytes)
    sig_map = make_map(batch)
    del batch, raw, fa
    with tempfile.TemporaryDirectory() as tmp:
        res["end_to_end"] = [end_to_end(tmp, sig_map, int(a.bases), rl, a.batch_bytes, 2 + rl) for rl in (150, 10_000)]
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "fastx_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
