"""gzip input (inflate.cuh, kmc_b200.reads' gzip reader): BGZF members inflated on a resident buffer, and reads -> database from BGZF, plain
text and single-member gzip.

    python scripts/gzip_bench.py --out DIR [--bases 1e9] [--reps 20]

Reports, into DIR/gzip_bench.json and one JSON line on stdout:
  * resident inflate: BGZF of 150-bp FASTQ (binned Illumina-like qualities) at zlib levels 1, 6 and 9, calls of 2^24 .. 2^28 text bytes
    (the first members that fit): the median of `reps` CUDA-event timings of kmcb200_dev_gunzip_inflate, GB/s of text; every call's
    text is checked against zlib's.  For level 6 at 2^28, gunzip_kernel's own time from torch.profiler in a separate pass, and the bytes it
    moves (compressed data read, text written, text read again for the CRC) over that time, as a share of 3.35 TB/s;
  * end to end: `bases` of the same FASTQ -> database (k = 31, the map chosen from the reads, parse="gpu"), as BGZF, as plain text and as
    single-member gzip (zlib on the reader thread), alternated, two runs each; `kmc -k31 -sr1` on the two gzip files where
    oracle/_ref/kmc_ref is present, with the host's core count; the time of copying the text back from the GPU and to it again, from
    CUDA-event timings of pinned copies of one piece, scaled to the text size;
  * the card's name and power limit, read in the same run.
Scratch files go to a temporary directory.
"""
import argparse
import hashlib
import json
import multiprocessing
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from split_bench import gpu_info, synth_batch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12                                              # H100 SXM data sheet
READ_LEN = 150
QUALS = np.frombuffer(b"FFFFFFF:::,#", dtype=np.uint8)                  # binned qualities, F most often


def fastq_text(seed, n_bases):
    """150-bp reads of a random genome as FASTQ ("@r<i>" headers, binned qualities): bytes."""
    rows = synth_batch(seed, n_bases, READ_LEN).reshape(-1, READ_LEN + 1)
    rng = np.random.default_rng(seed + 1)
    out = []
    for c0 in range(0, rows.shape[0], 1 << 16):
        r = rows[c0:c0 + (1 << 16)]
        q = QUALS[rng.integers(0, QUALS.size, r.shape)]
        q[:, -1] = 10
        head = np.frombuffer(b"".join(b"@r%09d\n" % (c0 + i) for i in range(r.shape[0])), dtype=np.uint8).reshape(r.shape[0], -1)
        plus = np.tile(np.frombuffer(b"+\n", dtype=np.uint8), (r.shape[0], 1))
        out.append(np.hstack([head, r, plus, q]).tobytes())
    return b"".join(out)


def _member(args):
    from gzip_testlib import bgzf_member
    text, level = args
    return bgzf_member(text, level=level)


def bgzf_parallel(text, level, pool):
    from gzip_testlib import BGZF_EOF, BGZF_PIECE
    pieces = [(text[i:i + BGZF_PIECE], level) for i in range(0, len(text), BGZF_PIECE)]
    return b"".join(pool.map(_member, pieces, chunksize=64)) + BGZF_EOF


def cuda_time(fn, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    return float(np.median(times))


def resident(text, raw, level, sizes, reps, g, res, profile_dir=None):
    import torch
    import kmc_b200
    from gzip_testlib import inflate_all
    d_raw = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
    d_err = torch.zeros(1, dtype=torch.int64, device="cuda")
    for size in sizes:
        used, tbytes, m = kmc_b200.bgzf_scan(raw, size)
        d_m = torch.from_numpy(m.view(np.uint8).copy()).cuda()
        d_text = torch.empty(tbytes, dtype=torch.uint8, device="cuda")
        st = torch.cuda.current_stream().cuda_stream

        def call():
            g.dev_inflate(d_m.data_ptr(), len(m), d_raw.data_ptr(), used, d_text.data_ptr(), tbytes, d_err.data_ptr(), st)

        for _ in range(3):
            call()
        t = cuda_time(call, reps)
        ok = int(d_err.item()) == -1 and d_text.cpu().numpy().tobytes() == inflate_all(raw[:used]) == text[:tbytes]
        if not ok:
            raise SystemExit("level %d, %d bytes: the GPU text differs from zlib's" % (level, size))
        row = {"level": level, "call_text_bytes": tbytes, "members": len(m), "compressed_bytes": used, "median_s": t,
               "text_GB_per_s": tbytes / t / 1e9, "checked_vs_zlib": True}
        res["resident"].append(row)
        print(json.dumps(row), flush=True)
        if profile_dir and size == sizes[-1]:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    call()
                torch.cuda.synchronize()
            ks = [e for e in prof.key_averages() if "gunzip_kernel" in e.key]
            k_s = ks[0].device_time / 1e6 if hasattr(ks[0], "device_time") else ks[0].cuda_time / 1e6
            moved = used + 2 * tbytes
            res["kernel_profile"] = {"level": level, "text_bytes": tbytes, "gunzip_kernel_s": k_s, "bytes_moved": moved,
                                     "hbm_share": moved / k_s / HBM_BYTES_PER_S}
            print(json.dumps(res["kernel_profile"]), flush=True)
        del d_m, d_text


def end_to_end(tmp, text, raw_bgzf, res):
    import torch
    from gzip_testlib import gzip_single, write
    from kmc_b200.reads import count_reads
    paths = {"bgzf": write(os.path.join(tmp, "r.bgzf.fq.gz"), raw_bgzf), "plain": write(os.path.join(tmp, "r.fq"), text)}
    t = time.perf_counter()
    paths["gzip"] = write(os.path.join(tmp, "r.gzip.fq.gz"), gzip_single(text, 6))
    res["gzip_write_s"] = time.perf_counter() - t
    res["files"] = {k: os.path.getsize(v) for k, v in paths.items()}
    digests = {}
    for rep in range(2):
        for name in ("bgzf", "plain", "gzip"):
            out = os.path.join(tmp, "db_" + name)
            torch.cuda.synchronize()
            t = time.perf_counter()
            r = count_reads([paths[name]], out, 31, 9, None, parse="gpu")
            dt = time.perf_counter() - t
            d = tuple(hashlib.md5(open(out + ext, "rb").read()).hexdigest() for ext in (".kmc_pre", ".kmc_suf"))
            digests.setdefault(name, d)
            row = {"input": name, "run": rep, "s": dt, "bases_per_s": r["n_bases"] / dt, "read_wait_s": r["read_s"], "n_unique": r["n_unique"]}
            res["end_to_end"].append(row)
            print(json.dumps(row), flush=True)
    res["databases_identical"] = digests["bgzf"] == digests["plain"] == digests["gzip"]
    kmc = os.path.join(ROOT, "oracle", "_ref", "kmc_ref")
    if os.path.exists(kmc):
        res["host_cores"] = os.cpu_count()
        for name in ("bgzf", "gzip"):
            wd = os.path.join(tmp, "wd_" + name)
            os.makedirs(wd, exist_ok=True)
            t = time.perf_counter()
            subprocess.run([kmc, "-k31", "-sr1", "-t%d" % os.cpu_count(), paths[name], os.path.join(tmp, "kmc_" + name), wd], check=True,
                           stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            row = {"input": name, "kmc_s": time.perf_counter() - t, "threads": os.cpu_count()}
            res["kmc"].append(row)
            print(json.dumps(row), flush=True)
    # the text's round trip: back from the GPU after the inflate, and to it again for the parser
    piece = 1 << 25
    h = torch.empty(piece, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(piece, dtype=torch.uint8, device="cuda")
    d2h = cuda_time(lambda: h.copy_(d, non_blocking=True), 10)
    h2d = cuda_time(lambda: d.copy_(h, non_blocking=True), 10)
    res["text_round_trip"] = {"text_bytes": len(text), "d2h_s": d2h * len(text) / piece, "h2d_s": h2d * len(text) / piece,
                              "d2h_GB_per_s": piece / d2h / 1e9, "h2d_GB_per_s": piece / h2d / 1e9}
    print(json.dumps(res["text_round_trip"]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bases", type=float, default=1e9)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--max-log2", type=int, default=28)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    import torch
    import kmc_b200
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this benchmark measures the H100")
    res = {"gpu": gpu_info(), "resident": [], "end_to_end": [], "kmc": []}
    sizes = [1 << s for s in range(24, a.max_log2 + 1)]
    t = time.perf_counter()
    text = fastq_text(7, int(max(a.bases, sizes[-1] / 2.1 * 1.1)))
    res["text_bytes"] = len(text)
    with multiprocessing.Pool() as pool:
        raws = {lv: bgzf_parallel(text[:sizes[-1] + (1 << 17)] if lv != 6 else text, lv, pool) for lv in (1, 6, 9)}
    res["prepare_s"] = time.perf_counter() - t
    g = kmc_b200.Gunzip(0, max_in_bytes=1 << 20, max_out_bytes=1 << 20)    # dev_inflate: the buffers are the caller's
    try:
        for lv in (1, 6, 9):
            resident(text, raws[lv], lv, sizes, a.reps, g, res, a.out if lv == 6 else None)
            res.setdefault("ratio", {})[lv] = len(text if lv == 6 else text[:sizes[-1] + (1 << 17)]) / len(raws[lv])
    finally:
        g.close()
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as tmp:
        end_to_end(tmp, text, raws[6], res)
    with open(os.path.join(a.out, "gzip_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k not in ("resident", "end_to_end")}))


if __name__ == "__main__":
    main()
