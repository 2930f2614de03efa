"""Measures KMC database input (`kmc -fkmc`) on the GPU and writes DIR/kmc_input_bench.json.

1. The resident decode (KmcDbDecoder's device twin, records and output in HBM) of up to 2^26 records at k = 31, 55 and 128 (at most
   2^31 / (k + 1) records, the decoder's chunk limit): CUDA-event median over the timed calls, and GB/s of input plus output bytes
   against the H100 SXM data sheet's 3.35 TB/s.
2. A database -> database run, kmc_b200.reads.count_reads(parse="gpu"), against `kmc -fkmc -sr1` on the host cores when
   oracle/_ref/kmc_ref exists.

    python scripts/kmc_input_bench.py --out DIR
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

HBM_BYTES_PER_S = 3.35e12


def gpu_name():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def resident_decode(k, reps):
    import torch
    from kmc_b200 import KmcDbDecoder
    lp = {31: 7, 55: 7, 128: 4}[k]
    n = min(1 << 26, (1 << 31) // (k + 1))
    rec = (k - lp) // 4 + 1
    g = torch.Generator(device="cuda").manual_seed(k)
    d_suf = torch.randint(0, 256, (n * rec,), dtype=torch.uint8, device="cuda", generator=g)
    d_suf.view(n, rec)[:, rec - 1] = 2                                  # every counter kept
    lut = np.linspace(0, n, 512 * 4 ** lp + 1).astype(np.uint64)      # records spread over every prefix of 512 bins
    lut[-1] = n
    dec = KmcDbDecoder(k, lp, 1, 2, 255, n, lut, max_records=n)
    d_out = torch.empty(n * (k + 1), dtype=torch.uint8, device="cuda")
    d_res = torch.zeros(2, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        dec.dev_decode(d_suf.data_ptr(), n, 0, d_out.data_ptr(), d_out.numel(), d_res.data_ptr(), st)
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dec.dev_decode(d_suf.data_ptr(), n, 0, d_out.data_ptr(), d_out.numel(), d_res.data_ptr(), st)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    assert int(d_res[1].item()) == n
    dec.close()
    med = float(np.median(ms))
    moved = n * rec + n * (k + 1)
    return {"k": k, "records": n, "record_bytes": rec, "median_ms": med, "bytes_moved": moved, "GB_per_s": moved / med / 1e6,
            "share_of_3.35TB_per_s": moved / (med * 1e-3) / HBM_BYTES_PER_S}


def db_to_db(tmp):
    from kmc_input_testlib import write_reads
    from kmc_b200.reads import count_reads
    ref = os.path.join(ROOT, "oracle", "_ref", "kmc_ref")
    if not os.path.exists(ref):
        return {"skipped": "oracle/_ref/kmc_ref not built"}
    fq = os.path.join(tmp, "reads.fq")
    write_reads(fq, 1, n_reads=400_000, read_len=150, genome_len=5_000_000)
    db = os.path.join(tmp, "in31")
    subprocess.run([ref, "-k31", "-ci1", "-t16", "-m8", fq, db, tmp], check=True, stdout=subprocess.DEVNULL)
    t = time.perf_counter()
    subprocess.run([ref, "-k25", "-fkmc", "-ci1", "-t16", "-m8", "-sr1", db, os.path.join(tmp, "ref25"), tmp], check=True, stdout=subprocess.DEVNULL)
    ref_s = time.perf_counter() - t
    count_reads([db], os.path.join(tmp, "warm"), 25, 9, None, cutoff_min=1, parse="gpu", small_k=False)
    t = time.perf_counter()
    res = count_reads([db], os.path.join(tmp, "gpu25"), 25, 9, None, cutoff_min=1, parse="gpu", small_k=False)
    gpu_s = time.perf_counter() - t
    same = all(open(os.path.join(tmp, "gpu25" + e), "rb").read() == open(os.path.join(tmp, "ref25" + e), "rb").read() for e in (".kmc_pre", ".kmc_suf"))
    return {"input_records": res["n_reads"], "kmc_ref_s": ref_s, "kmc_ref_threads": 16, "count_reads_gpu_s": gpu_s, "files_identical": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_name(), "decode": [resident_decode(k, a.reps) for k in (31, 55, 128)]}
    with tempfile.TemporaryDirectory() as tmp:
        res["db_to_db"] = db_to_db(tmp)
    print(json.dumps(res, indent=1))
    with open(os.path.join(a.out, "kmc_input_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
