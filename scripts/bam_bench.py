"""BAM input (bam.cuh, kmc_b200.reads' BAM reader): decompressed BAM records walked and decoded on a resident buffer, and BAM -> database.

    python scripts/bam_bench.py --out DIR [--bases 1e9] [--reps 20]

Reports, into DIR/bam_bench.json and one JSON line on stdout:
  * resident parse: a chunk of 2^28 bytes (the whole records that fit) of short-read records (150 bp, one CIGAR op, qualities and three
    tags, as an aligned BAM has), of 15 kb HiFi-like records and of 100 kb records, each with KMCB200_BAM and KMCB200_BAM_ORIGINAL_STRAND;
    of adversarial 3 kb records whose qualities and tags are tiled with well-formed little records, so that nearly every tile guess
    is wrong and the resolve walks the tiles again; and of 36-byte records without a name, the worst case: no tile has a guess and one
    warp walks every record (3 timings).  The median of `reps` CUDA-event timings of kmcb200_dev_fastx_parse, GB/s of record
    bytes; every output is checked against the host model on the first call.  The parser sees decompressed bytes only, so the member
    layout does not enter these numbers;
  * end to end: `bases` of 150-bp records -> database (k = 31, the map chosen from the reads, parse="gpu"), the same records in two member
    layouts: members ending on records (htslib) and fixed 65,280-byte members (htsjdk-like, records straddle members).  The input is a
    block of 2^24 bases repeated, its members compressed once (zlib level 1).  `kmc -k31 -fbam -sr1` on the same files where
    oracle/_ref/kmc_ref is present, with the host's core count;
  * the card's name and power limit, read in the same run.
Scratch files go to a temporary directory.
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from split_bench import gpu_info, synth_batch  # noqa: E402

CHUNK = 1 << 28
_CODE = np.zeros(256, dtype=np.uint8)
_CODE[np.frombuffer(b"ACGT", dtype=np.uint8)] = [1, 2, 4, 8]


def records(seed, n_bases, read_len):
    """Records of read_len bases (reads of a random genome, half of them stored reverse complemented as FLAG 0x10, 2 % secondary), each
    with a 10-byte name, one CIGAR op, qualities and the tags NM:C, AS:C, XS:C: bytes, and the record starts."""
    rows = synth_batch(seed, n_bases, read_len).reshape(-1, read_len + 1)[:, :read_len]
    n = rows.shape[0]
    rng = np.random.default_rng(seed)
    tags = b"NMC\x01ASC\x96XSC\x10"
    seq_b = (read_len + 1) // 2
    size = 36 + 10 + 4 + seq_b + read_len + len(tags)
    out = np.zeros((n, size), dtype=np.uint8)
    flags = np.where(rng.random(n) < 0.5, 0x10, 0) | np.where(rng.random(n) < 0.02, 0x100, 0)
    fixed = np.zeros(n, dtype=[("bs", "<i4"), ("ref", "<i4"), ("pos", "<i4"), ("l_name", "u1"), ("mapq", "u1"), ("bin", "<u2"),
                               ("n_cigar", "<u2"), ("flag", "<u2"), ("l_seq", "<i4"), ("nref", "<i4"), ("npos", "<i4"), ("tlen", "<i4")])
    fixed["bs"], fixed["l_name"], fixed["mapq"], fixed["n_cigar"], fixed["flag"], fixed["l_seq"] = size - 4, 10, 60, 1, flags, read_len
    fixed["pos"] = rng.integers(0, 1 << 30, n)
    fixed["nref"], fixed["npos"] = -1, -1
    out[:, :36] = fixed.view(np.uint8).reshape(n, 36)
    out[:, 36:45] = np.frombuffer(b"%09d" % 0, dtype=np.uint8)          # the name's digits only matter as bytes
    out[:, 45] = 0
    out[:, 46:50] = np.frombuffer(struct.pack("<I", read_len << 4), dtype=np.uint8)
    codes = _CODE[rows]
    if read_len % 2:
        codes = np.hstack([codes, np.zeros((n, 1), dtype=np.uint8)])
    out[:, 50:50 + seq_b] = (codes[:, 0::2] << 4) | codes[:, 1::2]
    out[:, 50 + seq_b:50 + seq_b + read_len] = rng.integers(2, 41, (n, read_len), dtype=np.uint8)
    out[:, 50 + seq_b + read_len:] = np.frombuffer(tags, dtype=np.uint8)
    return out.tobytes(), np.arange(n, dtype=np.int64) * size


def adversarial(seed):
    from bam_testlib import adversarial_records
    block = b"".join(adversarial_records(seed, 200))
    return block * (CHUNK // len(block))


def no_guess():
    """The worst case of the walk: 36-byte records (no SEQ) without a name, so no position of any tile is a guess and the resolve walks
    every record of the chunk serially."""
    n = CHUNK // 36
    rec = np.zeros((n, 9), dtype="<i4")
    rec[:, 0] = 32
    return rec.tobytes()


def time_parse(data, fmt, reps):
    import torch
    import kmc_b200
    from kmc_b200.reads import bam_records_to_batch
    dev = torch.device("cuda:0")
    p = kmc_b200.FastxParser(fmt, max_chunk_bytes=len(data))
    d_raw = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(dev)
    d_seq = torch.empty(len(data) + 1, dtype=torch.uint8, device=dev)
    d_res = torch.zeros(4, dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    p.dev_parse(d_raw.data_ptr(), len(data), True, None, d_seq.data_ptr(), d_seq.numel(), d_res.data_ptr(), st)
    torch.cuda.synchronize()
    want = bam_records_to_batch(data, fmt == kmc_b200.BAM_ORIGINAL_STRAND)
    res = [int(x) for x in d_res.cpu()]
    ok = res[0] == len(data) and res[3] == 0 and res[1] == want.size and d_seq[:res[1]].cpu().numpy().tobytes() == want.tobytes()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        p.dev_parse(d_raw.data_ptr(), len(data), True, None, d_seq.data_ptr(), d_seq.numel(), d_res.data_ptr(), st)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    p.close()
    ms = float(np.median(times))
    return {"bytes": len(data), "records": res[2], "out_bytes": res[1], "ms": ms, "gb_s": len(data) / ms / 1e6, "equals_model": bool(ok)}


def write_bam(path, block, starts, n_rep, layout):
    from bam_testlib import bgzf_text, header
    from gzip_testlib import BGZF_EOF, bgzf_member
    members = bgzf_text(block, layout, [int(s) for s in starts[1:]])[:-len(BGZF_EOF)]
    with open(path, "wb") as f:
        f.write(bgzf_member(header(b"@HD\tVN:1.6\tSO:unsorted\n", [(b"chr1", 1 << 30)]), level=1))
        for _ in range(n_rep):
            f.write(members)
        f.write(BGZF_EOF)
    return os.path.getsize(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bases", type=float, default=1e9)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import kmc_b200
    from kmc_b200 import reads
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info(), "parse": [], "end_to_end": []}
    for name, read_len in (("short_150bp", 150), ("hifi_15kb", 15000), ("long_100kb", 100_000)):
        rec_size = 36 + 10 + 4 + (read_len + 1) // 2 + read_len + 12
        data, _ = records(31, (CHUNK // rec_size) * read_len, read_len)
        for fmt, fname in ((kmc_b200.BAM, "BAM"), (kmc_b200.BAM_ORIGINAL_STRAND, "BAM_ORIGINAL_STRAND")):
            row = {"records": name, "format": fname}
            row.update(time_parse(data, fmt, a.reps))
            res["parse"].append(row)
            print(json.dumps(row), flush=True)
    for name, data, reps in (("adversarial_3kb", adversarial(5), a.reps), ("no_guess_36B", no_guess(), 3)):
        row = {"records": name, "format": "BAM"}
        row.update(time_parse(data, kmc_b200.BAM, reps))
        res["parse"].append(row)
        print(json.dumps(row), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        block, starts = records(41, 1 << 24, 150)
        n_rep = max(1, int(a.bases) // (1 << 24))
        paths = {layout: os.path.join(tmp, "reads_%s.bam" % layout) for layout in ("aligned", "fixed")}
        sizes = {layout: write_bam(p, block, starts, n_rep, layout) for layout, p in paths.items()}
        kmc = os.path.join(ROOT, "oracle", "_ref", "kmc_ref")
        for layout in ("aligned", "fixed", "aligned", "fixed"):
            t = time.perf_counter()
            r = reads.count_reads([paths[layout]], os.path.join(tmp, "db_" + layout), 31, 9, None, parse="gpu")
            row = {"layout": layout, "bam_bytes": sizes[layout], "bases": n_rep * (1 << 24), "s": time.perf_counter() - t,
                   "n_unique": r["n_unique"], "n_total": r["n_total"], "read_s": r["read_s"]}
            res["end_to_end"].append(row)
            print(json.dumps(row), flush=True)
        if os.path.exists(kmc):
            for layout in ("aligned", "fixed"):
                wd = os.path.join(tmp, "wd_" + layout)
                os.makedirs(wd, exist_ok=True)
                t = time.perf_counter()
                subprocess.run([kmc, "-k31", "-fbam", "-sr1", "-t%d" % os.cpu_count(), paths[layout], os.path.join(tmp, "kmc_" + layout), wd],
                               check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
                row = {"layout": layout, "kmc_s": time.perf_counter() - t, "threads": os.cpu_count()}
                res["end_to_end"].append(row)
                print(json.dumps(row), flush=True)
    with open(os.path.join(a.out, "bam_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
