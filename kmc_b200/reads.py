"""Reads -> KMC database with this library alone: FASTQ / FASTA -> batches -> GPU stage 1 (Splitter) -> GPU stage 2 (Stage2Context) ->
.kmc_pre / .kmc_suf (DbWriter).  For the same signature map and parameters the files are byte-identical to the reference CLI's
(`kmc -sr1`): the bins hold the same k-mers, and stage 2 and the writer reproduce the reference's output per bin.

    python -m kmc_b200.reads -k31 -p9 --map-from ref_db.kmc_pre reads.fq out_prefix

The caller chooses the signature map (4^p + 1 entries); `signature_map_from_kmc_pre` reads the one a KMC database was built with.
"""
import argparse
import json
import struct
import sys
import time

import numpy as np

from . import DbWriter, KmcB200Error, ERR_INVALID, Splitter, Stage2Context, Stage2Params

_NL, _GT, _AT = 10, ord(">"), ord("@")


def sequences_to_batch(data):
    """FASTQ or FASTA (multi-line records are joined) -> one uint8 array of the sequences, one newline after each.  Every byte other than
    ACGTacgt separates k-mers on the GPU, so only the record boundaries matter; '\\r' and IUPAC codes act like N."""
    a = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.asarray(data, dtype=np.uint8)
    if a.size == 0:
        return np.zeros(0, dtype=np.uint8)
    if a[-1] != _NL:
        a = np.append(a, np.uint8(_NL))
    ends = np.flatnonzero(a == _NL)                                     # line ends
    starts = np.concatenate([[0], ends[:-1] + 1])
    first = a[starts[np.flatnonzero(starts < ends)[0]]]
    delta = np.zeros(a.size + 1, dtype=np.int8)                        # +1 where a kept span starts, -1 past its end
    if first == _AT:                                                    # FASTQ: line 1 of every 4, with its newline
        seq = np.arange(1, ends.size, 4)
        delta[starts[seq]] += 1
        delta[ends[seq] + 1] -= 1
        keep = np.cumsum(delta[:-1], dtype=np.int8).view(bool)
    elif first == _GT:                                                  # FASTA: sequence bytes without their newlines, a newline per header
        hdr = np.flatnonzero(a[starts] == _GT)
        delta[starts[hdr]] += 1
        delta[ends[hdr]] -= 1
        keep = np.cumsum(delta[:-1], dtype=np.int8) == 0               # outside the header text ...
        keep[ends] = False                                              # ... no line breaks ...
        keep[ends[hdr]] = True                                          # ... but one at the end of every header
    else:
        raise KmcB200Error(ERR_INVALID, "input is neither FASTQ ('@') nor FASTA ('>')")
    return a[keep]


def batches(seq, batch_bytes):
    """Cuts a batch between records into pieces of at most batch_bytes (a record longer than that is an error)."""
    seps = np.flatnonzero(seq == _NL)
    pos = 0
    while pos < seq.size:
        end = pos + batch_bytes
        if end >= seq.size:
            yield seq[pos:]
            return
        i = int(np.searchsorted(seps, end, side="right")) - 1
        if i < 0 or seps[i] < pos:
            raise KmcB200Error(ERR_INVALID, "a sequence is longer than batch_bytes = %d" % batch_bytes)
        yield seq[pos:int(seps[i]) + 1]
        pos = int(seps[i]) + 1


def signature_map_from_kmc_pre(path):
    """(signature_len, map) stored in a KMC database's .kmc_pre (kb_completer.cpp:211-221, 290): the file position of every signature's bin."""
    pre = open(path, "rb").read()
    header_offset = struct.unpack("<I", pre[-8:-4])[0]
    h = len(pre) - 8 - header_offset
    sig_len = struct.unpack("<I", pre[h + 16:h + 20])[0]
    n = (1 << (2 * sig_len)) + 1
    return sig_len, np.frombuffer(pre[h - 4 * n:h], dtype=np.uint32).copy()


def count_reads(paths, out_prefix, k, signature_len, signature_map, lut_prefix_len, cutoff_min=2, cutoff_max=1_000_000_000, counter_max=255,
                both_strands=True, batch_bytes=1 << 26, device=0, n_bins=None):
    """KMC's two stages on one GPU in RAM mode: every batch of every file is split on the GPU and the bin fragments stay in host memory;
    then bin by bin, in bin-id order, stage 2 and the database writer.  Bin b's signatures (the map's preimage of b) go into .kmc_pre.
    n_bins defaults to the largest map value + 1.  Returns the writer's totals and the split's counts."""
    sig_map = np.ascontiguousarray(signature_map, dtype=np.uint32)
    n_bins = int(sig_map.max()) + 1 if n_bins is None else int(n_bins)
    t0 = time.perf_counter()
    # the splitter first: the stage-2 context sizes its block limit from the HBM that is free when it is created
    sp = Splitter(k, signature_len, sig_map, n_bins, device, max_batch_bytes=batch_bytes)
    parts = [[] for _ in range(n_bins)]
    n_super = n_kmers = n_bases = 0
    for path in paths:
        with open(path, "rb") as f:
            seq = sequences_to_batch(f.read())
        for batch in batches(seq, batch_bytes):
            out, packs, frags = sp.split_raw(batch)
            n_bases += batch.size
            for b, fr in enumerate(frags):
                if fr.bytes:
                    parts[b].append((out[fr.byte_off:fr.byte_off + fr.bytes].copy(), packs[fr.pack0:fr.pack0 + fr.n_packs].copy(), int(fr.n_rec)))
                    n_super += int(fr.n_super_kmers)
                    n_kmers += int(fr.n_rec)
    sp.close()
    t1 = time.perf_counter()
    ctx = Stage2Context(Stage2Params(k, both_strands, cutoff_min, cutoff_max, counter_max, lut_prefix_len), device=device)
    counter_size = ctx.out_rec_bytes - (k - lut_prefix_len) // 4
    w = DbWriter(out_prefix, k, counter_size, lut_prefix_len, signature_len, cutoff_min, cutoff_max, both_strands)
    lut = np.empty(ctx.lut_entries, dtype=np.uint64)
    order = np.argsort(sig_map, kind="stable")
    first = np.searchsorted(sig_map[order], np.arange(n_bins + 1))
    for b in range(n_bins):
        data = np.concatenate([p[0] for p in parts[b]]) if parts[b] else np.zeros(0, dtype=np.uint8)
        data = np.concatenate([data, np.zeros(64, dtype=np.uint8)])    # the stage-2 walk reads past the end of a bin
        packs = np.concatenate([p[1] for p in parts[b]]).astype(np.uint64) if parts[b] else np.zeros(0, dtype=np.uint64)
        n_rec = sum(p[2] for p in parts[b])
        parts[b] = None
        cap = max(ctx.out_capacity(n_rec), 64)
        ptr = w.reserve(cap)
        ctx.submit_bin(0, data.ctypes.data, data.size - 64, n_rec, packs, ptr, cap, lut.ctypes.data, bin_id=b)
        nbytes, stats = ctx.wait_bin_scanned(0, w.records)
        w.commit_bin(nbytes, lut, stats, order[first[b]:first[b + 1]])
    totals = w.close()
    ctx.close()
    t2 = time.perf_counter()
    return {"n_unique": totals[0], "n_cutoff_min": totals[1], "n_cutoff_max": totals[2], "n_total": totals[3], "n_super_kmers": n_super,
            "n_kmers": n_kmers, "n_bases": n_bases, "split_s": t1 - t0, "stage2_s": t2 - t1}


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m kmc_b200.reads", description=__doc__.split("\n\n")[0])
    ap.add_argument("inputs", nargs="+", help="FASTQ / FASTA files, then the output prefix")
    ap.add_argument("-k", type=int, default=25)
    ap.add_argument("-p", "--signature-len", type=int, default=9)
    ap.add_argument("--map", help=".npy file with the 4^p + 1 map entries")
    ap.add_argument("--map-from", help="take p and the map from this .kmc_pre")
    ap.add_argument("--lut-prefix-len", type=int, default=None, help="default: the smallest of 7, 3, 11, ... with (k - p) %% 4 == 0")
    ap.add_argument("--ci", type=int, default=2)
    ap.add_argument("--cx", type=int, default=1_000_000_000)
    ap.add_argument("--cs", type=int, default=255)
    ap.add_argument("-b", action="store_true", help="count k-mers as they are, not canonical ones")
    ap.add_argument("--batch-bytes", type=int, default=1 << 26)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    if len(a.inputs) < 2:
        ap.error("give at least one input and the output prefix")
    if a.map_from:
        m, sig_map = signature_map_from_kmc_pre(a.map_from)
    elif a.map:
        m, sig_map = a.signature_len, np.load(a.map)
    else:
        ap.error("give --map or --map-from")
    lp = a.lut_prefix_len
    if lp is None:
        lp = next(p for p in (7, 3, 11, 15, 4, 5, 6, 2, 8, 9, 10, 12, 13, 14, 1) if p < a.k and (a.k - p) % 4 == 0)
    res = count_reads(a.inputs[:-1], a.inputs[-1], a.k, m, sig_map, lp, a.ci, a.cx, a.cs, not a.b, a.batch_bytes, a.device)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
