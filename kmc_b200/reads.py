"""Reads -> KMC database with this library alone: FASTQ / FASTA -> [GPU stage 0 (SignatureStats)] -> batches -> GPU stage 1 (Splitter) ->
GPU stage 2 (Stage2Context) -> .kmc_pre / .kmc_suf (DbWriter).

    python -m kmc_b200.reads -k31 -p9 -n512 reads.fq out_prefix                  # the map chosen from the reads, as KMC does
    python -m kmc_b200.reads -k31 -p9 --map-from ref_db.kmc_pre reads.fq out_prefix

Without a map, the signature map is KMC's: k-mers per signature are counted on the GPU over a sample of the input (the raw bytes of the
files in input order up to the end of the first record at or beyond max(2^28, total input bytes / 100)), the signatures are grouped into
n_bins bins by CSignatureMapper's rule, the split also counts the (k+x)-mers of every bin, and the bins are written in the order the
reference's stage 2 reads them with one thread.  When the sample covers the whole input (one input file of at most 2^28 bytes, or any
input that fits in the sample) the two files are byte-identical to the reference CLI's (`kmc -sr1`, same -n).  For larger inputs the
reference's sample ends on a boundary of its own input parts (their size follows -m / -t, and with several files its reader order), so
its map can differ slightly: the k-mers and their counts are the same, the bins and their order in the files need not be.

With a map (4^p + 1 entries; `signature_map_from_kmc_pre` reads the one a KMC database was built with) the bins are written in bin-id
order, and for the same map and parameters the files are byte-identical to the reference CLI's: the bins hold the same k-mers, and stage 2
and the writer reproduce the reference's output per bin.
"""
import argparse
import json
import struct
import sys
import time

import numpy as np

from . import DbWriter, KmcB200Error, ERR_INVALID, SignatureStats, Splitter, Stage2Context, Stage2Params, signature_map as _signature_map, \
    stage2_bin_order

_NL, _GT, _AT = 10, ord(">"), ord("@")
STATS_SAMPLE_BYTES = 1 << 28                                            # STATS_FASTQ_SIZE (kmc_core/defs.h)
DEFAULT_N_BINS = 512                                                    # kmc -n


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


def _record_end(data, at):
    """End (exclusive) of the FASTQ / FASTA record of `data` that contains byte `at`, or of the last one."""
    a = np.frombuffer(data, dtype=np.uint8)
    ends = np.flatnonzero(a == _NL)
    if a[0] == _AT:                                                     # FASTQ: every 4th line ends a record
        rec_ends = ends[3::4] + 1
    else:                                                               # FASTA: a record ends where the next header starts
        rec_ends = np.append(ends[:-1][a[ends[:-1] + 1] == _GT] + 1, a.size)
    i = int(np.searchsorted(rec_ends, at, side="right"))
    return int(rec_ends[i]) if i < rec_ends.size else a.size


def signature_sample_counts(paths, k, signature_len, batch_bytes=1 << 26, device=0):
    """Stage 0's statistics (CKMC::buildSignatureMapping, kmc_core/kmc.h:974-1075): k-mers per signature, counted on the GPU, over the
    raw bytes of the files in input order up to the end of the first record at or beyond max(2^28, total bytes / 100)."""
    import os
    budget = max(STATS_SAMPLE_BYTES, sum(os.path.getsize(p) for p in paths) // 100)
    st = SignatureStats(k, signature_len, device, max_batch_bytes=batch_bytes)
    for path in paths:
        if budget <= 0:
            break
        with open(path, "rb") as f:
            data = f.read()
        if not data:
            continue
        if len(data) > budget:
            data = data[:_record_end(data, budget - 1)]
        budget -= len(data)
        for batch in batches(sequences_to_batch(data), batch_bytes):
            st.add(batch)
    counts = st.read()
    st.close()
    return counts


def count_reads(paths, out_prefix, k, signature_len, signature_map, lut_prefix_len, cutoff_min=2, cutoff_max=1_000_000_000, counter_max=255,
                both_strands=True, batch_bytes=1 << 26, device=0, n_bins=None):
    """KMC's stages on one GPU in RAM mode: every batch of every file is split on the GPU and the bin fragments stay in host memory;
    then bin by bin, stage 2 and the database writer.  Returns the writer's totals and the split's counts.
    With a signature_map: the bins are written in bin-id order, bin b's signatures (the map's preimage of b) go into .kmc_pre, and n_bins
    defaults to the largest map value + 1.
    With signature_map=None: stage 0 first (signature_sample_counts, then kmc_b200.signature_map with n_bins, default 512), the split
    counts the (k+x)-mers of every bin, and the bins are written in the reference's stage-2 order (kmc_b200.stage2_bin_order); the map in
    .kmc_pre holds every signature's file position, 0 for the signatures that are not allowed."""
    t0 = time.perf_counter()
    if signature_map is None:
        n_bins = DEFAULT_N_BINS if n_bins is None else int(n_bins)
        mapper = _signature_map(signature_sample_counts(paths, k, signature_len, batch_bytes, device), signature_len, n_bins)
        sig_map = np.maximum(mapper, 0).astype(np.uint32)              # no k-mer has a signature that is not allowed
    else:
        mapper = None
        sig_map = np.ascontiguousarray(signature_map, dtype=np.uint32)
        n_bins = int(sig_map.max()) + 1 if n_bins is None else int(n_bins)
    t_stats = time.perf_counter() - t0
    # the splitter first: the stage-2 context sizes its block limit from the HBM that is free when it is created
    sp = Splitter(k, signature_len, sig_map, n_bins, device, max_batch_bytes=batch_bytes)
    if mapper is not None:
        sp.count_kxmers(both_strands)
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
    if mapper is None:
        file_order = np.arange(n_bins)
        order = np.argsort(sig_map, kind="stable")
    else:
        bin_bytes = [sum(p[0].size for p in parts[b]) for b in range(n_bins)]
        bin_recs = [sum(p[2] for p in parts[b]) for b in range(n_bins)]
        file_pos = stage2_bin_order(bin_bytes, bin_recs, sp.kxmer_totals(), k, cutoff_min, cutoff_max, counter_max, lut_prefix_len)
        file_order = np.argsort(file_pos)                               # the bin at every file position
        order = np.argsort(mapper, kind="stable")                      # signatures by bin id; the disallowed ones (-1) come first
        mapper = mapper.astype(np.int64)
    sp.close()
    t1 = time.perf_counter()
    ctx = Stage2Context(Stage2Params(k, both_strands, cutoff_min, cutoff_max, counter_max, lut_prefix_len), device=device)
    counter_size = ctx.out_rec_bytes - (k - lut_prefix_len) // 4
    w = DbWriter(out_prefix, k, counter_size, lut_prefix_len, signature_len, cutoff_min, cutoff_max, both_strands)
    lut = np.empty(ctx.lut_entries, dtype=np.uint64)
    bin_of = sig_map if mapper is None else mapper
    first = np.searchsorted(bin_of[order], np.arange(n_bins + 1))
    for b in file_order:
        b = int(b)
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
            "n_kmers": n_kmers, "n_bases": n_bases, "stats_s": t_stats, "split_s": t1 - t0 - t_stats, "stage2_s": t2 - t1}


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m kmc_b200.reads", description=__doc__.split("\n\n")[0])
    ap.add_argument("inputs", nargs="+", help="FASTQ / FASTA files, then the output prefix")
    ap.add_argument("-k", type=int, default=25)
    ap.add_argument("-p", "--signature-len", type=int, default=9)
    ap.add_argument("-n", "--n-bins", type=int, default=None, help="bins when the map is chosen from the reads (default %d, KMC's -n)" % DEFAULT_N_BINS)
    ap.add_argument("--map", help=".npy file with the 4^p + 1 map entries (default: chosen from the reads, as KMC does)")
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
        m, sig_map = a.signature_len, None
    lp = a.lut_prefix_len
    if lp is None:
        lp = next(p for p in (7, 3, 11, 15, 4, 5, 6, 2, 8, 9, 10, 12, 13, 14, 1) if p < a.k and (a.k - p) % 4 == 0)
    res = count_reads(a.inputs[:-1], a.inputs[-1], a.k, m, sig_map, lp, a.ci, a.cx, a.cs, not a.b, a.batch_bytes, a.device,
                      a.n_bins if sig_map is None else None)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
