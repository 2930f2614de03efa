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

Parsing: by default (parse="host") every file is read whole and parsed in numpy (sequences_to_batch).  With parse="gpu" (`--gpu-parse`)
files are read in chunks of at most batch_bytes - 1 bytes into pinned host buffers by a reader thread, while the GPU parses
(kmc_b200.FastxParser) and splits the previous chunk; the databases, totals and counts are the same.  A FASTQ / FASTA record must then fit
in about half a chunk of raw bytes (the rest of a chunk after its last record end is carried into the next one).

Small k (k <= 13, `count_reads_small_k`, `--small-k`): KMC's small-k mode.  Every k-mer is counted in a direct array of 4^k counters on the
GPU (kmc_b200.SmallKCounter), with no bins, and the database is written in the KMC1 format the reference writes in that mode (version word
0, no signature map), byte for byte `kmc -kK`'s when the reference takes its small-k path.  count_reads takes this path by itself where the
bin path cannot run, k <= signature_len.
"""
import argparse
import json
import os
import queue
import struct
import sys
import threading
import time

import numpy as np

from . import DbWriter, FASTA, FASTQ, FastxParser, KmcB200Error, ERR_INVALID, SignatureStats, SmallKCounter, Splitter, Stage2Context, \
    Stage2Params, signature_map as _signature_map, stage2_bin_order

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
        i = int(np.searchsorted(seps, end - 1, side="right")) - 1      # the last separator that keeps the piece within batch_bytes
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


def fastx_format(data):
    """FASTQ or FASTA (kmc_b200.FASTQ / FASTA) by the first byte of the first non-empty line, as sequences_to_batch decides."""
    a = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.asarray(data, dtype=np.uint8)
    text = np.flatnonzero(a != _NL)
    first = int(a[text[0]]) if text.size else -1
    if first == _AT:
        return FASTQ
    if first == _GT:
        return FASTA
    raise KmcB200Error(ERR_INVALID, "input is neither FASTQ ('@') nor FASTA ('>')")


def _pinned(nbytes):
    import torch
    t = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    return t, t.numpy()


class _RawChunks:
    """One file as raw chunks of at most chunk_bytes in pinned host memory, for the GPU parser.  A reader thread fills two pinned buffers
    in turn with the next chunk_bytes / 2 bytes of the file, so reading the next piece overlaps the work on the current chunk.  Iterating
    gives (chunk, is_final); the caller reports how much of each non-final chunk it parsed with .consumed(n), and the rest (an unfinished
    record) is copied in front of the next piece, so every chunk starts on a record.  close() (or leaving the `with`) ends the thread."""

    def __init__(self, path, chunk_bytes):
        self.size = os.path.getsize(path)
        self.piece = max(1, chunk_bytes // 2)
        self.head = chunk_bytes - self.piece                           # room for the carried rest of the previous chunk
        self.bufs = [_pinned(chunk_bytes) for _ in range(2)]
        self.free, self.full = queue.Queue(), queue.Queue()
        for i in range(2):
            self.free.put(i)
        self.wait_s = 0.0                                               # time the consumer waited for the reader
        self._consumed = None
        self._f = open(path, "rb")
        self._thread = threading.Thread(target=self._read, name="kmc_b200-reader", daemon=True)
        self._thread.start()

    def _read(self):
        try:
            off = 0
            while off < self.size:
                i = self.free.get()
                if i is None:
                    return
                want = min(self.piece, self.size - off)
                n = self._f.readinto(memoryview(self.bufs[i][1])[self.head:self.head + want])
                if n != want:
                    raise KmcB200Error(ERR_INVALID, "short read: the file changed while it was read")
                off += n
                self.full.put((i, n, off >= self.size))
        except BaseException as e:  # noqa: BLE001 - handed to the consumer
            self.full.put(e)

    def consumed(self, n):
        self._consumed = int(n)

    def __iter__(self):
        carry = None                                                    # (buffer, start, end) of the unparsed rest
        while self.size:
            t = time.perf_counter()
            item = self.full.get()
            self.wait_s += time.perf_counter() - t
            if isinstance(item, BaseException):
                raise item
            i, n, final = item
            buf = self.bufs[i][1]
            start = self.head
            if carry is not None:
                j, s, e = carry
                if e - s > self.head:
                    raise KmcB200Error(ERR_INVALID, "a record is longer than the chunk (%d bytes)" % (self.head + self.piece))
                start = self.head - (e - s)
                buf[start:self.head] = self.bufs[j][1][s:e]
                self.free.put(j)
            self._consumed = None
            yield buf[start:self.head + n], final
            if final:
                self.free.put(i)
                return
            if self._consumed is None:
                raise KmcB200Error(ERR_INVALID, "consumed() was not reported for a non-final chunk")
            carry = (i, start + self._consumed, self.head + n)

    def close(self):
        if self._thread.is_alive():
            self.free.put(None)
            self.free.put(None)
            self._thread.join()
        self._f.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class _Parsers:
    """One FastxParser per format met, created on first use."""

    def __init__(self, device, max_chunk_bytes):
        self.device, self.max_chunk_bytes, self.by_format = device, max_chunk_bytes, {}

    def __call__(self, chunk):
        fmt = fastx_format(chunk)
        if fmt not in self.by_format:
            self.by_format[fmt] = FastxParser(fmt, self.device, self.max_chunk_bytes)
        return self.by_format[fmt]

    def close(self):
        for p in self.by_format.values():
            p.close()
        self.by_format = {}


def signature_sample_counts(paths, k, signature_len, batch_bytes=1 << 26, device=0, parse="host"):
    """Stage 0's statistics (CKMC::buildSignatureMapping, kmc_core/kmc.h:974-1075): k-mers per signature, counted on the GPU, over the
    raw bytes of the files in input order up to the end of the first record at or beyond max(2^28, total bytes / 100).
    parse="gpu": the files are parsed on the GPU in chunks of batch_bytes - 1, the sample's end found by the parser's limit."""
    budget = max(STATS_SAMPLE_BYTES, sum(os.path.getsize(p) for p in paths) // 100)
    st = SignatureStats(k, signature_len, device, max_batch_bytes=batch_bytes)
    if parse == "gpu":
        parsers = _Parsers(device, batch_bytes - 1)
        try:
            for path in paths:
                if budget <= 0:
                    break
                size, pos = os.path.getsize(path), 0
                with _RawChunks(path, batch_bytes - 1) as chunks:
                    parser = None
                    for chunk, final in chunks:
                        parser = parser or parsers(chunk)
                        limit = budget - pos if size > budget else None
                        used = st.add_fastx(parser, chunk, final, limit)
                        chunks.consumed(used)
                        pos += used
                        if size > budget and pos >= budget:
                            break
                budget -= pos
        finally:
            parsers.close()
        counts = st.read()
        st.close()
        return counts
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


SMALL_K_MAX = 13


def count_reads_small_k(paths, out_prefix, k, cutoff_min=2, cutoff_max=1_000_000_000, counter_max=255, both_strands=True, batch_bytes=1 << 26,
                        device=0, parse="host"):
    """KMC's small-k mode (kmc_core/kmc.h:677-960) on one GPU, for 1 <= k <= 13: every batch of every file is counted into 4^k counters
    (kmc_b200.SmallKCounter), then the KMC1 database is written (CSmallKCompleter::CompleteKMCFormat).  There are no bins: no signature
    length, no map, and the LUT prefix length is the reference's choice for this mode, returned as `lut_prefix_len`.  parse as for
    count_reads.  Returns the keys count_reads returns (n_super_kmers is 0, n_kmers equals n_total) plus lut_prefix_len."""
    if parse not in ("host", "gpu"):
        raise KmcB200Error(ERR_INVALID, "parse must be 'host' or 'gpu', not %r" % (parse,))
    if not 1 <= k <= SMALL_K_MAX:
        raise KmcB200Error(ERR_INVALID, "the small-k path counts k = 1..%d, not %d" % (SMALL_K_MAX, k))
    t0 = time.perf_counter()
    sk = SmallKCounter(k, both_strands, device, max_batch_bytes=batch_bytes)
    n_bases = 0
    read_s = 0.0
    parsers = _Parsers(device, batch_bytes - 1) if parse == "gpu" else None
    try:
        for path in paths:
            if parsers is not None:
                with _RawChunks(path, batch_bytes - 1) as chunks:
                    parser = None
                    for chunk, final in chunks:
                        parser = parser or parsers(chunk)
                        chunks.consumed(sk.add_fastx(parser, chunk, final))
                        n_bases += sk.last_seq_bytes
                read_s += chunks.wait_s
                continue
            t = time.perf_counter()
            with open(path, "rb") as f:
                data = f.read()
            read_s += time.perf_counter() - t
            seq = sequences_to_batch(data)
            del data
            for batch in batches(seq, batch_bytes):
                sk.add(batch)
                n_bases += batch.size
        t1 = time.perf_counter()
        lp = sk.finish(cutoff_min, cutoff_max, counter_max)[0]
        totals = sk.write_db(out_prefix, cutoff_min, cutoff_max, counter_max)
    finally:
        if parsers is not None:
            parsers.close()
        sk.close()
    t2 = time.perf_counter()
    return {"n_unique": totals[0], "n_cutoff_min": totals[1], "n_cutoff_max": totals[2], "n_total": totals[3], "n_super_kmers": 0,
            "n_kmers": totals[3], "n_bases": n_bases, "stats_s": 0.0, "split_s": t1 - t0, "stage2_s": t2 - t1, "read_s": read_s,
            "lut_prefix_len": lp}


def count_reads(paths, out_prefix, k, signature_len, signature_map, lut_prefix_len, cutoff_min=2, cutoff_max=1_000_000_000, counter_max=255,
                both_strands=True, batch_bytes=1 << 26, device=0, n_bins=None, parse="host", small_k=None):
    """KMC's stages on one GPU in RAM mode: every batch of every file is split on the GPU and the bin fragments stay in host memory;
    then bin by bin, stage 2 and the database writer.  Returns the writer's totals and the split's counts.
    With a signature_map: the bins are written in bin-id order, bin b's signatures (the map's preimage of b) go into .kmc_pre, and n_bins
    defaults to the largest map value + 1.
    With signature_map=None: stage 0 first (signature_sample_counts, then kmc_b200.signature_map with n_bins, default 512), the split
    counts the (k+x)-mers of every bin, and the bins are written in the reference's stage-2 order (kmc_b200.stage2_bin_order); the map in
    .kmc_pre holds every signature's file position, 0 for the signatures that are not allowed.
    parse="host" reads every file whole and parses it in numpy; parse="gpu" reads chunks of batch_bytes - 1 bytes on a reader thread and
    parses them on the GPU (kmc_b200.FastxParser, see the module docstring); the files and counts are the same either way.
    small_k: None takes the small-k path (count_reads_small_k) where the bin path cannot run, k <= signature_len; True takes it for any
    k <= 13, as `kmc` does; False keeps the bin path.  On the small-k path signature_len, signature_map, n_bins and lut_prefix_len are not
    used, and the result also holds the lut_prefix_len the path chose."""
    if parse not in ("host", "gpu"):
        raise KmcB200Error(ERR_INVALID, "parse must be 'host' or 'gpu', not %r" % (parse,))
    if small_k or (small_k is None and k <= signature_len):
        return count_reads_small_k(paths, out_prefix, k, cutoff_min, cutoff_max, counter_max, both_strands, batch_bytes, device, parse)
    t0 = time.perf_counter()
    if signature_map is None:
        n_bins = DEFAULT_N_BINS if n_bins is None else int(n_bins)
        mapper = _signature_map(signature_sample_counts(paths, k, signature_len, batch_bytes, device, parse), signature_len, n_bins)
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
    read_s = 0.0

    def keep(out, packs, frags):
        nonlocal n_super, n_kmers
        for b, fr in enumerate(frags):
            if fr.bytes:
                parts[b].append((out[fr.byte_off:fr.byte_off + fr.bytes].copy(), packs[fr.pack0:fr.pack0 + fr.n_packs].copy(), int(fr.n_rec)))
                n_super += int(fr.n_super_kmers)
                n_kmers += int(fr.n_rec)

    parsers = _Parsers(device, batch_bytes - 1) if parse == "gpu" else None
    try:
        for path in paths:
            if parsers is not None:
                with _RawChunks(path, batch_bytes - 1) as chunks:
                    parser = None
                    for chunk, final in chunks:
                        parser = parser or parsers(chunk)
                        out, packs, frags, used, nseq = sp.split_fastx(parser, chunk, final)
                        chunks.consumed(used)
                        n_bases += nseq
                        keep(out, packs, frags)
                read_s += chunks.wait_s
                continue
            t = time.perf_counter()
            with open(path, "rb") as f:
                data = f.read()
            read_s += time.perf_counter() - t
            seq = sequences_to_batch(data)
            del data
            for batch in batches(seq, batch_bytes):
                out, packs, frags = sp.split_raw(batch)
                n_bases += batch.size
                keep(out, packs, frags)
    finally:
        if parsers is not None:
            parsers.close()
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
            "n_kmers": n_kmers, "n_bases": n_bases, "stats_s": t_stats, "split_s": t1 - t0 - t_stats, "stage2_s": t2 - t1, "read_s": read_s}


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
    ap.add_argument("--gpu-parse", action="store_true", help="parse FASTQ / FASTA on the GPU in chunks of batch-bytes - 1 (default: numpy, whole files)")
    ap.add_argument("--small-k", action="store_true",
                    help="k <= 13: count in 4^k direct counters and write a KMC1 database, as kmc does (taken without the flag when k <= p)")
    a = ap.parse_args(argv)
    if len(a.inputs) < 2:
        ap.error("give at least one input and the output prefix")
    parse = "gpu" if a.gpu_parse else "host"
    if a.map_from:
        m, sig_map = signature_map_from_kmc_pre(a.map_from)
    elif a.map:
        m, sig_map = a.signature_len, np.load(a.map)
    else:
        m, sig_map = a.signature_len, None
    if a.small_k or a.k <= m:                                           # no bins: no map, and the path picks its own LUT prefix length
        print(json.dumps(count_reads_small_k(a.inputs[:-1], a.inputs[-1], a.k, a.ci, a.cx, a.cs, not a.b, a.batch_bytes, a.device, parse)))
        return 0
    lp = a.lut_prefix_len
    if lp is None:
        lp = next(p for p in (7, 3, 11, 15, 4, 5, 6, 2, 8, 9, 10, 12, 13, 14, 1) if p < a.k and (a.k - p) % 4 == 0)
    res = count_reads(a.inputs[:-1], a.inputs[-1], a.k, m, sig_map, lp, a.ci, a.cx, a.cs, not a.b, a.batch_bytes, a.device,
                      a.n_bins if sig_map is None else None, parse=parse, small_k=False)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
