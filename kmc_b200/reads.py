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

Histogram estimation (`estimate_histogram`, `-e`): KMC's ntHash estimator (`kmc -e`) on the GPU (kmc_b200.HistogramEstimator), for
1 <= k <= 256; the file `-e` writes is the reference's, "i<TAB>count" per line.  count_reads(opt_out_size=True) runs the same estimator over
the chunks it splits and picks the LUT prefix length from the estimated number of counted k-mers, as `kmc --opt-out-size` does.

    python -m kmc_b200.reads -e -k31 reads.fq hist.txt

Homopolymer compression (`homopolymer_compressed=True`, `--hc`): `kmc -hc`.  Every run of one base in a read (case ignored) is collapsed
to a single base on the GPU before the statistics, the split and the small-k count see it (Splitter / SignatureStats / SmallKCounter
set_homopolymer_compressed).  The histogram estimator sees the reads uncompressed, as in the reference, so `-e --hc` writes the file `-e`
writes and `--opt-out-size --hc` picks the LUT prefix length from the uncompressed k-mers.  n_bases counts the input bases; n_kmers and
n_super_kmers are counted after compression.  The files are `kmc -hc -sr1`'s for records shorter than 524,296 symbols: the reference cuts
longer records into parts and compresses each part on its own (DESIGN.md section 3.13), the GPU compresses every record whole.

    python -m kmc_b200.reads --hc -k31 reads.fq out_prefix

gzip input: a file that starts with 1f 8b is gzip (a FASTQ / FASTA text never does), whatever its name, and FASTQ or FASTA is decided on
its text.  parse="host" inflates the whole file with zlib, every member.  parse="gpu" inflates BGZF members (what `bgzip` writes) on the
GPU (kmc_b200.Gunzip) on the reader thread, into the chunk behind the carried rest; from the first member that is not BGZF on (plain
`gzip`, concatenated members) zlib inflates the rest on that thread.  The text is zlib's byte for byte, so the databases, -e files and
totals are those of the same text uncompressed.  As in the reference, a gzip file counts 3.2 times its bytes in the predicted input size
(stage 0's sample budget, the estimator's s); the sample itself and the parser's limit count text bytes.

    python -m kmc_b200.reads --gpu-parse -k31 reads.fq.gz out_prefix

BAM input (`kmc -fbam`): a gzip file whose text starts with "BAM\\1" is BAM, whatever its name.  It must be BGZF throughout and end with
the 28-byte BGZF EOF member (as in the reference, binary_reader.h:159-174).  The header (text and references) is skipped; every record
whose FLAG has neither 0x100 (secondary) nor 0x800 (supplementary) is one read, its SEQ decoded to A, C, G, T and N for every other code
(CSplitter::GetSeq, splitter.cpp:326-418).  With both_strands=False (`-b`) the records of FLAG 0x10 are reverse complemented back to their
original strand, as the reference does; canonical counting uses SEQ as stored, which gives the same k-mers but other super-k-mer cuts.
parse="host" walks the records serially and decodes in numpy (bam_to_batch); parse="gpu" inflates the members on the GPU, skips the header
on the reader thread and walks and decodes the records on the GPU (kmc_b200.FastxParser with BAM / BAM_ORIGINAL_STRAND).  A BAM file counts
0.7 times its bytes in the predicted input size; stage 0's sample counts record bytes.  The files are the reference's for records shorter
than 524,296 bases (its read buffer, kmc.h:419).

    python -m kmc_b200.reads --gpu-parse -k31 reads.bam out_prefix

KMC database input (`kmc -fkmc`): an input named by its prefix, where P.kmc_pre and P.kmc_suf exist, is a KMC database; either every
input is one or none is.  Every record whose counter passes the database's own cutoffs is one read, its k-mer (CKMCFile::ReadNextKmer,
printed as FASTA by CBinaryFilesReader::ProcessKMC); a k above the database's gives no k-mers.  KMC1 and KMC2 databases are read; on the
bin path stage 0 is skipped and the signature map is the first database's (kmc_input_signature_map: it must be KMC2, with the same
signature length and number of bins, or the run is refused with the reference's message).  n_reads counts the kept records, and the
predicted input size is the last database's total_kmers.  parse="host" decodes in numpy (kmc_db_to_batch); parse="gpu" reads .kmc_suf
in chunks of whole records on a reader thread and decodes them on the GPU (kmc_b200.KmcDbDecoder).

    python -m kmc_b200.reads --gpu-parse -k25 db31 out_prefix
"""
import argparse
import json
import os
import queue
import struct
import sys
import threading
import time
import zlib

import numpy as np

from . import BAM, BAM_ORIGINAL_STRAND, DbWriter, FASTA, FASTQ, FastxParser, Gunzip, HistogramEstimator, KmcB200Error, KmcDbDecoder, ERR_INVALID, SignatureStats, SmallKCounter, \
    Splitter, Stage2Context, Stage2Params, bgzf_scan, signature_map as _signature_map, stage2_bin_order

_NL, _GT, _AT = 10, ord(">"), ord("@")
STATS_SAMPLE_BYTES = 1 << 28                                            # STATS_FASTQ_SIZE (kmc_core/defs.h)
DEFAULT_N_BINS = 512                                                    # kmc -n
GZIP_MAGIC = b"\x1f\x8b"
GZIP_SIZE_FACTOR = 3.2                                                  # binary_reader.h:378-386: a gzip file's predicted text size
BGZF_MAX_TEXT = 1 << 16                                                 # text of one BGZF member, at most
_ZLIB_READ = 1 << 18                                                    # compressed bytes per zlib step on the reader thread
BAM_MAGIC = b"BAM\1"
BAM_SIZE_FACTOR = 0.7                                                   # binary_reader.h:368-371: a BAM file's predicted size
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")   # the SAM/BAM specification's empty last member
_BAM_FIXED = 36                                                         # block_size and the 32 bytes of fixed fields


def is_gzip(path):
    """The file starts with the gzip magic 1f 8b.  A FASTQ / FASTA text never does (its first byte is '@', '>' or a line break)."""
    with open(path, "rb") as f:
        return f.read(2) == GZIP_MAGIC


def is_bam(path):
    """A gzip file whose text starts with the BAM magic "BAM\\1" (decided on content: the name does not matter)."""
    with open(path, "rb") as f:
        data = f.read(1 << 16)
    if data[:2] != GZIP_MAGIC:
        return False
    try:
        return zlib.decompressobj(31).decompress(data, len(BAM_MAGIC)) == BAM_MAGIC
    except zlib.error:
        return False


def _input_size(path):
    size = os.path.getsize(path)
    if is_bam(path):
        return int(BAM_SIZE_FACTOR * size)
    return int(GZIP_SIZE_FACTOR * size) if is_gzip(path) else size


def predicted_size(paths):
    """The input size the reference plans with (CBinaryFilesReader, binary_reader.h:360-386): a plain file counts its bytes, a gzip file
    (uint64)(3.2 * its bytes), a BAM file (uint64)(0.7 * its bytes).  The reference tells gzip by the name's ".gz" and BAM by -fbam, this
    library both by the file's first bytes.  KMC database input (every path a database prefix) is the last database's total_kmers: the
    reference assigns it rather than adding it up (binary_reader.h:372-375)."""
    if _kmc_inputs(paths):
        return _kmc_predicted_size(paths)
    return sum(_input_size(p) for p in paths)


def _gzip_error(e):
    return KmcB200Error(ERR_INVALID, "gzip input: %s" % e)


def _zlib_members(data, more=None):
    """Text blocks of gzip data with zlib, member after member (inflateReset for each further member, as the reference's reader does).
    more(): further compressed bytes (b"" at the end of the file).  A member cut short at the end is an error."""
    d, fresh = zlib.decompressobj(31), True
    while True:
        if not data:
            data = more() if more else b""
            if not data:
                if not fresh:
                    raise _gzip_error("the last member is truncated")
                return
        try:
            t = d.decompress(data)
        except zlib.error as e:
            raise _gzip_error(e) from None
        fresh = False
        if d.eof:
            data, d, fresh = d.unused_data, zlib.decompressobj(31), True
        else:
            data = b""
        if t:
            yield t


def read_text(path):
    """The whole text of a FASTQ / FASTA file, inflated with zlib (every member) when it is gzip."""
    with open(path, "rb") as f:
        data = f.read()
    return b"".join(_zlib_members(data)) if data[:2] == GZIP_MAGIC else data


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


def _bam_error(msg):
    return KmcB200Error(ERR_INVALID, "BAM input: %s" % msg)


def check_bgzf_members(data):
    """A BAM file's members: every one BGZF (its BC subfield gives its length), the last one the EOF member."""
    if not data.endswith(BGZF_EOF):
        raise _bam_error("wrong EOF marker (the file does not end with the BGZF EOF member)")
    pos = 0
    while pos < len(data):
        size = _bgzf_member_size(data, pos)
        if size is None:
            raise _bam_error("member at byte %d is not BGZF" % pos)
        pos += size
    if pos != len(data):
        raise _bam_error("the last member is truncated")


def _bgzf_member_size(data, pos):
    """BSIZE + 1 of the BGZF member at data[pos:], or None when it is not one: the gzip header with FEXTRA alone and a BC subfield of
    length 2 among its extra subfields (any others are skipped), the rule kmcb200_bgzf_scan applies."""
    if len(data) - pos < 12 or data[pos:pos + 4] != b"\x1f\x8b\x08\x04":
        return None
    xlen, = struct.unpack_from("<H", data, pos + 10)
    end = pos + 12 + xlen
    if end > len(data):
        return None
    q = pos + 12
    while q + 4 <= end:
        slen, = struct.unpack_from("<H", data, q + 2)
        if data[q:q + 2] == b"BC" and slen == 2 and q + 6 <= end:
            size = struct.unpack_from("<H", data, q + 4)[0] + 1
            return size if size >= 12 + xlen + 8 + 2 else None
        q += 4 + slen
    return None


class BamHeader:
    """The BAM header (magic, l_text, text, n_ref, and l_name, name, l_ref of every reference), skipped piece by piece: feed(piece) returns
    where the records start in the piece, or None while the whole piece is header.  A header may span any number of pieces."""

    def __init__(self):
        self.need, self.field, self.buf = 4, "magic", b""              # bytes still wanted for the current field
        self.n_ref = 0
        self.done = False

    def feed(self, piece):
        mv = memoryview(piece).cast("B")
        pos = 0
        while not self.done:
            take = min(self.need, len(mv) - pos)
            if self.field in ("text", "name"):                          # skipped bytes
                self.need -= take
            else:
                self.buf += bytes(mv[pos:pos + take])
                self.need -= take
            pos += take
            if self.need:
                return None
            self._next()
        return pos

    def _next(self):
        f, v = self.field, self.buf
        self.buf = b""
        if f == "magic":
            if v != BAM_MAGIC:
                raise _bam_error("the text does not start with the BAM magic")
            self.field, self.need = "l_text", 4
        elif f == "l_text":
            self.field, self.need = "text", self._count(v, "l_text")
        elif f == "text":
            self.field, self.need = "n_ref", 4
        elif f == "n_ref":
            self.n_ref = self._count(v, "n_ref")
            self._ref_or_done()
        elif f == "l_name":
            self.field, self.need = "name", self._count(v, "l_name")
        elif f == "name":
            self.field, self.need = "l_ref", 4
        else:                                                           # l_ref
            self.n_ref -= 1
            self._ref_or_done()
        if self.field in ("text", "name") and self.need == 0:
            self._next()

    def _ref_or_done(self):
        if self.n_ref:
            self.field, self.need = "l_name", 4
        else:
            self.done = True

    @staticmethod
    def _count(v, name):
        n = struct.unpack("<i", v)[0]
        if n < 0:
            raise _bam_error("negative %s in the header" % name)
        return n

    def finish(self):
        if not self.done:
            raise _bam_error("the header is truncated")


def bam_records(data):
    """The record bytes of a whole decompressed BAM file: the text after its header."""
    h = BamHeader()
    at = h.feed(data)
    h.finish()
    return memoryview(data)[at:]


def bam_walk(records):
    """The records of decompressed BAM record bytes, serially (CSplitter::GetSeq): (start, l_seq, flag, seq offset) per record.  A
    block_size below 32, a negative l_seq, fixed fields longer than block_size, or bytes after the last whole record raise ERR_INVALID."""
    out = []
    p, n = 0, len(records)
    while p < n:
        if n - p < 4:
            raise _bam_error("the last record is truncated")
        bs = struct.unpack_from("<i", records, p)[0]
        if bs < 32:
            raise _bam_error("a malformed record at byte %d: block_size %d" % (p, bs))
        if n - p - 4 < bs:
            raise _bam_error("the last record is truncated")
        l_name, n_cigar, flag, l_seq = records[p + 12], *struct.unpack_from("<HHi", records, p + 16)
        if l_seq < 0 or 32 + l_name + 4 * n_cigar + (l_seq + 1) // 2 + l_seq > bs:
            raise _bam_error("a malformed record at byte %d" % p)
        out.append((p, l_seq, flag, p + _BAM_FIXED + l_name + 4 * n_cigar))
        p += 4 + bs
    return out


def bam_record_end(records, at):
    """End (exclusive) of the BAM record of `records` that contains byte `at` (records of a whole walk)."""
    ends = np.array([r[0] for r in bam_walk(records)[1:]] + [len(records)], dtype=np.int64)
    return int(ends[np.searchsorted(ends, at, side="right")])


_BAM_BASE = np.frombuffer(b"NACNGNNNTNNNNNNN", dtype=np.uint8)      # =ACMGRSVTWYHKDBN: A C G T at codes 1 2 4 8, N elsewhere
_BAM_COMP = np.frombuffer(b"NTGNCNNNANNNNNNN", dtype=np.uint8)


def bam_records_to_batch(records, original_strand=False):
    """Decompressed BAM record bytes -> the batch CSplitter::GetSeq reads: every record without FLAG 0x100 / 0x800 becomes its SEQ
    (A C G T, N for every other code) and one newline; with original_strand, the records of FLAG 0x10 reverse complemented."""
    a = _as_array(records)
    recs = [r for r in bam_walk(records) if not r[2] & 0x900]
    if not recs:
        return np.zeros(0, dtype=np.uint8)
    r = np.array(recs, dtype=np.int64)
    lens, flags, seq = r[:, 1], r[:, 2], r[:, 3]
    rev = (flags & 0x10) != 0 if original_strand else np.zeros(len(r), dtype=bool)
    out = np.full(int(lens.sum()) + len(r), _NL, dtype=np.uint8)
    out_off = np.concatenate([[0], np.cumsum(lens + 1)[:-1]])
    cum = np.cumsum(lens)
    i = 0
    while i < len(r):                                                   # about 2^22 bases per step, at least one record
        j = max(i + 1, int(np.searchsorted(cum, cum[i] - lens[i] + (1 << 22), side="right")))
        ln = lens[i:j]
        rid = np.repeat(np.arange(j - i), ln)
        within = np.arange(int(ln.sum()), dtype=np.int64) - np.repeat(np.concatenate([[0], np.cumsum(ln)[:-1]]), ln)
        rv = rev[i:j][rid]
        k = np.where(rv, ln[rid] - 1 - within, within)
        byte = a[seq[i:j][rid] + k // 2]
        nib = np.where(k & 1, byte & 15, byte >> 4)
        out[out_off[i:j][rid] + within] = np.where(rv, _BAM_COMP[nib], _BAM_BASE[nib])
        i = j
    return out


def bam_to_batch(data, original_strand=False):
    """A whole decompressed BAM file -> its batch: the header skipped, then bam_records_to_batch."""
    return bam_records_to_batch(bam_records(data), original_strand)


def read_bam(path):
    """The decompressed text of a BAM file (every member checked to be BGZF, the EOF member last), inflated with zlib."""
    with open(path, "rb") as f:
        data = f.read()
    check_bgzf_members(data)
    return b"".join(_zlib_members(data))


def bam_n_reads(records):
    """The reads a BAM file gives: its records without FLAG 0x100 / 0x800."""
    return sum(1 for r in bam_walk(records) if not r[2] & 0x900)


def _read_input(path):
    """(data, bam): a BAM file's record bytes (header skipped), or the text of a FASTQ / FASTA file."""
    if is_bam(path):
        return bam_records(read_bam(path)), True
    return read_text(path), False


def _to_batch(data, bam, original_strand=False):
    return bam_records_to_batch(data, original_strand) if bam else sequences_to_batch(data)


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


KMC_PRE_MARKER, KMC_SUF_MARKER = b"KMCP", b"KMCS"
KMC1_VERSION, KMC2_VERSION = 0, 0x200
_KMC_ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
_KMC_NOT_V2 = ("currently only KMC databases in version 2 can be readed. If needed to read other version please post an GitHub issue.")


def is_kmc_db(path):
    """`path` names a KMC database by its prefix: path.kmc_pre and path.kmc_suf both exist (what `kmc -fkmc` takes)."""
    return os.path.isfile(path + ".kmc_pre") and os.path.isfile(path + ".kmc_suf")


def _kmc_inputs(paths):
    """True when every input is a KMC database, False when none is: kmc's -f applies to all inputs."""
    db = [is_kmc_db(p) for p in paths]
    if any(db) and not all(db):
        raise KmcB200Error(ERR_INVALID, "either every input is a KMC database or none is (kmc's -f applies to all inputs)")
    return bool(db) and all(db)


class KmcDbInfo:
    """The header of a KMC database as the reference's reader takes it (CKMCFile::ReadParamsFrom_prefix_file_buf, kmc_file.cpp:178-325),
    and the LUT as its listing reader sees it: for KMC2 every stored word, for KMC1 the 4^lut_prefix_len stored words followed by
    total_kmers (the guard of kmc_file.h:57-58).  n_bins and signature_map (the stored file positions) are those of a KMC2 database."""

    def __init__(self, prefix):
        self.prefix = prefix
        with open(prefix + ".kmc_pre", "rb") as f:
            pre = f.read()
        if len(pre) < 16 or pre[:4] != KMC_PRE_MARKER or pre[-4:] != KMC_PRE_MARKER:
            raise KmcB200Error(ERR_INVALID, "%s.kmc_pre is not a KMC database (no KMCP markers)" % prefix)
        u32 = lambda at: struct.unpack_from("<I", pre, at)[0]                                            # noqa: E731
        self.version = u32(len(pre) - 12)
        if self.version not in (KMC1_VERSION, KMC2_VERSION):
            raise KmcB200Error(ERR_INVALID, "%s.kmc_pre: version word %#x is neither KMC1 (0) nor KMC2 (0x200)" % (prefix, self.version))
        header_offset = u32(len(pre) - 8)
        h = len(pre) - 8 - header_offset
        self.kmer_len, mode, self.counter_size, self.lut_prefix_len = (u32(h + 4 * i) for i in range(4))
        if mode != 0:
            raise KmcB200Error(ERR_INVALID, "%s: Quake compatible counters are not supported anymore" % prefix)
        if self.counter_size > 4:
            raise KmcB200Error(ERR_INVALID, "%s: counters of %d bytes are not read (the reference accumulates a counter into 32 bits)"
                               % (prefix, self.counter_size))
        if self.lut_prefix_len > self.kmer_len or (self.kmer_len - self.lut_prefix_len) % 4:
            raise KmcB200Error(ERR_INVALID, "%s: lut_prefix_len %d does not fit k = %d" % (prefix, self.lut_prefix_len, self.kmer_len))
        lut_words = 1 << (2 * self.lut_prefix_len)
        if self.version == KMC2_VERSION:
            self.signature_len, self.min_count, self.max_count = u32(h + 16), u32(h + 20), u32(h + 24)
            self.total_kmers = struct.unpack_from("<Q", pre, h + 28)[0]
            self.both_strands = pre[h + 36] == 0
            map_size = (1 << (2 * self.signature_len)) + 1
            map_at = h - 4 * map_size
            self.lut = np.frombuffer(pre, dtype=np.uint64, count=(map_at - 4) // 8, offset=4).copy()
            self.n_bins = (map_at - 4 - 8) // (8 * lut_words)
            self.signature_map = np.frombuffer(pre, dtype=np.uint32, count=map_size, offset=map_at).copy()
        else:
            self.signature_len, self.min_count = None, u32(h + 16)
            self.total_kmers = struct.unpack_from("<Q", pre, h + 24)[0]
            self.both_strands = pre[h + 32] == 0
            self.max_count = u32(h + 20) + (u32(h + 33) << 32)
            self.lut = np.append(np.frombuffer(pre, dtype=np.uint64, count=lut_words, offset=4), np.uint64(self.total_kmers))
            self.n_bins = self.signature_map = None
        self.suffix_bytes = (self.kmer_len - self.lut_prefix_len) // 4
        self.record_bytes = self.suffix_bytes + self.counter_size
        suf_size = os.path.getsize(prefix + ".kmc_suf")
        if suf_size < 4 + self.total_kmers * self.record_bytes:
            raise KmcB200Error(ERR_INVALID, "%s.kmc_suf holds fewer than total_kmers = %d records" % (prefix, self.total_kmers))

    def decoder(self, device=0, max_records=1 << 22):
        """A KmcDbDecoder of this database with its LUT on the GPU."""
        return KmcDbDecoder(self.kmer_len, self.lut_prefix_len, self.counter_size, self.min_count, self.max_count, self.total_kmers,
                            self.lut, device, max_records)


def kmc_db_info(prefix):
    """The header and the listing LUT of the KMC database `prefix` (KmcDbInfo).  ERR_INVALID for what the reference refuses to read
    (neither version 0 nor 0x200, Quake-compatible counters) and for counters of more than 4 bytes."""
    return KmcDbInfo(prefix)


def kmc_db_records(info):
    """The records of .kmc_suf, uint8[total_kmers, record_bytes] (after the KMCS marker)."""
    with open(info.prefix + ".kmc_suf", "rb") as f:
        if f.read(4) != KMC_SUF_MARKER:
            raise KmcB200Error(ERR_INVALID, "%s.kmc_suf does not start with KMCS" % info.prefix)
        data = np.fromfile(f, dtype=np.uint8, count=info.total_kmers * info.record_bytes)
    return data.reshape(info.total_kmers, info.record_bytes)


def kmc_records_to_batch(info, recs, first_record):
    """The host model of KmcDbDecoder: records first_record .. (uint8[n, record_bytes]) -> the batch, every kept record's k-mer in ACGT
    and '\\n' (CKMCFile::ReadNextKmer, kmc_file.cpp:427-499, printed by CBinaryFilesReader::ProcessKMC, binary_reader.h:238-304)."""
    recs = np.asarray(recs, dtype=np.uint8).reshape(-1, info.record_bytes)
    g = np.arange(first_record, first_record + recs.shape[0], dtype=np.uint64)
    if info.counter_size:
        cnt = np.zeros(recs.shape[0], dtype=np.uint64)
        for b in range(info.counter_size):
            cnt |= recs[:, info.suffix_bytes + b].astype(np.uint64) << np.uint64(8 * b)
        keep = (cnt >= info.min_count) & (cnt <= min(int(info.max_count), (1 << 64) - 1))
        recs, g = recs[keep], g[keep]
    k, lp = info.kmer_len, info.lut_prefix_len
    prefix = np.searchsorted(info.lut[1:], g, side="right").astype(np.uint64) & np.uint64((1 << (2 * lp)) - 1)
    out = np.empty((recs.shape[0], k + 1), dtype=np.uint8)
    for i in range(lp):
        out[:, i] = _KMC_ACGT[(prefix >> np.uint64(2 * (lp - 1 - i))) & np.uint64(3)]
    for j in range(4):
        out[:, lp + j:k:4] = _KMC_ACGT[(recs[:, :info.suffix_bytes] >> (6 - 2 * j)) & 3]
    out[:, k] = _NL
    return out.reshape(-1)


def kmc_db_to_batch(prefix):
    """The batch `kmc -fkmc` reads from the KMC database `prefix`: kmc_records_to_batch of all its records."""
    info = kmc_db_info(prefix)
    return kmc_records_to_batch(info, kmc_db_records(info), 0)


def kmc_input_signature_map(prefix, signature_len, n_bins=None):
    """CSignatureMapper::InitKMC (kmc_core/s_mapper.h:47-140): the signature map of a bin-path run on KMC database input, taken from the
    first database.  The stored map values (file positions) are grouped in ascending order and the groups numbered 0, 1, ...; the special
    signature 4^p goes to n_bins - 1 and its group does not advance the number.  Returns (int64[4^p + 1], n_bins).  n_bins=None takes
    the database's number of LUT arrays; like kmc, ERR_INVALID for a KMC1 database, another signature length or another n_bins."""
    info = kmc_db_info(prefix)
    if info.version != KMC2_VERSION:
        raise KmcB200Error(ERR_INVALID, _KMC_NOT_V2)
    if info.signature_len != signature_len:
        raise KmcB200Error(ERR_INVALID, "Wrong signature length, should be the same as input KMC database: %d" % info.signature_len)
    if n_bins is not None and int(n_bins) != info.n_bins:
        raise KmcB200Error(ERR_INVALID, "Wrong number of bins, should be the same as input KMC database: %d" % info.n_bins)
    stored = info.signature_map
    special = stored.size - 1
    order = np.argsort(stored, kind="stable")
    vals = stored[order]
    group = np.cumsum(np.r_[True, vals[1:] != vals[:-1]]) - 1
    special_group = group[np.flatnonzero(order == special)[0]]
    bins = np.empty(stored.size, dtype=np.int64)
    bins[order] = group - (group > special_group)
    bins[special] = info.n_bins - 1
    return bins, info.n_bins


def _kmc_predicted_size(paths):
    """binary_reader.h:372-375: with KMC input the predicted size is the last database's total_kmers (assigned, not added)."""
    return kmc_db_info(paths[-1]).total_kmers if paths else 0


class _KmcSufChunks:
    """The records of one KMC database as chunks of at most max_records whole records in pinned host memory, read by a reader thread into
    two buffers in turn, so reading the next chunk overlaps the work on the current one.  Iterating gives (records, first_record)."""

    def __init__(self, info, max_records):
        self.info, self.per = info, max(1, int(max_records))
        nbytes = self.per * info.record_bytes
        self.bufs = [_pinned(max(1, nbytes)) for _ in range(2)]
        self.free, self.full = queue.Queue(), queue.Queue()
        for i in range(2):
            self.free.put(i)
        self.wait_s = 0.0
        self._f = open(info.prefix + ".kmc_suf", "rb")
        if self._f.read(4) != KMC_SUF_MARKER:
            self._f.close()
            raise KmcB200Error(ERR_INVALID, "%s.kmc_suf does not start with KMCS" % info.prefix)
        self._thread = threading.Thread(target=self._read, name="kmc_b200-kmc-reader", daemon=True)
        self._thread.start()

    def _read(self):
        try:
            first = 0
            while first < self.info.total_kmers:
                i = self.free.get()
                if i is None:
                    return
                n = min(self.per, self.info.total_kmers - first)
                want = n * self.info.record_bytes
                if self._f.readinto(memoryview(self.bufs[i][1])[:want]) != want:
                    raise KmcB200Error(ERR_INVALID, "short read: the file changed while it was read")
                self.full.put((i, want, first))
                first += n
            self.full.put(None)
        except BaseException as e:  # noqa: BLE001 - handed to the consumer
            self.full.put(e)

    def __iter__(self):
        prev = None
        while True:
            t = time.perf_counter()
            item = self.full.get()
            self.wait_s += time.perf_counter() - t
            if prev is not None:
                self.free.put(prev)
            if isinstance(item, BaseException):
                raise item
            if item is None:
                return
            i, want, first = item
            prev = i
            yield self.bufs[i][1][:want], first

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


def _kmc_chunks(paths, batch_bytes, device, parse):
    """The databases' records in chunks whose batch fits batch_bytes: (info, decoder, records, first_record, batch) per chunk.
    parse="host": decoder and records are None and batch is the numpy model's (kmc_records_to_batch).  parse="gpu": .kmc_suf is read on a
    reader thread into pinned buffers, batch is None, and the caller decodes the records on the GPU with the decoder (KmcDbDecoder)."""
    for path in paths:
        info = kmc_db_info(path)
        per = max(1, batch_bytes // (info.kmer_len + 1))
        if parse == "gpu":
            dec = info.decoder(device, per)
            try:
                with _KmcSufChunks(info, per) as chunks:
                    for recs, first in chunks:
                        yield info, dec, recs, first, None
            finally:
                dec.close()
            continue
        recs = kmc_db_records(info)
        for first in range(0, info.total_kmers, per):
            yield info, None, None, first, kmc_records_to_batch(info, recs[first:first + per], first)


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
    record) is copied in front of the next piece, so every chunk starts on a record.  close() (or leaving the `with`) ends the thread.
    A gzip file gives its text the same way, chunk_bytes / 2 text bytes per piece (_GzText); a BAM file its record bytes, the header
    skipped on the reader thread (.bam is True)."""

    def __init__(self, path, chunk_bytes, device=0):
        self.size = os.path.getsize(path)
        self.piece = max(1, chunk_bytes // 2)
        self.head = chunk_bytes - self.piece                           # room for the carried rest of the previous chunk
        self.bufs = [_pinned(chunk_bytes) for _ in range(2)]
        self.free, self.full = queue.Queue(), queue.Queue()
        for i in range(2):
            self.free.put(i)
        self.wait_s = 0.0                                               # time the consumer waited for the reader
        self._consumed = None
        self.bam = is_bam(path)
        self._f = open(path, "rb")
        if self.bam:
            self._f.seek(-min(len(BGZF_EOF), self.size), os.SEEK_END)
            if self._f.read(len(BGZF_EOF)) != BGZF_EOF:
                self._f.close()
                raise _bam_error("wrong EOF marker (the file does not end with the BGZF EOF member)")
            self._f.seek(0)
        self._gz = _GzText(self._f, self.piece, device, bgzf_only=self.bam) if is_gzip(path) else None
        self._thread = threading.Thread(target=self._read if self._gz is None else self._read_gzip, name="kmc_b200-reader", daemon=True)
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

    def _read_gzip(self):
        hdr = BamHeader() if self.bam else None                          # a BAM file's pieces hold record bytes only
        try:
            while True:
                i = self.free.get()
                if i is None:
                    return
                out = self.bufs[i][1][self.head:self.head + self.piece]
                while True:
                    n, final = self._gz.fill(out)
                    if hdr is not None and not hdr.done:
                        at = hdr.feed(out[:n])
                        if at is None:
                            if final:
                                hdr.finish()
                            continue
                        out[:n - at] = out[at:n].copy()
                        n -= at
                    if n or final:
                        break
                self.full.put((i, n, final))
                if final:
                    return
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
            if final and n == 0 and (carry is None or carry[1] == carry[2]):   # a gzip text that ended with the previous piece
                self.free.put(i)
                if carry is not None:
                    self.free.put(carry[0])
                return
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
        if self._gz is not None:
            self._gz.close()
        self._f.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class _GzText:
    """The text of a gzip file, piece by piece, for _RawChunks' reader thread.  BGZF members are inflated on the GPU (Gunzip, on its own
    stream, so this overlaps the parse and split of the previous chunk): compressed bytes are read into a pinned buffer, the whole members
    that fit the piece are inflated straight into it, and a partial member stays for the next read.  From the first member that is not BGZF
    on (plain `gzip`, concatenated members, or a later part of a mixed file), zlib inflates the rest of the file, member after member;
    with bgzf_only (BAM) such a member is an error."""

    def __init__(self, f, piece, device, bgzf_only=False):
        self.f, self.piece, self.device, self.bgzf_only = f, piece, device, bgzf_only
        self.zcap = piece + (1 << 17)                                  # a piece of text in members, and the partial member after them
        self._zt, self.z = _pinned(self.zcap)
        self.zlen, self.eof = 0, False
        self.gz = None                                                  # the GPU inflater, created with the first BGZF member
        self.blocks = None                                              # zlib's text blocks, from the first member that is not BGZF on
        self.pending, self.pending_off = b"", 0

    def _read_more(self):
        if not self.eof and self.zlen < self.zcap:
            n = self.f.readinto(memoryview(self.z)[self.zlen:])
            self.eof = n < self.zcap - self.zlen
            self.zlen += n

    def _bgzf_next(self):
        try:
            bgzf_scan(self.z[:self.zlen], 0, max_members=1)
            return True
        except KmcB200Error:
            return False

    def fill(self, out):
        """Text into out[0, n); returns (n, final).  n > 0 unless final."""
        n = 0
        while self.blocks is None:
            self._read_more()
            if self.zlen == 0:
                return n, True
            if not self._bgzf_next():
                if self.bgzf_only:
                    raise _bam_error("a member is not BGZF")
                rest = bytes(self.z[:self.zlen])
                self.zlen = 0
                self.blocks = _zlib_members(rest, lambda: self.f.read(_ZLIB_READ))
                break
            if self.gz is None:
                if self.piece < BGZF_MAX_TEXT:
                    raise KmcB200Error(ERR_INVALID, "BGZF input needs pieces of at least 64 KiB of text: batch_bytes of at least %d" %
                                       (2 * BGZF_MAX_TEXT + 2))
                self.gz = Gunzip(self.device, self.zcap, self.piece)
            used, t = self.gz.inflate(self.z[:self.zlen], out[n:])
            n += t
            if used:
                self.z[:self.zlen - used] = self.z[used:self.zlen]
                self.zlen -= used
            if self.eof and self.zlen == 0:
                return n, True
            if used == 0:
                if n:
                    return n, False                                     # the next member does not fit this piece
                raise _gzip_error("the last BGZF member is truncated")
        while n < out.size:                                             # zlib
            if self.pending_off == len(self.pending):
                self.pending, self.pending_off = next(self.blocks, None), 0
                if self.pending is None:
                    return n, True
            take = min(out.size - n, len(self.pending) - self.pending_off)
            out[n:n + take] = np.frombuffer(self.pending, dtype=np.uint8, count=take, offset=self.pending_off)
            n += take
            self.pending_off += take
        return n, False

    def close(self):
        if self.gz is not None:
            self.gz.close()


class _Parsers:
    """One FastxParser per format met, created on first use."""

    def __init__(self, device, max_chunk_bytes):
        self.device, self.max_chunk_bytes, self.by_format = device, max_chunk_bytes, {}

    def __call__(self, chunk, fmt=None):
        """The parser of `fmt`, by default FASTQ or FASTA as the chunk's text says."""
        fmt = fmt or fastx_format(chunk)
        if fmt not in self.by_format:
            self.by_format[fmt] = FastxParser(fmt, self.device, self.max_chunk_bytes)
        return self.by_format[fmt]

    def close(self):
        for p in self.by_format.values():
            p.close()
        self.by_format = {}


def signature_sample_counts(paths, k, signature_len, batch_bytes=1 << 26, device=0, parse="host", homopolymer_compressed=False):
    """Stage 0's statistics (CKMC::buildSignatureMapping, kmc_core/kmc.h:974-1075): k-mers per signature, counted on the GPU, over the
    text of the files in input order up to the end of the first record at or beyond max(2^28, predicted_size / 100) text bytes (a gzip
    file counts 3.2 times its bytes in the prediction, its text in the sample; a BAM file 0.7 times its bytes, its record bytes).  BAM
    records are counted as stored: a k-mer's signature is the same on either strand, so -b's reverse complement changes no count.
    parse="gpu": the files are parsed on the GPU in chunks of batch_bytes - 1, the sample's end found by the parser's limit.
    homopolymer_compressed: the k-mers of the compressed reads are counted (`kmc -hc`); the sample's end is still found on the raw bytes."""
    budget = max(STATS_SAMPLE_BYTES, predicted_size(paths) // 100)
    st = SignatureStats(k, signature_len, device, max_batch_bytes=batch_bytes, homopolymer_compressed=homopolymer_compressed)
    if parse == "gpu":
        parsers = _Parsers(device, batch_bytes - 1)
        try:
            for path in paths:
                if budget <= 0:
                    break
                cut, pos = is_gzip(path) or os.path.getsize(path) > budget, 0     # a gzip text's size is known once it is read
                with _RawChunks(path, batch_bytes - 1, device) as chunks:
                    parser = None
                    for chunk, final in chunks:
                        parser = parser or parsers(chunk, BAM if chunks.bam else None)
                        limit = budget - pos if cut else None
                        used = st.add_fastx(parser, chunk, final, limit)
                        chunks.consumed(used)
                        pos += used
                        if cut and pos >= budget:
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
        data, bam = _read_input(path)
        if not len(data):
            continue
        if len(data) > budget:
            data = data[:(bam_record_end if bam else _record_end)(data, budget - 1)]
        budget -= len(data)
        for batch in batches(_to_batch(data, bam), batch_bytes):
            st.add(batch)
    counts = st.read()
    st.close()
    return counts


SMALL_K_MAX = 13
ESTIMATE_MAX_K = 256
ESTIMATE_LARGE_INPUT = 50_000_000_000                                   # kmc.h:1118-1121: s = 11 from this many input bytes on


def estimate_s(paths):
    """The reference's sampling exponent for these inputs: 7, or 11 when their predicted size (predicted_size: gzip files count 3.2 times
    their bytes, BAM files 0.7 times) is at least 5 * 10^10 bytes."""
    return 11 if predicted_size(paths) >= ESTIMATE_LARGE_INPUT else 7


def n_records(data):
    """FASTQ records or FASTA headers in a chunk of whole records: the reads CSplitter::GetSeq counts (splitter.cpp:68-417)."""
    a = _as_array(data)
    if a.size == 0:
        return 0
    starts = np.concatenate([[0], np.flatnonzero(a[:-1] == _NL) + 1])
    if fastx_format(a) == FASTA:
        return int(np.count_nonzero(a[starts] == _GT))
    return (int(np.count_nonzero(a[starts] != _NL)) + 3) // 4


def _as_array(data):
    return np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.asarray(data, dtype=np.uint8)


def kmc_lut_prefix_len(k, n_est_kmers, n_bins):
    """The LUT prefix length `kmc` picks for a bin database (kmc.h:1432-1468): lp of 2..15 with (k - lp) % 4 == 0 (uint32 arithmetic)
    of least n_est * (k - lp) / 4 + n_bins * 4^lp * 8 (uint64), the first on a tie.  n_est is 4 * n_reads, or with --opt-out-size the
    estimated number of counted k-mers."""
    m64 = (1 << 64) - 1
    best, best_mem = 0, 1 << 62
    for lp in range(2, 16):
        suffix = (k - lp) & 0xFFFFFFFF
        if suffix % 4:
            continue
        mem = (((n_est_kmers * suffix) & m64) // 4 + n_bins * (1 << (2 * lp)) * 8) & m64
        if mem < best_mem:
            best, best_mem = lp, mem
    return best


def estimated_counted_kmers(hist, cutoff_min, cutoff_max):
    """kmc.h:1441-1447: the estimate summed over cutoff_min .. min(cutoff_max + 1, len) - 1."""
    end = min(int(cutoff_max) + 1, len(hist))
    return int(sum(int(v) for v in hist[int(cutoff_min):end])) & ((1 << 64) - 1)


def estimate_histogram(paths, k, s=None, batch_bytes=1 << 26, device=0, parse="host"):
    """`kmc -e` on one GPU: the reference's ntHash estimate of the k-mer count histogram of the files (canonical k-mers, 1 <= k <= 256),
    uint64[max_occ + 1] with entry 0 = 0.  s: 7 or 11, default the reference's rule on the input size (estimate_s).  parse as for
    count_reads."""
    if parse not in ("host", "gpu"):
        raise KmcB200Error(ERR_INVALID, "parse must be 'host' or 'gpu', not %r" % (parse,))
    est = HistogramEstimator(k, estimate_s(paths) if s is None else s, device, max_batch_bytes=batch_bytes)
    if _kmc_inputs(paths):
        try:
            for _, dec, recs, first, batch in _kmc_chunks(paths, batch_bytes, device, parse):
                if dec is None:
                    est.add(batch)
                else:
                    est.add_kmcdb(dec, recs, first)
            return est.histogram()
        finally:
            est.close()
    parsers = _Parsers(device, batch_bytes - 1) if parse == "gpu" else None
    try:
        for path in paths:
            if parsers is not None:
                with _RawChunks(path, batch_bytes - 1, device) as chunks:
                    parser = None
                    for chunk, final in chunks:
                        parser = parser or parsers(chunk, BAM if chunks.bam else None)   # canonical hashes: either strand
                        chunks.consumed(est.add_fastx(parser, chunk, final))
                continue
            data, bam = _read_input(path)
            if not len(data):
                continue
            for batch in batches(_to_batch(data, bam), batch_bytes):
                est.add(batch)
        return est.histogram()
    finally:
        if parsers is not None:
            parsers.close()
        est.close()


def write_histogram(path, hist):
    """The file `kmc -e` writes (kmc_CLI/kmc.cpp:308-321): "i\tcount\n" for i = 1 .. len - 1."""
    with open(path, "w") as f:
        f.write("".join("%d\t%d\n" % (i, int(v)) for i, v in enumerate(hist) if i))


def count_reads_small_k(paths, out_prefix, k, cutoff_min=2, cutoff_max=1_000_000_000, counter_max=255, both_strands=True, batch_bytes=1 << 26,
                        device=0, parse="host", homopolymer_compressed=False):
    """KMC's small-k mode (kmc_core/kmc.h:677-960) on one GPU, for 1 <= k <= 13: every batch of every file is counted into 4^k counters
    (kmc_b200.SmallKCounter), then the KMC1 database is written (CSmallKCompleter::CompleteKMCFormat).  There are no bins: no signature
    length, no map, and the LUT prefix length is the reference's choice for this mode, returned as `lut_prefix_len`.  parse as for
    count_reads.  homopolymer_compressed: `kmc -hc` (see the module docstring).  Returns the keys count_reads returns (n_super_kmers is 0,
    n_kmers equals n_total) plus lut_prefix_len."""
    if parse not in ("host", "gpu"):
        raise KmcB200Error(ERR_INVALID, "parse must be 'host' or 'gpu', not %r" % (parse,))
    if not 1 <= k <= SMALL_K_MAX:
        raise KmcB200Error(ERR_INVALID, "the small-k path counts k = 1..%d, not %d" % (SMALL_K_MAX, k))
    t0 = time.perf_counter()
    sk = SmallKCounter(k, both_strands, device, max_batch_bytes=batch_bytes, homopolymer_compressed=homopolymer_compressed)
    n_bases = 0
    read_s = 0.0
    kmc_input = _kmc_inputs(paths)
    parsers = _Parsers(device, batch_bytes - 1) if parse == "gpu" and not kmc_input else None
    try:
        for _, dec, recs, first, batch in _kmc_chunks(paths, batch_bytes, device, parse) if kmc_input else ():
            if dec is None:
                sk.add(batch)
                n_bases += batch.size
            else:
                sk.add_kmcdb(dec, recs, first)
                n_bases += sk.last_seq_bytes
        for path in paths if not kmc_input else ():
            if parsers is not None:
                with _RawChunks(path, batch_bytes - 1, device) as chunks:
                    parser = None
                    for chunk, final in chunks:
                        parser = parser or parsers(chunk, (BAM if both_strands else BAM_ORIGINAL_STRAND) if chunks.bam else None)
                        chunks.consumed(sk.add_fastx(parser, chunk, final))
                        n_bases += sk.last_seq_bytes
                read_s += chunks.wait_s
                continue
            t = time.perf_counter()
            data, bam = _read_input(path)
            read_s += time.perf_counter() - t
            seq = _to_batch(data, bam, not both_strands)
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


def count_reads(paths, out_prefix, k, signature_len, signature_map, lut_prefix_len=None, cutoff_min=2, cutoff_max=1_000_000_000, counter_max=255,
                both_strands=True, batch_bytes=1 << 26, device=0, n_bins=None, parse="host", small_k=None, opt_out_size=False,
                homopolymer_compressed=False):
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
    used, and the result also holds the lut_prefix_len the path chose.
    lut_prefix_len=None picks it as `kmc` does (kmc_lut_prefix_len): from 4 * n_reads, the records of the input (FASTQ records, FASTA
    headers), or with opt_out_size=True from the estimate of the counted k-mers, which the histogram estimator (HistogramEstimator, s by
    estimate_s) computes over the same batches as the split, as `kmc --opt-out-size` does.  opt_out_size needs canonical k-mers and the
    bin path.  The result holds n_reads and the lut_prefix_len used.
    homopolymer_compressed=True counts the k-mers of the homopolymer-compressed reads, as `kmc -hc` does: stage 0, the split and the
    small-k path compress every batch on the GPU; the estimator and n_reads see the reads as they are (see the module docstring)."""
    if parse not in ("host", "gpu"):
        raise KmcB200Error(ERR_INVALID, "parse must be 'host' or 'gpu', not %r" % (parse,))
    if opt_out_size and not both_strands:
        raise KmcB200Error(ERR_INVALID, "k-mer histogram estimation possible only for canonical k-mers")
    if opt_out_size and lut_prefix_len is not None:
        raise KmcB200Error(ERR_INVALID, "opt_out_size chooses the LUT prefix length: give lut_prefix_len=None")
    if small_k or (small_k is None and k <= signature_len):
        if opt_out_size:
            raise KmcB200Error(ERR_INVALID, "histogram estimation is not supported on the small-k path, as in kmc")
        return count_reads_small_k(paths, out_prefix, k, cutoff_min, cutoff_max, counter_max, both_strands, batch_bytes, device, parse,
                                   homopolymer_compressed)
    t0 = time.perf_counter()
    kmc_input = _kmc_inputs(paths)
    if kmc_input:                                                       # stage 0 is skipped: the map comes from the first database
        if signature_map is not None:
            raise KmcB200Error(ERR_INVALID, "KMC database input takes its signature map from the first database: give signature_map=None")
        mapper, n_bins = kmc_input_signature_map(paths[0], signature_len, n_bins)
        sig_map = mapper.astype(np.uint32)
    elif signature_map is None:
        n_bins = DEFAULT_N_BINS if n_bins is None else int(n_bins)
        mapper = _signature_map(signature_sample_counts(paths, k, signature_len, batch_bytes, device, parse, homopolymer_compressed),
                                signature_len, n_bins)
        sig_map = np.maximum(mapper, 0).astype(np.uint32)              # no k-mer has a signature that is not allowed
    else:
        mapper = None
        sig_map = np.ascontiguousarray(signature_map, dtype=np.uint32)
        n_bins = int(sig_map.max()) + 1 if n_bins is None else int(n_bins)
    t_stats = time.perf_counter() - t0
    # the splitter first: the stage-2 context sizes its block limit from the HBM that is free when it is created
    sp = Splitter(k, signature_len, sig_map, n_bins, device, max_batch_bytes=batch_bytes, homopolymer_compressed=homopolymer_compressed)
    if mapper is not None:
        sp.count_kxmers(both_strands)
    est = HistogramEstimator(k, estimate_s(paths), device, max_batch_bytes=batch_bytes) if opt_out_size else None
    parts = [[] for _ in range(n_bins)]
    n_super = n_kmers = n_bases = n_reads = 0
    read_s = 0.0

    def keep(out, packs, frags):
        nonlocal n_super, n_kmers
        for b, fr in enumerate(frags):
            if fr.bytes:
                parts[b].append((out[fr.byte_off:fr.byte_off + fr.bytes].copy(), packs[fr.pack0:fr.pack0 + fr.n_packs].copy(), int(fr.n_rec)))
                n_super += int(fr.n_super_kmers)
                n_kmers += int(fr.n_rec)

    parsers = _Parsers(device, batch_bytes - 1) if parse == "gpu" and not kmc_input else None
    try:
        for info, dec, recs, first, batch in _kmc_chunks(paths, batch_bytes, device, parse) if kmc_input else ():
            if dec is None:
                out, packs, frags = sp.split_raw(batch)
                nseq, kept = batch.size, batch.size // (info.kmer_len + 1)
                if est is not None:
                    est.add(batch)
            else:
                out, packs, frags, nseq, kept = sp.split_kmcdb(dec, recs, first)
                if est is not None:
                    est.add_kmcdb(dec, recs, first)
            n_reads += kept
            n_bases += nseq
            keep(out, packs, frags)
        for path in paths if not kmc_input else ():
            if parsers is not None:
                with _RawChunks(path, batch_bytes - 1, device) as chunks:
                    parser = None
                    for chunk, final in chunks:
                        parser = parser or parsers(chunk, (BAM if both_strands else BAM_ORIGINAL_STRAND) if chunks.bam else None)
                        out, packs, frags, used, nseq = sp.split_fastx(parser, chunk, final)
                        if est is not None:
                            est.add_fastx(parser, chunk[:used], True)
                            n_reads += est.last_records
                        elif chunks.bam:
                            n_reads += parser.last_records()
                        else:
                            n_reads += n_records(chunk[:used])
                        chunks.consumed(used)
                        n_bases += nseq
                        keep(out, packs, frags)
                read_s += chunks.wait_s
                continue
            t = time.perf_counter()
            data, bam = _read_input(path)
            read_s += time.perf_counter() - t
            n_reads += bam_n_reads(data) if bam else n_records(data)
            seq = _to_batch(data, bam, not both_strands)
            del data
            for batch in batches(seq, batch_bytes):
                out, packs, frags = sp.split_raw(batch)
                if est is not None:
                    est.add(batch)
                n_bases += batch.size
                keep(out, packs, frags)
        if lut_prefix_len is None:
            n_est = estimated_counted_kmers(est.histogram(), cutoff_min, cutoff_max) if est is not None else 4 * n_reads
            lut_prefix_len = kmc_lut_prefix_len(k, n_est, n_bins)
    finally:
        if parsers is not None:
            parsers.close()
        if est is not None:                                             # before the stage-2 context sizes itself from free HBM
            est.close()
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
            "n_kmers": n_kmers, "n_bases": n_bases, "stats_s": t_stats, "split_s": t1 - t0 - t_stats, "stage2_s": t2 - t1, "read_s": read_s,
            "n_reads": n_reads, "lut_prefix_len": lut_prefix_len}


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m kmc_b200.reads", description=__doc__.split("\n\n")[0])
    ap.add_argument("inputs", nargs="+", help="FASTQ / FASTA / BAM files or KMC database prefixes, then the output prefix")
    ap.add_argument("-k", type=int, default=25)
    ap.add_argument("-p", "--signature-len", type=int, default=9)
    ap.add_argument("-n", "--n-bins", type=int, default=None, help="bins when the map is chosen from the reads (default %d, KMC's -n)" % DEFAULT_N_BINS)
    ap.add_argument("--map", help=".npy file with the 4^p + 1 map entries (default: chosen from the reads, as KMC does)")
    ap.add_argument("--map-from", help="take p and the map from this .kmc_pre")
    ap.add_argument("--lut-prefix-len", type=int, default=None, help="default: the smallest of 7, 3, 11, ... with (k - p) %% 4 == 0")
    ap.add_argument("--opt-out-size", action="store_true",
                    help="pick the LUT prefix length from the estimated number of counted k-mers, as kmc --opt-out-size does")
    ap.add_argument("-e", action="store_true", help="write the estimated k-mer count histogram to the last argument instead of counting (kmc -e)")
    ap.add_argument("--ci", type=int, default=2)
    ap.add_argument("--cx", type=int, default=1_000_000_000)
    ap.add_argument("--cs", type=int, default=255)
    ap.add_argument("-b", action="store_true", help="count k-mers as they are, not canonical ones")
    ap.add_argument("--hc", action="store_true", help="count homopolymer-compressed k-mers, as kmc -hc does (-e ignores it, as kmc does)")
    ap.add_argument("--batch-bytes", type=int, default=1 << 26)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--gpu-parse", action="store_true", help="parse FASTQ / FASTA on the GPU in chunks of batch-bytes - 1 (default: numpy, whole files)")
    ap.add_argument("--small-k", action="store_true",
                    help="k <= 13: count in 4^k direct counters and write a KMC1 database, as kmc does (taken without the flag when k <= p)")
    a = ap.parse_args(argv)
    if len(a.inputs) < 2:
        ap.error("give at least one input and the output prefix")
    parse = "gpu" if a.gpu_parse else "host"
    if a.e:
        if a.b:
            ap.error("k-mer histogram estimation possible only for canonical k-mers")
        if not 1 <= a.k <= ESTIMATE_MAX_K:
            ap.error("-e takes k = 1..%d" % ESTIMATE_MAX_K)
        write_histogram(a.inputs[-1], estimate_histogram(a.inputs[:-1], a.k, None, a.batch_bytes, a.device, parse))
        return 0
    if a.opt_out_size and a.lut_prefix_len is not None:
        ap.error("--opt-out-size picks the LUT prefix length: it cannot be combined with --lut-prefix-len")
    if a.map_from:
        m, sig_map = signature_map_from_kmc_pre(a.map_from)
    elif a.map:
        m, sig_map = a.signature_len, np.load(a.map)
    else:
        m, sig_map = a.signature_len, None
    if a.small_k or a.k <= m:                                           # no bins: no map, and the path picks its own LUT prefix length
        if a.opt_out_size:
            ap.error("histogram estimation is not supported on the small-k path, as in kmc")
        print(json.dumps(count_reads_small_k(a.inputs[:-1], a.inputs[-1], a.k, a.ci, a.cx, a.cs, not a.b, a.batch_bytes, a.device, parse, a.hc)))
        return 0
    lp = a.lut_prefix_len
    if lp is None and not a.opt_out_size and not _kmc_inputs(a.inputs[:-1]):     # KMC input: kmc's rule (from 4 * n_reads)
        lp = next(p for p in (7, 3, 11, 15, 4, 5, 6, 2, 8, 9, 10, 12, 13, 14, 1) if p < a.k and (a.k - p) % 4 == 0)
    res = count_reads(a.inputs[:-1], a.inputs[-1], a.k, m, sig_map, lp, a.ci, a.cx, a.cs, not a.b, a.batch_bytes, a.device,
                      a.n_bins if sig_map is None else None, parse=parse, small_k=False, opt_out_size=a.opt_out_size, homopolymer_compressed=a.hc)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
