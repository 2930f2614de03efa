"""Seam inputs for the batch kernels (TEST INFRASTRUCTURE): batches and reads texts that put a chosen event on the positions where a kernel
divides its work (tiles, warps, thread spans, scan CTAs, record tiles, expander packs), and a numpy model of the super-k-mer rule that says
where every run and record of such a batch starts and ends, so that each case can check it hit what it aims at.

Events: a separator or 'N'; a lower-case switch; a homopolymer run edge; the start and end of a signature run.  A run of a chosen signature
comes from a planted m-mer: in a background of C and G only, every m-mer and its reverse complement starts with C or G, so an allowed m-mer
'A' + (C|G)^(m-1) is smaller than every other m-mer a k-mer around it can hold.  The k-mers that contain it form one run of exactly
w = k - m + 1 k-mers that starts k - m bases before it.  Poly-A segments between 'N's give runs of the special signature 4^m of any length."""
import numpy as np

# where the kernels divide their work (kmc_b200/csrc/split.cuh, small_k.cuh, estimate.cuh, fastx.cuh, hc.cuh)
THREAD = 16                                 # k-mer positions per thread of the position kernels
WARP = 32 * THREAD
TILE = 4096                                 # positions per CTA of stage 0, stage 1, small k and the estimator
SCAN_BLOCK = 4096                           # elements per CTA of the device scans: tile values of 2^24 positions
REC_TILE = 8192                             # records per tile of the bin histogram and the rank kernel
PACK_WINDOW = 65536 - 128                   # a record at offset s of a bin is in expander pack s / PACK_WINDOW
FASTX_SPAN = 64                             # bytes per thread of the parser and of homopolymer compression
FASTX_TILE = 256 * FASTX_SPAN               # 16 KiB

CODE = np.full(256, 4, dtype=np.uint8)
for _i, _c in enumerate(b"ACGT"):
    CODE[_c] = CODE[_c + 32] = _i
ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
CG = np.frombuffer(b"CG", dtype=np.uint8)


def tiled(n, alphabet, seed, block=1 << 16):
    """n bytes drawn from `alphabet`: a seeded block tiled, so that large batches cost no Python loop."""
    rng = np.random.default_rng(seed)
    a = np.frombuffer(alphabet, dtype=np.uint8) if isinstance(alphabet, bytes) else np.asarray(alphabet, dtype=np.uint8)
    blk = a[rng.integers(0, a.size, min(block, max(n, 1)))]
    return np.tile(blk, n // blk.size + 1)[:n].copy()


def offsets(j):
    """-1, 0, +1 in turn: the offset from the seam of the j-th event"""
    return j % 3 - 1


class SeamBatch:
    """A batch (uint8 array) with events planted at chosen positions; `events` keeps (kind, position) of each for the target checks."""

    def __init__(self, n, seed, alphabet=b"CG"):
        self.a = tiled(n, alphabet, seed)
        self.rng = np.random.default_rng(seed + 1)
        self.events = []

    def __len__(self):
        return self.a.size

    def tobytes(self):
        return self.a.tobytes()

    def sep(self, pos, byte=b"N"):
        """a separator (any byte other than ACGTacgt) at pos"""
        self.a[pos] = byte[0]
        self.events.append(("sep", pos))

    def lower(self, lo, hi):
        """bases [lo, hi) in lower case: a switch at lo and one at hi"""
        self.a[lo:hi] |= np.where(CODE[self.a[lo:hi]] < 4, 0x20, 0).astype(np.uint8)
        self.events.append(("lower", lo))

    def homopolymer(self, lo, hi, base=b"A"):
        """a run of one base over [lo, hi), its neighbours made different from it so the run starts at lo and ends at hi - 1"""
        self.a[lo:hi] = base[0]
        others = ACGT[ACGT != base[0]]
        for p in (lo - 1, hi):
            if 0 <= p < self.a.size and CODE[self.a[p]] == CODE[base[0]]:
                self.a[p] = others[self.rng.integers(0, 3)]
        self.events.append(("homopolymer", lo))

    def plant_run(self, t, k, m):
        """the run of w = k - m + 1 k-mers at t .. t + w - 1 with one signature: 'A' + (C|G)^(m-1) at base t + k - m (C/G background only).
        Returns the planted m-mer's value."""
        p = t + k - m
        mm = np.concatenate([[ord("A")], CG[self.rng.integers(0, 2, m - 1)]]).astype(np.uint8)
        self.a[p:p + m] = mm
        self.events.append(("run", t))
        return int(sum(int(CODE[c]) << (2 * (m - 1 - i)) for i, c in enumerate(mm)))

    def poly_a(self, t, n_kmers, k):
        """a run of n_kmers k-mers of the special signature at t .. t + n_kmers - 1: 'N', poly-A of n_kmers + k - 1 bases, 'N'"""
        lo, hi = t, t + n_kmers + k - 1
        self.a[lo:hi] = ord("A")
        for p in (lo - 1, hi):
            if 0 <= p < self.a.size:
                self.a[p] = ord("N")
        self.events.append(("poly_a", t))


def seam_anchors(n, step, margin=0):
    """(j, anchor) for every multiple of `step` in [margin, n - margin)"""
    return [(j, a) for j, a in enumerate(range(0, n, step)) if margin <= a < n - margin]


# ----------------------------------------------------------------------------- the super-k-mer rule in numpy
def norm_table(m):
    """norm(x) of every m-mer value (the stage-1 oracle's table: min of the allowed orientations, 4^m when neither is)"""
    from stage1_testlib import Stage1Oracle
    return Stage1Oracle().norm_table(m)


def kmer_signatures(batch, k, m, norm):
    """int64 per k-mer start position t (0 .. len - k): the least norm of its m-mers, -1 when it holds a non-ACGT byte"""
    a = np.asarray(np.frombuffer(batch, dtype=np.uint8) if isinstance(batch, (bytes, bytearray)) else batch, dtype=np.uint8)
    c = CODE[a]
    n = a.size - k + 1
    if n <= 0:
        return np.zeros(0, dtype=np.int64)
    nm = a.size - m + 1
    x = np.zeros(nm, dtype=np.int64)
    for q in range(m):
        x = (x << 2) | (c[q:q + nm] & 3).astype(np.int64)
    cur = np.asarray(norm, dtype=np.int64)[x]
    w, span = k - m + 1, 1
    while 2 * span <= w:
        cur = np.minimum(cur[:-span], cur[span:])
        span *= 2
    sig = np.minimum(cur[:n], cur[w - span:w - span + n])
    bad = np.concatenate([[0], np.cumsum(c > 3)])
    return np.where(bad[k:k + n] - bad[:n] == 0, sig, -1)


def runs(sig):
    """(starts, ends) of the maximal runs of one valid signature"""
    valid = sig >= 0
    prev = np.concatenate([[-2], sig[:-1]])
    nxt = np.concatenate([sig[1:], [-2]])
    return np.flatnonzero(valid & (sig != prev)), np.flatnonzero(valid & (sig != nxt))


def super_kmers(sig):
    """(starts, ends) of the records: runs cut every 256 k-mers counted from the run's start"""
    t = np.arange(sig.size)
    valid = sig >= 0
    start = valid & (sig != np.concatenate([[-2], sig[:-1]]))
    rs = np.maximum.accumulate(np.where(start, t, -1))
    rec = valid & ((t - rs) % 256 == 0)
    nxt_rec = np.concatenate([rec[1:], [True]])
    nxt_valid = np.concatenate([valid[1:], [False]])
    return np.flatnonzero(rec), np.flatnonzero(valid & (~nxt_valid | nxt_rec))


def record_bytes(starts, ends, k):
    return 1 + (ends - starts + k + 3) // 4


# ----------------------------------------------------------------------------- records of chosen sizes (one bin)
def poly_a_segment(nbytes, k):
    """poly-A bases that make exactly one record of `nbytes` bytes (1 + k/4 .. 97 at k = 128): n symbols with 1 + ceil(n / 4) = nbytes"""
    n = max(k, 4 * nbytes - 5)
    assert k <= n <= k + 255 and 1 + (n + 3) // 4 == nbytes, (nbytes, k)
    return b"A" * n


def sizes_to(total, lo, hi=97):
    """record sizes in [lo, hi] that add up to `total` (0 or at least lo)"""
    if total == 0:
        return []
    q = -(-total // hi)
    assert total >= q * lo, (total, lo)
    return [total // q + (1 if i < total % q else 0) for i in range(q)]


def records_batch(sizes, k):
    """one poly-A segment per record size, each ended by 'N'"""
    return b"".join(poly_a_segment(s, k) + b"N" for s in sizes)


# ----------------------------------------------------------------------------- reads text with line ends on chosen bytes
def text_with_line_ends(fmt, targets, n_bytes, seed):
    """FASTQ or FASTA text of about n_bytes whose lines end where `targets` say: a list of (kind, pos) with kind 'lf' ('\\n' at pos),
    'crlf' ('\\r' at pos - 1 and '\\n' at pos) or, FASTA only, 'hdr' (a header line starting at pos, so '\\n' at pos - 1, '>' at pos).
    Line contents are random; FASTQ lines cycle header / sequence / '+' / quality, FASTA lines are headers now and then.
    Returns the text and the targets it placed (a target closer than 3 bytes to the previous line end is dropped)."""
    rng = np.random.default_rng(seed)
    out = bytearray()
    placed = []
    line = 0
    pending = sorted(targets, key=lambda x: x[1])
    qual = np.arange(33, 75, dtype=np.uint8)

    def content(n, kind):
        if kind == "hdr":
            return b">" + bytes(qual[rng.integers(0, qual.size, n - 1)]) if n > 1 else b">"
        if kind == "seq":
            return ACGT[rng.integers(0, 4, n)].tobytes()
        if kind == "qual":
            return qual[rng.integers(0, qual.size, n)].tobytes()
        return (b"@" if kind == "at" else b"+") + b"r" * (n - 1)

    def kind_of(i, header):
        if fmt == "fastq":
            return ("at", "seq", "plus", "qual")[i % 4]
        return "hdr" if header else "seq"

    while len(out) < n_bytes or pending:
        cur = len(out)
        header = fmt == "fasta" and (line == 0 or rng.random() < 0.1)
        if pending and pending[0][1] - cur < 3:
            pending.pop(0)                                                  # too close to place: drop it
            continue
        if pending and pending[0][1] - cur <= 300:
            kind, pos = pending.pop(0)
            cr = kind == "crlf"
            if kind == "hdr":
                # the line before ends at pos - 1, the header starts at pos
                ln = pos - 1 - cur
                out += content(ln, kind_of(line, header)) + b"\n"
                line += 1
                out += content(int(rng.integers(2, 40)), "hdr" if fmt == "fasta" else kind_of(line, False)) + b"\n"
                line += 1
                placed.append((kind, pos))
                continue
            ln = pos - cur - (1 if cr else 0)
            out += content(ln, kind_of(line, header)) + (b"\r\n" if cr else b"\n")
            line += 1
            placed.append((kind, pos))
            continue
        ln = int(rng.integers(1, 200))
        if pending:
            ln = min(ln, pending[0][1] - cur - 4)
        out += content(max(ln, 1), kind_of(line, header)) + b"\n"
        line += 1
    if fmt == "fastq":
        while line % 4:
            out += content(5, kind_of(line, False)) + b"\n"
            line += 1
    return bytes(out), placed


def check_line_ends(text, placed):
    """every placed target is where it was asked to be"""
    for kind, pos in placed:
        if kind == "lf":
            assert text[pos] == 10, (kind, pos)
        elif kind == "crlf":
            assert text[pos - 1:pos + 1] == b"\r\n", (kind, pos)
        else:
            assert text[pos - 1] == 10 and text[pos] == ord(">"), (kind, pos)


# ----------------------------------------------------------------------------- k-mers the estimator samples
def sampled_kmers(k, s, count, seed, max_tries=200_000):
    """up to `count` seeded random k-mers (bytes) that the estimator oracle samples on their own"""
    from estimate_testlib import oracle_increments
    rng = np.random.default_rng(seed)
    found = []
    for _ in range(max_tries):
        if len(found) == count:
            break
        km = ACGT[rng.integers(0, 4, k)].tobytes()
        if oracle_increments(km, k, s).size:
            found.append(km)
    return found
