"""Helpers for the stage-1 tests (TEST INFRASTRUCTURE): the sequential C oracle of KMC's splitter (oracle/stage1_oracle.c), seeded read
generators, and brute-force checks of a split straight from the definition."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGE1_SRC = os.path.join(ROOT, "oracle", "stage1_oracle.c")
STAGE1_SO = os.path.join(ROOT, "oracle", "_build", "libkmc_stage1_oracle.so")
PACK_WINDOW = 65536 - 128
STAGE1_GOLDEN = os.path.join(ROOT, "tests", "golden", "stage1_reference.json")


def ensure_stage1_oracle_built():
    if (not os.path.exists(STAGE1_SO)) or os.path.getmtime(STAGE1_SO) < max(os.path.getmtime(STAGE1_SRC), os.path.getmtime(STAGE1_SRC[:-1] + "h")):
        os.makedirs(os.path.dirname(STAGE1_SO), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-o", STAGE1_SO, STAGE1_SRC])
    return STAGE1_SO


class Split:
    """One batch split into bins: out (bins concatenated in bin order), pack_bytes, frags[n_bins, 6] =
    byte_off, bytes, n_rec, n_super_kmers, pack0, n_packs."""

    def __init__(self, out, pack_bytes, frags, k):
        self.out, self.pack_bytes, self.frags, self.k = out, pack_bytes, frags, k

    def bin_data(self, b):
        f = self.frags[b]
        return self.out[int(f[0]):int(f[0] + f[1])]

    def bin_packs(self, b):
        f = self.frags[b]
        return self.pack_bytes[int(f[4]):int(f[4] + f[5])]

    @property
    def n_bins(self):
        return self.frags.shape[0]

    def to_bin(self, b):
        """bin b as a kmc_testlib.Bin (what the stage-2 oracle and Stage2Context take)."""
        from kmc_testlib import Bin
        f = self.frags[b]
        pb = self.bin_packs(b).astype(np.uint64)
        return Bin(data=np.ascontiguousarray(self.bin_data(b)), n_rec=int(f[2]), n_super_kmers=int(f[3]), pack_bytes=pb, pack_recs=pb, k=self.k)


def concat_splits(splits):
    """Batches -> one Split: per bin, the fragments in batch order (streams and pack lists concatenated)."""
    n_bins, k = splits[0].n_bins, splits[0].k
    outs, packs, frags = [], [], np.zeros((n_bins, 6), dtype=np.uint64)
    off = npk = 0
    for b in range(n_bins):
        d = [s.bin_data(b) for s in splits]
        p = [s.bin_packs(b) for s in splits]
        nb, np_ = sum(x.size for x in d), sum(x.size for x in p)
        frags[b] = (off, nb, sum(int(s.frags[b][2]) for s in splits), sum(int(s.frags[b][3]) for s in splits), npk, np_)
        outs += d
        packs += p
        off += nb
        npk += np_
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)
    return Split(cat(outs, np.uint8), cat(packs, np.uint64), frags, k)


class Stage1Oracle:
    def __init__(self):
        self.lib = C.CDLL(ensure_stage1_oracle_built())
        self.lib.kmcs_split.restype = C.c_int
        self.lib.kmcs_split.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                        C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p]
        self.lib.kmcs_norm_table.restype = None
        self.lib.kmcs_norm_table.argtypes = [C.c_uint32, C.c_void_p]

    def norm_table(self, m):
        t = np.zeros(1 << (2 * m), dtype=np.uint32)
        self.lib.kmcs_norm_table(m, t.ctypes.data)
        return t

    def split(self, batch, k, m, sig_map, n_bins=None) -> Split:
        seq = np.ascontiguousarray(np.frombuffer(batch, dtype=np.uint8) if isinstance(batch, (bytes, bytearray)) else batch, dtype=np.uint8)
        sig_map = np.ascontiguousarray(sig_map, dtype=np.uint32)
        n_bins = int(sig_map.max()) + 1 if n_bins is None else n_bins
        prm = (C.c_uint32 * 3)(k, m, n_bins)
        frags = np.zeros((n_bins, 6), dtype=np.uint64)
        nb, npk = C.c_uint64(0), C.c_uint64(0)
        rc = self.lib.kmcs_split(prm, sig_map.ctypes.data, seq.ctypes.data, seq.size, None, 0, C.byref(nb), None, 0, C.byref(npk), frags.ctypes.data)
        if rc == 0:
            return Split(np.zeros(0, np.uint8), np.zeros(0, np.uint64), frags, k)
        assert rc == -5, rc
        out = np.zeros(nb.value, dtype=np.uint8)
        packs = np.zeros(npk.value, dtype=np.uint64)
        rc = self.lib.kmcs_split(prm, sig_map.ctypes.data, seq.ctypes.data, seq.size, out.ctypes.data, out.size, C.byref(nb),
                                 packs.ctypes.data, packs.size, C.byref(npk), frags.ctypes.data)
        assert rc == 0, rc
        return Split(out, packs, frags, k)

    def signature_counts(self, batch, k, m):
        """k-mers per signature (CSplitter::CalcStats, splitter.cpp:439-530): the split with the identity map, n_bins = 4^m + 1."""
        ident = np.arange((1 << (2 * m)) + 1, dtype=np.uint32)
        return self.split(batch, k, m, ident).frags[:, 2].astype(np.int64)


# ----------------------------------------------------------------------------- maps
def random_map(seed, m, n_bins):
    """A map as CSignatureMapper would hand it to the splitter: every entry < n_bins, the special signature in the last bin."""
    rng = np.random.default_rng(seed)
    mp = rng.integers(0, max(n_bins - 1, 1), (1 << (2 * m)) + 1).astype(np.uint32)
    mp[-1] = n_bins - 1
    return mp


def greedy_map(counts, n_bins):
    """Signatures grouped greedily onto n_bins - 1 bins by their k-mer counts (heaviest first, each onto the lightest bin), the special
    signature alone in the last bin."""
    import heapq
    m_size = counts.size
    mp = np.zeros(m_size, dtype=np.uint32)
    heap = [(0, b) for b in range(n_bins - 1)]
    for s in np.argsort(-counts[:-1], kind="stable"):
        load, b = heapq.heappop(heap)
        mp[s] = b
        heapq.heappush(heap, (load + int(counts[s]) + 1, b))
    mp[-1] = n_bins - 1
    return mp


# ----------------------------------------------------------------------------- reads
LETTERS = np.frombuffer(b"ACGT", dtype=np.uint8)


def make_reads(seed, profile, n_reads=200, read_len=150, genome_len=100_000):
    """Seeded reads as a list of bytes.  Profiles: 'short' / 'long' (noisy samples of a random genome, both strands), 'n_dense'
    (N and IUPAC bytes every ~20 bases, some lowercase), 'low_complexity' (poly-A, poly-T and tandem repeats of several hundred bases
    between random stretches: runs of far more than 256 k-mers, the special signature's bin fills)."""
    rng = np.random.default_rng(seed)
    genome = rng.integers(0, 4, max(genome_len, read_len + 1), dtype=np.uint8)
    comp = np.array([3, 2, 1, 0], dtype=np.uint8)
    reads = []
    for i in range(n_reads):
        if profile == "low_complexity":
            parts = []
            for _ in range(max(1, read_len // 400)):
                kind = rng.integers(0, 4)
                n = int(rng.integers(100, 700))
                if kind == 0:
                    parts.append(b"A" * n)
                elif kind == 1:
                    parts.append(b"T" * n)
                elif kind == 2:
                    unit = LETTERS[rng.integers(0, 4, int(rng.integers(2, 7)))].tobytes()
                    parts.append((unit * (n // len(unit) + 1))[:n])
                else:
                    parts.append(LETTERS[rng.integers(0, 4, n)].tobytes())
            reads.append(b"".join(parts)[:max(read_len, 1)])
            continue
        p = int(rng.integers(0, genome.size - read_len + 1))
        r = genome[p:p + read_len].copy()
        if rng.integers(0, 2):
            r = comp[r[::-1]]
        err = rng.random(read_len) < 0.01
        r = np.where(err, (r + rng.integers(1, 4, read_len)) % 4, r).astype(np.uint8)
        s = LETTERS[r].copy()
        if profile == "n_dense":
            bad = rng.random(read_len) < 0.05
            s[bad] = np.frombuffer(b"NRYKMSWnx.", dtype=np.uint8)[rng.integers(0, 10, int(bad.sum()))]
            low = rng.random(read_len) < 0.1
            s[low & ~bad] += 32
        reads.append(s.tobytes())
    return reads


def batch_of(reads, sep=b"\n"):
    return sep.join(reads)


def write_fastq_reads(path, reads):
    with open(path, "wb") as f:
        for i, r in enumerate(reads):
            f.write(b"@r%d\n%s\n+\n%s\n" % (i, r, b"I" * len(r)))


def write_fasta_reads(path, reads, line=60):
    with open(path, "wb") as f:
        for i, r in enumerate(reads):
            f.write(b">r%d\n" % i + b"\n".join(r[j:j + line] for j in range(0, max(len(r), 1), line)) + b"\n")


# ----------------------------------------------------------------------------- brute force from the definition
def records(data, k):
    """A bin's stream -> list of (n_extra, symbols uint8 array)."""
    d = np.asarray(data, dtype=np.uint8)
    out, pos = [], 0
    while pos < d.size:
        a = int(d[pos])
        n = k + a
        nb = (n + 3) // 4
        b = d[pos + 1:pos + 1 + nb]
        sym = np.stack([(b >> 6) & 3, (b >> 4) & 3, (b >> 2) & 3, b & 3], axis=1).reshape(-1)[:n]
        out.append((a, sym.astype(np.uint8)))
        pos += 1 + nb
    assert pos == d.size
    return out


def kmer_signature(sym, m, norm):
    """signature of the k-mer given by its symbols: the least normalised value of its m-mers"""
    w = 0
    best = None
    mask = (1 << (2 * m)) - 1
    for i, s in enumerate(sym):
        w = ((w << 2) | int(s)) & mask
        if i >= m - 1:
            v = int(norm[w])
            best = v if best is None else min(best, v)
    return best


def expected_kmer_bins(batch, k, m, sig_map, norm):
    """{bin: sorted list of k-mer strings} straight from the definition: every ACGT-only k-mer goes to map[min norm m-mer]."""
    codes = {ord(c): i for i, c in enumerate("ACGT")}
    codes.update({ord(c): i for i, c in enumerate("acgt")})
    res = {}
    seq = bytes(batch)
    i = 0
    n = len(seq)
    while i < n:
        j = i
        while j < n and seq[j] in codes:
            j += 1
        seg = seq[i:j]
        if len(seg) >= k:
            sym = np.array([codes[c] for c in seg], dtype=np.uint8)
            mask = (1 << (2 * m)) - 1
            vals = np.zeros(len(seg) - m + 1, dtype=np.int64)
            w = 0
            for q in range(len(seg)):
                w = ((w << 2) | int(sym[q])) & mask
                if q >= m - 1:
                    vals[q - m + 1] = norm[w]
            for t in range(len(seg) - k + 1):
                b = int(sig_map[int(vals[t:t + k - m + 1].min())])
                res.setdefault(b, []).append("".join("ACGT"[x] for x in sym[t:t + k]))
        i = j + 1
    return {b: sorted(v) for b, v in res.items()}


# ----------------------------------------------------------------------------- stored reference cases (tests/golden/make_stage1_reference.py)
STAGE1_MAPS = os.path.join(ROOT, "tests", "golden", "stage1_maps.npz")
# name: (seed, read profile, n_reads, read_len, k, reference CLI options); the reference runs with -sr1 -n64
STAGE1_CASES = {
    "k17_p5_canon": (101, "short", 3000, 150, 17, ("-p5", "-ci1")),
    "k31_p7_b": (102, "short", 3000, 150, 31, ("-p7", "-ci1", "-b")),
    "k31_p9_lowcomplex": (103, "low_complexity", 300, 1500, 31, ("-p9", "-ci1")),
    "k55_p9_ndense_b": (104, "n_dense", 2000, 200, 55, ("-p9", "-ci1", "-b")),
    "k96_p7_canon": (105, "short", 2000, 250, 96, ("-p7", "-ci1", "-cs65535")),
    "k17_p7_ndense": (106, "n_dense", 3000, 150, 17, ("-p7", "-ci2")),
}


def case_reads(case):
    seed, profile, n_reads, read_len = STAGE1_CASES[case][:4]
    return make_reads(seed, profile, n_reads=n_reads, read_len=read_len, genome_len=50_000)


def load_map(case):
    return np.load(STAGE1_MAPS)[case].astype(np.uint32)


def kmc_pre_bins(pre_path, suf_path):
    """A KMC database split per file bin: header fields, map, and per bin (payload bytes, raw LUT counts)."""
    pre = open(pre_path, "rb").read()
    suf = open(suf_path, "rb").read()
    import struct
    header_offset = struct.unpack("<I", pre[-8:-4])[0]
    h = len(pre) - 8 - header_offset
    k, mode, counter_size, p, sig_len, cmin, cmax = struct.unpack("<7I", pre[h:h + 28])
    both = pre[h + 36] == 0
    n_map = (1 << (2 * sig_len)) + 1
    m0 = h - 4 * n_map
    sig_map = np.frombuffer(pre[m0:h], dtype=np.uint32)
    n_recs, = struct.unpack("<Q", pre[m0 - 8:m0])
    luts = np.frombuffer(pre[4:m0 - 8], dtype=np.uint64).reshape(-1, 1 << (2 * p))
    rec = (k - p) // 4 + counter_size
    flat = np.append(luts.reshape(-1), np.uint64(n_recs)).astype(np.int64)
    raw = np.diff(flat).reshape(luts.shape).astype(np.uint64)
    starts = np.append(luts[:, 0], np.uint64(n_recs)).astype(np.int64)
    payloads = [suf[4 + int(starts[b]) * rec:4 + int(starts[b + 1]) * rec] for b in range(luts.shape[0])]
    header = dict(k=k, counter_size=counter_size, p=p, sig_len=sig_len, cmin=cmin, cmax=cmax, both=bool(both))
    return header, sig_map, payloads, raw
