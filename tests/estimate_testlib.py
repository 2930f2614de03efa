"""Helpers for the histogram-estimator tests (TEST INFRASTRUCTURE): the C restatement of KMC's CntHashEstimator (oracle/estimate_oracle.c),
the reference's own estimator where build() compiled it (oracle/ref/nthash_harness.cpp), the seeded inputs of the stored reference cases
(tests/golden/estimate_reference.json) and the `kmc -e` text format."""
import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SRC = os.path.join(ROOT, "oracle", "estimate_oracle.c")
ORACLE_SO = os.path.join(ROOT, "oracle", "_build", "libkmc_estimate_oracle.so")
HARNESS_SO = os.path.join(ROOT, "oracle", "_ref", "libkmc_nthash_ref.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "estimate_reference.json")
TABLE = 1 << 27
MAX_OCC = 65536
_lib = None


def ensure_estimate_oracle_built():
    if (not os.path.exists(ORACLE_SO)) or os.path.getmtime(ORACLE_SO) < os.path.getmtime(ORACLE_SRC):
        os.makedirs(os.path.dirname(ORACLE_SO), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-o", ORACLE_SO, ORACLE_SRC, "-lm"])
    return ORACLE_SO


def _oracle():
    global _lib
    if _lib is None:
        lib = C.CDLL(ensure_estimate_oracle_built())
        lib.est_oracle_increments.restype = C.c_uint64
        lib.est_oracle_increments.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64]
        lib.est_oracle_histogram.restype = None
        lib.est_oracle_histogram.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        _lib = lib
    return _lib


def _u8(batch):
    return np.ascontiguousarray(np.frombuffer(batch, dtype=np.uint8) if isinstance(batch, (bytes, bytearray)) else batch, dtype=np.uint8)


def oracle_increments(batch, k, s):
    """uint64 counter indices (table * 2^27 + index) the oracle's Process increments, one per sampled hash."""
    seq = _u8(batch)
    lib = _oracle()
    n = lib.est_oracle_increments(seq.ctypes.data, seq.size, k, s, None, 0)
    out = np.zeros(max(int(n), 1), dtype=np.uint64)
    lib.est_oracle_increments(seq.ctypes.data, seq.size, k, s, out.ctypes.data, out.size)
    return out[:n]


class SparseCounters:
    """The two counter tables as (index, value) of their non-zero counters, from increments."""

    def __init__(self, increments):
        self.index, self.value = np.unique(np.asarray(increments, dtype=np.uint64), return_counts=True)
        self.value = self.value.astype(np.uint32)

    @classmethod
    def from_dense(cls, counters):
        c = cls(np.zeros(0, dtype=np.uint64))
        nz = np.flatnonzero(counters)
        c.index, c.value = nz.astype(np.uint64), np.asarray(counters)[nz].astype(np.uint32)
        return c

    def value_histograms(self):
        """(hist0, hist1, max): the two tables' histograms of min(65536, counter), bins 0..65536, and the largest counter."""
        hists = []
        for t in range(2):
            sel = (self.index >> np.uint64(27)) == t
            h = np.bincount(np.minimum(self.value[sel], MAX_OCC), minlength=MAX_OCC + 1).astype(np.uint32)
            h[0] = TABLE - int(sel.sum())
            hists.append(h)
        return hists[0], hists[1], int(self.value.max()) if self.value.size else 0


def oracle_recursion(h0, h1, mx, s):
    """EstimateHistogram (the oracle's restatement) from the two value histograms: uint64[max_occ + 1]."""
    max_occ = min(max(mx, 2), MAX_OCC)
    a = np.ascontiguousarray(h0[:max_occ + 1], dtype=np.uint32)
    b = np.ascontiguousarray(h1[:max_occ + 1], dtype=np.uint32)
    out = np.zeros(max_occ + 1, dtype=np.uint64)
    _oracle().est_oracle_histogram(a.ctypes.data, b.ctypes.data, max_occ, s, out.ctypes.data)
    return out


def oracle_histogram(batch, k, s):
    """The estimate of one batch by the oracle: uint64[max_occ + 1], entry 0 is 0."""
    h0, h1, mx = SparseCounters(oracle_increments(batch, k, s)).value_histograms()
    return oracle_recursion(h0, h1, mx, s)


def have_harness():
    return os.path.exists(HARNESS_SO)


def harness_histogram(batch, k, s):
    """The reference's own CntHashEstimator fed the batch's records (oracle/ref/nthash_harness.cpp)."""
    lib = C.CDLL(HARNESS_SO)
    lib.nthash_ref_histogram.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
    seq = _u8(batch)
    out = np.zeros(MAX_OCC + 1, dtype=np.uint64)
    n = C.c_uint64(0)
    assert lib.nthash_ref_histogram(seq.ctypes.data, seq.size, k, s, out.ctypes.data, out.size, C.byref(n)) == 0
    return out[:n.value]


def hist_text(hist):
    """The file `kmc -e` writes (kmc_CLI/kmc.cpp:308-321): "i\\tvalue\\n" for i = 1..len - 1."""
    return "".join("%d\t%d\n" % (i, int(v)) for i, v in enumerate(hist) if i).encode()


def md5(data):
    return hashlib.md5(data).hexdigest()


# ---- the seeded inputs of the stored cases ---------------------------------------------------------------------------------------------

def make_reads(seed, n_reads, read_len, genome_len=300_000, err=0.01, n_frac=0.002, lower_frac=0.0):
    """Reads sampled from a random genome (both strands), with substitution errors, N's and optionally lower-case bases."""
    rng = np.random.default_rng(seed)
    genome = rng.integers(0, 4, genome_len, dtype=np.uint8)
    acgt, comp = np.frombuffer(b"ACGT", dtype=np.uint8), np.frombuffer(b"TGCA", dtype=np.uint8)
    reads = []
    for _ in range(n_reads):
        ln = int(read_len) if np.isscalar(read_len) else int(rng.integers(read_len[0], read_len[1] + 1))
        p = int(rng.integers(0, genome_len - ln))
        r = genome[p:p + ln].copy()
        e = rng.random(ln) < err
        r[e] = rng.integers(0, 4, int(e.sum()))
        txt = (comp[r[::-1]] if rng.random() < 0.5 else acgt[r]).copy()
        txt[rng.random(ln) < n_frac] = ord("N")
        if lower_frac:
            low = (rng.random(ln) < lower_frac) & (txt != ord("N"))
            txt[low] += 32
        reads.append(txt.tobytes())
    return reads


def fastq_text(reads):
    return b"".join(b"@r%d\n%s\n+\n%s\n" % (i, r, b"I" * len(r)) for i, r in enumerate(reads))


def fasta_multiline_text(reads, width=60):
    out = []
    for i, r in enumerate(reads):
        out.append(b">r%d\n" % i)
        out.extend(r[j:j + width] + b"\n" for j in range(0, len(r), width))
    return b"".join(out)


def case_reads(case):
    """The reads of a stored case from its parameters."""
    g = case["gen"]
    kind = g["kind"]
    if kind == "reads":
        rl = g["read_len"] if isinstance(g["read_len"], int) else tuple(g["read_len"])
        return make_reads(g["seed"], g["n_reads"], rl, g.get("genome_len", 300_000), g.get("err", 0.01), g.get("n_frac", 0.002),
                          g.get("lower_frac", 0.0))
    if kind == "empty":
        return []
    if kind == "repeat":                                                # one k-mer as many reads of its own
        return [g["kmer"].encode()] * g["copies"] + make_reads(g["seed"], g["n_reads"], g["read_len"])
    raise ValueError(kind)


def case_text(case):
    reads = case_reads(case)
    return fasta_multiline_text(reads) if case["format"] == "fasta" else fastq_text(reads)


def case_batch(case):
    """The batch (kmcb200_split's format) of a case's reads: every read followed by a newline."""
    return b"".join(r + b"\n" for r in case_reads(case))


def load_golden():
    with open(GOLDEN) as f:
        return json.load(f)
