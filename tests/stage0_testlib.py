"""Helpers for the stage-0 tests (TEST INFRASTRUCTURE): the C restatement of KMC's signature statistics and of the collector's (k+x)-mer
count (oracle/stage0_oracle.c), and straight Python restatements to check it against."""
import ctypes as C
import os
import subprocess

import numpy as np

from stage1_testlib import ROOT, Split

STAGE0_SRC = [os.path.join(ROOT, "oracle", "stage0_oracle.c"), os.path.join(ROOT, "oracle", "stage1_oracle.c")]
STAGE0_SO = os.path.join(ROOT, "oracle", "_build", "libkmc_stage0_oracle.so")
_lib = None


def ensure_stage0_oracle_built():
    deps = STAGE0_SRC + [s[:-1] + "h" for s in STAGE0_SRC]
    if (not os.path.exists(STAGE0_SO)) or os.path.getmtime(STAGE0_SO) < max(os.path.getmtime(d) for d in deps):
        os.makedirs(os.path.dirname(STAGE0_SO), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-o", STAGE0_SO] + STAGE0_SRC)
    return STAGE0_SO


def _stage0_lib():
    global _lib
    if _lib is not None:
        return _lib
    lib = C.CDLL(ensure_stage0_oracle_built())
    lib.kmcs_signature_stats.restype = C.c_int
    lib.kmcs_signature_stats.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
    lib.kmcs_kxmer_count.restype = C.c_uint64
    lib.kmcs_kxmer_count.argtypes = [C.c_uint32, C.c_int, C.c_void_p, C.c_uint64]
    _lib = lib
    return lib


def oracle_signature_stats(batch, k, m):
    """k-mers per signature by the oracle's literal restatement of CSplitter::CalcStats: uint32[4^m + 1]."""
    seq = np.ascontiguousarray(np.frombuffer(batch, dtype=np.uint8) if isinstance(batch, (bytes, bytearray)) else batch, dtype=np.uint8)
    stats = np.zeros((1 << (2 * m)) + 1, dtype=np.uint32)
    rc = _stage0_lib().kmcs_signature_stats(k, m, seq.ctypes.data, seq.size, stats.ctypes.data)
    assert rc == 0, rc
    return stats


def oracle_kxmer_totals(split: Split, both_strands):
    """Per bin of a split: the collector's n_plus_x_recs over the bin's records (uint64[n_bins])."""
    lib = _stage0_lib()
    out = np.zeros(split.n_bins, dtype=np.uint64)
    for b in range(split.n_bins):
        d = np.ascontiguousarray(split.bin_data(b))
        out[b] = lib.kmcs_kxmer_count(split.k, int(bool(both_strands)), d.ctypes.data, d.size)
    return out


def max_x_of(k):
    """kmc.h:139-142: the x of the (k+x)-mers stage 2 sorts"""
    return min(31 - k % 32, 3) if k % 32 else 0


def kxmer_count_restated(sym, k, both_strands):
    """update_n_plus_x_recs (kb_collector.h:66-116) / the plain-k-mer rule for one record given by its symbols, straight from the source."""
    max_x = max_x_of(k)
    if not max_x:
        return 0
    n = len(sym)
    if not both_strands:
        return 1 + (n - k) // (max_x + 1)
    s = [int(v) for v in sym]
    kmer = ((s[0] << 6) + (s[1] << 4) + (s[2] << 2) + s[3]) & 0xFF
    rev = (((3 - s[k - 1]) << 6) + ((3 - s[k - 2]) << 4) + ((3 - s[k - 3]) << 2) + (3 - s[k - 4])) & 0xFF
    state = lambda a, b: "kmer" if a < b else ("rev" if b < a else "eq")
    cur, x, total = state(kmer, rev), 0, 0
    for i in range(n - k):
        rev = ((rev >> 2) + ((3 - s[k + i]) << 6)) & 0xFF
        kmer = ((kmer << 2) + s[4 + i]) & 0xFF
        new = state(kmer, rev)
        if new == cur:
            if cur == "eq":
                total += 1
            else:
                x += 1
        else:
            cur = new
            total += 1 + x // (max_x + 1)
            x = 0
    return total + 1 + x // (max_x + 1)


def file_position_map(mapper, file_pos):
    """A .kmc_pre map from the mapper's bin ids and the bins' file positions: the completer stores 0 for signatures without a bin."""
    mapper = np.asarray(mapper, dtype=np.int64)
    return np.where(mapper < 0, 0, np.asarray(file_pos, dtype=np.int64)[np.maximum(mapper, 0)]).astype(np.uint32)
