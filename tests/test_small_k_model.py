"""A numpy model of KMC's small-k mode (k <= 13): the counts (CSplitter::ProcessReadsSmallK, kmc_core/splitter.cpp:681-805), the LUT prefix
length (kmc.h:906-936) and the KMC1 files (CSmallKCompleter::CompleteKMCFormat, kb_completer.h:148-308).  It is pinned here, with no GPU,
against a brute-force count and against what the unmodified reference CLI wrote (tests/golden/small_k_reference.json, made by
tests/golden/make_small_k_reference.py); tests/test_gpu_small_k.py then holds the GPU to it."""
import hashlib
import json
import os
import struct

import numpy as np
import pytest

from kmc_b200.reads import sequences_to_batch
from kmc_testlib import reference_digest
from test_gpu_kmc_files import write_fastq
from test_reference_cli import brute_force, dump_digest, small_fastq

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "small_k_reference.json")
_CODE = np.full(256, 4, dtype=np.uint8)
for _i, _c in enumerate(b"ACGT"):
    _CODE[_c] = _CODE[_c + 32] = _i


# ------------------------------------------------------------------------------------------------ the model
def kmer_values(batch, k, both_strands=True):
    """uint64 values of every k-mer of ACGT only in a batch (every other byte separates), in batch order."""
    c = _CODE[np.asarray(batch, dtype=np.uint8)]
    n = c.size - k + 1
    if n <= 0:
        return np.zeros(0, dtype=np.uint64)
    bad = np.concatenate([[0], np.cumsum(c > 3)])
    ok = bad[k:] - bad[:n] == 0
    s = (c & 3).astype(np.uint64)
    fw = np.zeros(n, dtype=np.uint64)
    rc = np.zeros(n, dtype=np.uint64)
    for j in range(k):
        fw |= s[j:j + n] << np.uint64(2 * (k - 1 - j))
        rc |= (np.uint64(3) - s[j:j + n]) << np.uint64(2 * j)
    v = np.minimum(fw, rc) if both_strands else fw
    return v[ok]


def counts(batch, k, both_strands=True):
    return np.bincount(kmer_values(batch, k, both_strands).astype(np.int64), minlength=1 << (2 * k)).astype(np.uint64)


def _byte_log(v, top):
    n = 1
    while n < top and v >= 1 << (8 * n):
        n += 1
    return n


def counter_size(cutoff_max, counter_max, ull=True):
    """calc_counter_size_ull (records) or calc_counter_size (the LUT prefix length's cost), defs.h:154-166."""
    if counter_max == 1:
        return 0
    return min(_byte_log(cutoff_max, 8 if ull else 4), _byte_log(counter_max, 8 if ull else 4))


def lut_prefix_len(k, n_unique, cutoff_max, counter_max):
    cs = counter_size(cutoff_max, counter_max, ull=False)
    best, best_mem = 0, 1 << 62
    for lp in range(1, 16):
        suffix_len = 0 if lp > k else k - lp
        if suffix_len % 4:
            continue
        mem = n_unique * (suffix_len // 4 + cs) + (1 << (2 * lp)) * 8
        if mem < best_mem:
            best, best_mem = lp, mem
    return best


def finish(cnt, k, cutoff_min, cutoff_max, counter_max):
    """(lut_prefix_len, counter_size, records, lut, (n_unique, n_cutoff_min, n_cutoff_max, n_total))."""
    cnt = np.asarray(cnt, dtype=np.uint64)
    present = cnt > 0
    below = present & (cnt < cutoff_min)
    above = present & ~below & (cnt > np.uint64(cutoff_max))
    kept = np.flatnonzero(present & ~below & ~above)
    stats = (int(present.sum()), int(below.sum()), int(above.sum()), int(cnt.sum(dtype=np.uint64)))
    lp = lut_prefix_len(k, stats[0], cutoff_max, counter_max)
    cs = counter_size(cutoff_max, counter_max)
    sb = (k - lp) // 4
    vals = kept.astype(np.uint64)
    c = np.minimum(cnt[kept], np.uint64(counter_max))
    cols = [(vals >> np.uint64(8 * (sb - 1 - j))) & np.uint64(255) for j in range(sb)] + [(c >> np.uint64(8 * j)) & np.uint64(255) for j in range(cs)]
    recs = np.stack(cols, axis=1).astype(np.uint8).reshape(-1) if cols else np.zeros(0, dtype=np.uint8)
    lut = np.searchsorted(kept, np.arange(1 << (2 * lp), dtype=np.int64) << (2 * (k - lp))).astype(np.uint64)
    return lp, cs, recs, lut, stats


def database(cnt, k, both_strands, cutoff_min, cutoff_max, counter_max):
    """(.kmc_pre bytes, .kmc_suf bytes, stats, lut_prefix_len) of the KMC1 database of the counts."""
    lp, cs, recs, lut, stats = finish(cnt, k, cutoff_min, cutoff_max, counter_max)
    footer = struct.pack("<IIIIIIQB3xI20xI", k, 0, cs, lp, cutoff_min, cutoff_max & 0xFFFFFFFF, stats[0] - stats[1] - stats[2],
                         0 if both_strands else 1, cutoff_max >> 32, 0)
    pre = b"KMCP" + lut.tobytes() + footer + struct.pack("<I", len(footer)) + b"KMCP"
    return pre, b"KMCS" + recs.tobytes() + b"KMCS", stats, lp


def md5(b):
    return hashlib.md5(b).hexdigest()


# ------------------------------------------------------------------------------------------------ the reference cases
_LETTERS = np.frombuffer(b"ACGTN", dtype=np.uint8)


def _low_complexity_fastq(path, seed):
    rng = np.random.default_rng(seed)
    units = [b"A", b"T", b"AC", b"GT", b"CAG", b"ACGT", b"AAAAC"]
    with open(path, "wb") as f:
        for i in range(300):
            u = units[i % len(units)]
            n = int(rng.integers(20, 400))
            s = (u * (n // len(u) + 1))[:n]
            if i % 3 == 0:
                s = s[:n // 2] + _LETTERS[rng.integers(0, 4, 7)].tobytes() + s[n // 2:]
            f.write(b"@r%d\n%s\n+\n%s\n" % (i, s, b"I" * len(s)))


def _fasta(path, seed):
    rng = np.random.default_rng(seed)
    with open(path, "wb") as f:
        for i in range(400):
            s = _LETTERS[rng.choice(5, int(rng.integers(1, 300)), p=[0.24, 0.24, 0.24, 0.24, 0.04])].tobytes()
            f.write(b">seq%d some header ACGT\n%s\n" % (i, s))


def _palindromes(path, _seed):
    kat = next(kt for kt in json.load(open(os.path.join(os.path.dirname(GOLDEN), "kats.json"))) if kt["k"] == 5)
    with open(path, "w") as f:
        for j, r in enumerate(kat["reads"]):
            f.write(">r%d\n%s\n" % (j, r))


INPUTS = {
    "reads": (lambda p, s: write_fastq(p, s, 2000, genome_len=50_000), "-fq"),
    "ndense": (lambda p, s: write_fastq(p, s, 500, genome_len=20_000, n_frac=0.15), "-fq"),
    "lowcx": (_low_complexity_fastq, "-fq"),
    "fasta": (_fasta, "-fa"),
    "palindromes": (_palindromes, "-fa"),
}

# (name, input, seed, k, both_strands, cutoff_min, cutoff_max, counter_max)
CASES = [("k%d_%s" % (k, "both" if both else "b"), "reads", 40 + k, k, both, 2, 1_000_000_000, 255)
         for k in (1, 2, 3, 4, 5, 7, 8, 9, 10, 11, 12, 13) for both in (True, False)] + [
    ("k9_ci1", "reads", 7, 9, True, 1, 1_000_000_000, 255),
    ("k7_ci3_cx40", "reads", 8, 7, True, 3, 40, 255),
    ("k11_ci2_cx3", "reads", 9, 11, False, 2, 3, 255),
    ("k8_cs1", "reads", 10, 8, True, 1, 1_000_000_000, 1),
    ("k3_cs1", "reads", 11, 3, True, 1, 1_000_000_000, 1),
    ("k6_cs300", "reads", 12, 6, True, 2, 1_000_000_000, 300),
    ("k5_cx2pow33", "reads", 13, 5, True, 1, 1 << 33, 1 << 33),
    ("k4_cx2pow33_cs255", "reads", 14, 4, False, 2, (1 << 33) + 5, 255),
    ("k10_ndense", "ndense", 15, 10, True, 1, 1_000_000_000, 255),
    ("k13_ndense", "ndense", 16, 13, True, 2, 1_000_000_000, 255),
    ("k5_lowcx", "lowcx", 17, 5, True, 1, 1_000_000_000, 255),
    ("k12_lowcx_b", "lowcx", 18, 12, False, 1, 1_000_000_000, 65535),
    ("k7_fasta", "fasta", 19, 7, True, 1, 1_000_000_000, 255),
    ("k5_palindromes", "palindromes", 0, 5, True, 1, 1_000_000_000, 255),
]


def kmc_args(case):
    name, inp, seed, k, both, cmin, cmax, cntmax = case
    return ["-k%d" % k, INPUTS[inp][1], "-ci%d" % cmin, "-cx%d" % cmax, "-cs%d" % cntmax] + ([] if both else ["-b"])


def write_input(case, path):
    INPUTS[case[1]][0](path, case[2])


def golden():
    return json.load(open(GOLDEN))


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 7, 9, 13])
@pytest.mark.parametrize("both", [True, False])
def test_model_counts_equal_brute_force(tmp_path, k, both):
    fq = os.path.join(str(tmp_path), "reads.fq")
    write_fastq(fq, 100 + k, 300, genome_len=5000, n_frac=0.02)
    cnt = counts(sequences_to_batch(open(fq, "rb").read()), k, both)
    exp = brute_force(fq, k, both)
    nz = np.flatnonzero(cnt)
    got = {"".join("ACGT"[(int(v) >> (2 * (k - 1 - j))) & 3] for j in range(k)): int(cnt[v]) for v in nz}
    assert got == exp


def test_model_reproduces_the_stored_k13_dump(tmp_path):
    """cli_fastq_k13 in reference_digests.json: what `kmc -k13 -ci2 -cs255` counted in test_reference_cli's FASTQ, as a sorted dump."""
    fq = os.path.join(str(tmp_path), "reads.fq")
    small_fastq(fq)
    ref = reference_digest("cli_fastq_k13")
    cnt = counts(sequences_to_batch(open(fq, "rb").read()), 13)
    lp, cs, recs, lut, stats = finish(cnt, 13, 2, 255, 255)
    kept = np.flatnonzero((cnt >= 2))
    dump = {"".join("ACGT"[(int(v) >> (2 * (12 - j))) & 3] for j in range(13)): min(int(cnt[v]), 255) for v in kept}
    assert dump_digest(dump) == ref["results"]["dump"]
    assert ref["results"]["unique_counted_kmers"] == len(kept)


def test_lut_prefix_len_rule():
    assert [lut_prefix_len(k, 0, 255, 255) for k in (1, 2, 3, 4, 5, 9, 13)] == [1, 2, 3, 4, 1, 1, 1]
    assert lut_prefix_len(3, 10 ** 6, 255, 255) == 3                    # k <= 3: the prefix is the whole k-mer
    assert lut_prefix_len(13, 4 ** 13, 255, 255) == 9                   # every k-mer present: 1 suffix byte and a 4^9 LUT are cheapest
    assert lut_prefix_len(8, 1000, 255, 1) == 4
    assert counter_size(1 << 33, 1 << 33) == 5 and counter_size(1 << 33, 1 << 33, ull=False) == 4 and counter_size(10, 1) == 0


def test_golden_cases_are_the_declared_ones():
    g = golden()
    assert sorted(g) == sorted(c[0] for c in CASES)
    for c in CASES:
        assert g[c[0]]["args"] == kmc_args(c)
        assert g[c[0]]["version"] == 0, "the reference did not take its small-k path"


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_model_database_equals_the_reference(tmp_path, case):
    name, inp, seed, k, both, cmin, cmax, cntmax = case
    path = os.path.join(str(tmp_path), "input")
    write_input(case, path)
    ref = golden()[name]
    data = open(path, "rb").read()
    assert md5(data) == ref["input_md5"], "the generated input is not the one the reference counted"
    pre, suf, stats, lp = database(counts(sequences_to_batch(data), k, both), k, both, cmin, cmax, cntmax)
    assert lp == ref["lut_prefix_len"] and stats[3] == ref["n_total"]
    assert [stats[0], stats[1], stats[2], stats[0] - stats[1] - stats[2]] == [ref["n_unique"], ref["n_cutoff_min"], ref["n_cutoff_max"],
                                                                             ref["n_counted"]]
    assert md5(pre) == ref["kmc_pre_md5"] and md5(suf) == ref["kmc_suf_md5"]
