"""CPU: the oracle against what the unmodified reference classes computed on the same bins (oracle/_ref, built from a KMC
source tree by oracle/Makefile).  The reference's results are stored as digests in tests/golden/reference_digests.json
(tests/golden/make_reference_digests.py regenerates them from the case builders below), so the tests need no reference build."""
import numpy as np
import pytest

from kmc_testlib import Params, synth_bin, pack_superkmers, choose_lut_prefix_len, bin_digest, result_digest, reference_digest

BIN_CASES = [(31, True, 2), (31, False, 1), (28, True, 1), (28, False, 2), (55, True, 2), (55, False, 1),
             (17, True, 1), (32, True, 2), (64, True, 1), (70, True, 2), (33, True, 1), (128, True, 1)]
# how each case was run through the reference: RADULS with one sorter, radix.h + CSmallSort (non-Intel hosts, kmc.h:1556-1560),
# RADULS with in-bin threads (packs with gaps, kxmer_set.h:299-314)
REF_VARIANTS = {"raduls": dict(), "radix_h": dict(sort_kind=1), "raduls_4_sorters": dict(n_sorters=4)}
CUTOFF_CASES = [(1, 10 ** 9, 255), (3, 9, 4), (2, 300, 65535), (1, 10 ** 9, 1)]
SORT_CASES = [(1, 8), (1, 5), (2, 14), (2, 15), (3, 18), (4, 32)]
SEVERAL_SIZES = [400, 0, 2500, 30, 1200]
# corners of the record and counter layout: k = 65 / 97 (the first k of 3- and 4-word records: the top symbols sit in the low bits of a
# fresh word), 4-byte counters with a count in the third byte, counter_max = 1 with wide records, cutoff_max setting the counter width, and
# p = 15 (a 4^15-entry LUT, with a small bin).  name: (k, both_strands, cutoff_min, cutoff_max, counter_max, lut_prefix_len, copies of one k-mer)
CORNER_CASES = {"corner_k65_cs4": (65, True, 1, 10 ** 9, 2 ** 32 - 1, 5, 70000), "corner_k97_cs3": (97, False, 2, 10 ** 9, 2 ** 24 - 1, 5, 0),
                "corner_k55_cs1": (55, True, 1, 10 ** 9, 1, 7, 0), "corner_k31_cs4_cx200": (31, True, 1, 200, 2 ** 32 - 1, 7, 300),
                "corner_k127_p15": (127, True, 1, 10 ** 9, 65535, 15, 0)}


def bin_case(k, both, cmin):
    p = Params(k=k, both_strands=both, cutoff_min=cmin, lut_prefix_len=choose_lut_prefix_len(k))
    return p, synth_bin(k + cmin, k, 2500, genome_len=3000, err=0.02)


def cutoff_case(cmin, cmax, cntmax):
    p = Params(k=31, cutoff_min=cmin, cutoff_max=cmax, counter_max=cntmax, lut_prefix_len=7)
    return p, synth_bin(cmin * 7 + cmax % 13, 31, 3000, genome_len=500, err=0.005)


def edge_bins():
    rng = np.random.default_rng(1)
    return [pack_superkmers(31, [rng.integers(0, 4, 31)]),
            pack_superkmers(31, [rng.integers(0, 4, 31 + 255) for _ in range(40)]),
            pack_superkmers(31, [np.zeros(31 + 255, dtype=np.uint8) for _ in range(30)]),
            pack_superkmers(31, [np.tile(np.array([0, 3], dtype=np.uint8), 100)[:31 + 150] for _ in range(20)])]


def corner_case(case):
    k, both, cmin, cmax, cntmax, p_len, copies = CORNER_CASES[case]
    rng = np.random.default_rng(900 + k + copies)
    genome = rng.integers(0, 4, 640 + k)
    starts, lens = rng.integers(0, 600, 1500), k + rng.integers(0, 40, 1500)
    lists = [genome[s:s + n] for s, n in zip(starts, lens)] + [genome[:k]] * copies
    return Params(k=k, both_strands=both, cutoff_min=cmin, cutoff_max=cmax, counter_max=cntmax, lut_prefix_len=p_len), pack_superkmers(k, lists)


def several_bins():
    return [synth_bin(50 + i, 31, n, genome_len=max(n, 400)) for i, n in enumerate(SEVERAL_SIZES)]


def sort_case(words, key_bytes):
    rng = np.random.default_rng(words * 100 + key_bytes)
    n = 20000
    raw = rng.integers(0, 256, size=(n, words * 8), dtype=np.uint8)
    raw[:, key_bytes:] = 0
    raw[n // 2:] = raw[rng.integers(0, n // 2, n - n // 2)]
    return raw.view(np.uint64).reshape(n, words)


def _check(oracle_result, case, b):
    exp = reference_digest(case)
    assert bin_digest(b) == exp["input"], "%s: the generated input is not the one the reference result was stored for" % case
    got = result_digest(oracle_result)
    for variant, r in exp["results"].items():
        assert got == r, "%s: oracle != reference (%s)" % (case, variant)


@pytest.mark.parametrize("k,both,cmin", BIN_CASES)
def test_bin_matches_reference(oracle, k, both, cmin):
    p, b = bin_case(k, both, cmin)
    _check(oracle.process_bin(b, p), "bin_k%d_both%d_ci%d" % (k, both, cmin), b)


def test_cutoffs_and_clamp_match_reference(oracle):
    for cmin, cmax, cntmax in CUTOFF_CASES:
        p, b = cutoff_case(cmin, cmax, cntmax)
        _check(oracle.process_bin(b, p), "cutoff_ci%d_cx%d_cs%d" % (cmin, cmax, cntmax), b)


@pytest.mark.parametrize("case", sorted(CORNER_CASES))
def test_corners_match_reference(oracle, case):
    p, b = corner_case(case)
    _check(oracle.process_bin(b, p), case, b)


def test_edge_bins_match_reference(oracle):
    p = Params(k=31, cutoff_min=1, lut_prefix_len=7)
    for i, b in enumerate(edge_bins()):
        _check(oracle.process_bin(b, p), "edge_%d" % i, b)


def test_several_bins_many_sorters(oracle):
    """The reference ran these bins together with three sorter objects; each bin's result must not depend on that."""
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    for i, b in enumerate(several_bins()):
        _check(oracle.process_bin(b, p), "several_%d" % i, b)


@pytest.mark.parametrize("words,key_bytes", SORT_CASES)
def test_sort_matches_raduls(oracle, words, key_bytes):
    recs = sort_case(words, key_bytes)
    exp = reference_digest("sort_w%d_kb%d" % (words, key_bytes))
    assert digest_recs(recs) == exp["input"]
    assert digest_recs(oracle.sort(recs, key_bytes)) == exp["results"]["raduls_2_threads"]


def digest_recs(recs):
    from kmc_testlib import digest
    return digest(np.ascontiguousarray(recs, dtype=np.uint64))
