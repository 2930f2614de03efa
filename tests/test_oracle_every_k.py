"""CPU: the oracle against the unmodified reference at every k = 5 .. 128, in both strand modes.  Much of the device code extracts bits at
positions that depend on k (k mod 4, k mod 32, where 2k falls relative to a 64-bit word, where the LUT prefix falls); a GPU result that
agrees with the oracle at some k proves something only once the oracle itself agrees with the reference there.  The reference's results
are stored as digests in tests/golden/reference_digests.json (tests/golden/make_reference_digests.py, group `every_k`).

The parameters of a (k, strand) case - LUT prefix, counter width, cutoff_min - are the ones tests/test_gpu_every_k.py runs the GPU with."""
import pytest

from kmc_testlib import Params, bin_digest, result_digest, reference_digest, synth_bin

EVERY_K = range(5, 129)
# counter widths rotated over 0 .. 4 bytes: (counter_max, cutoff_max)
WIDTHS = [(1, 10 ** 9), (255, 10 ** 9), (65535, 10 ** 9), (2 ** 24 - 1, 10 ** 9), (2 ** 32 - 1, 10 ** 9)]


def legal_prefixes(k, max_p=11):
    """LUT prefix lengths kmcb200_create takes for k (1 <= p < k, p <= 15, (k - p) % 4 == 0), up to max_p."""
    return [p for p in range(1, min(k - 1, max_p) + 1) if (k - p) % 4 == 0]


def splits_prefix(k, p):
    """Does the LUT prefix [2(k-p), 2k) of a k-mer span two 64-bit words of its record?"""
    return k > 32 and k % 32 != 0 and p > k % 32


def sweep_prefix(k, both):
    """The LUT prefix of case (k, both): the legal values rotated across k, the two strand modes of one k on different values where there
    are two; for k > 32, one of the two splits the prefix across a word wherever a legal p does."""
    legal = legal_prefixes(k)
    ci, b = legal[k % len(legal)], legal[(k + 1) % len(legal)]
    split = [p for p in legal if splits_prefix(k, p)]
    if split and not (splits_prefix(k, ci) or splits_prefix(k, b)):
        b = split[k % len(split)]
    return ci if both else b


def sweep_params(k, both):
    cntmax, cmax = WIDTHS[(2 * k + int(both)) % len(WIDTHS)]
    return Params(k=k, both_strands=both, cutoff_min=1 + (k + int(both)) % 2, cutoff_max=cmax, counter_max=cntmax, lut_prefix_len=sweep_prefix(k, both))


def every_k_case(k, both):
    """A small bin (2500 super-k-mers, ~3 x 10^4 k-mers of a 3000-symbol genome) for case (k, both)."""
    return sweep_params(k, both), synth_bin(5000 + 2 * k + int(both), k, 2500, genome_len=3000, err=0.02)


def case_name(k, both):
    return "every_k%d_both%d" % (k, int(both))


def test_sweep_covers_the_prefix_and_counter_classes():
    """Every legal p up to 11 of a k appears among the sweep's k of its residue mod 4; every k > 32 that has a word-splitting p uses one;
    every counter width appears in both strand modes."""
    used = {(k, sweep_prefix(k, both)) for k in EVERY_K for both in (True, False)}
    for k in EVERY_K:
        assert all(1 <= p < k and p <= 15 and (k - p) % 4 == 0 for kk, p in used if kk == k)
        if any(splits_prefix(k, p) for p in legal_prefixes(k)):
            assert any(splits_prefix(k, p) for kk, p in used if kk == k), k
    for r in range(4):
        want = {p for k in EVERY_K if k % 4 == r for p in legal_prefixes(k)}
        assert want == {p for k, p in used if k % 4 == r}, r
    for both in (True, False):
        assert {sweep_params(k, both).counter_bytes for k in EVERY_K} == {0, 1, 2, 3, 4}


@pytest.mark.parametrize("k", EVERY_K)
def test_every_k_matches_reference(oracle, k):
    for both in (True, False):
        p, b = every_k_case(k, both)
        exp = reference_digest(case_name(k, both))
        assert bin_digest(b) == exp["input"], "%s: the generated input is not the one the reference result was stored for" % case_name(k, both)
        got = result_digest(oracle.process_bin(b, p))
        for variant, r in exp["results"].items():
            assert got == r, "%s: oracle != reference (%s)" % (case_name(k, both), variant)
