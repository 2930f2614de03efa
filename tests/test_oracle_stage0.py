"""CPU: stage 0 — the oracle's signature statistics (a literal CalcStats) against the definition and the identity-map split, its (k+x)-mer
counts (oracle/stage0_oracle.c) against the collector's rule, and the library's host-only signature map and stage-2 bin order against the maps stored in the
reference's .kmc_pre files (tests/golden/stage1_maps.npz)."""
import json

import numpy as np
import pytest

from stage0_testlib import file_position_map, kxmer_count_restated, max_x_of, oracle_kxmer_totals, oracle_signature_stats
from stage1_testlib import (STAGE1_CASES, STAGE1_GOLDEN, Stage1Oracle, batch_of, case_reads, expected_kmer_bins, load_map, make_reads, random_map,
                            records)


@pytest.fixture(scope="module")
def s1():
    return Stage1Oracle()


def brute_stats(s1, batch, k, m):
    exp = expected_kmer_bins(batch, k, m, np.arange((1 << (2 * m)) + 1), s1.norm_table(m))
    out = np.zeros((1 << (2 * m)) + 1, dtype=np.uint32)
    for sig, kmers in exp.items():
        out[sig] = len(kmers)
    return out


def edge_reads(k, seed):
    rng = np.random.default_rng(seed)
    rnd = lambda n: bytes(np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)])
    return [rnd(k - 1), rnd(k), rnd(k + 1), b"", b"N" + rnd(40), rnd(3) + b"N" + rnd(50), rnd(30).lower(), b"ACGTRYKMSWBDHVN" * 4,
            rnd(k) + b"N" + rnd(k), b"A" * 900, b"T" * 700, b"AC" * 600, b"GATTACA" * 200 + rnd(60)]


@pytest.mark.parametrize("m", range(5, 12))
def test_signature_stats_equal_the_definition(s1, m):
    k = 2 * m + 3
    batches = {
        "n_dense": batch_of(make_reads(200 + m, "n_dense", n_reads=25, read_len=200)),
        "low_complexity": batch_of(make_reads(300 + m, "low_complexity", n_reads=3, read_len=1500)),
        "multi_read": batch_of(make_reads(400 + m, "short", n_reads=30, read_len=150)),
        "edge": batch_of(edge_reads(k, m)),
    }
    for name, batch in batches.items():
        got = oracle_signature_stats(batch, k, m)
        assert np.array_equal(got, brute_stats(s1, batch, k, m)), name
        if m <= 7:
            assert np.array_equal(got.astype(np.int64), s1.signature_counts(batch, k, m)), name


@pytest.mark.parametrize("k,m", [(6, 5), (31, 9), (64, 7), (128, 11)])
def test_signature_stats_other_k(s1, k, m):
    batch = batch_of(make_reads(k + m, "short", n_reads=20, read_len=300) + make_reads(k, "n_dense", n_reads=10, read_len=200) + edge_reads(k, 3))
    got = oracle_signature_stats(batch, k, m)
    assert np.array_equal(got, brute_stats(s1, batch, k, m))
    assert int(got.sum()) == int(s1.split(batch, k, m, np.zeros((1 << (2 * m)) + 1, np.uint32), 1).frags[0, 2])


@pytest.mark.parametrize("k", [17, 28, 29, 30, 55])
@pytest.mark.parametrize("both", [True, False])
def test_oracle_kxmer_counts_equal_the_collector_rule(s1, k, both):
    assert max_x_of(k) in (1, 2, 3)
    reads = make_reads(k, "short", n_reads=40, read_len=300) + make_reads(k + 1, "low_complexity", n_reads=3, read_len=1500) + \
        make_reads(k + 2, "n_dense", n_reads=30, read_len=200)
    sp = s1.split(batch_of(reads), k, 7, random_map(k, 7, 16), 16)
    got = oracle_kxmer_totals(sp, both)
    exp = [sum(kxmer_count_restated(sym, k, both) for _, sym in records(sp.bin_data(b), k)) for b in range(16)]
    assert [int(x) for x in got] == exp
    assert int(got.sum()) > 0


def test_kxmer_counts_are_zero_without_x(s1):
    sp = s1.split(batch_of(make_reads(1, "short", n_reads=20)), 32, 7, random_map(1, 7, 8), 8)
    assert not oracle_kxmer_totals(sp, True).any() and not oracle_kxmer_totals(sp, False).any()


def mapper_and_order(s1, case):
    """The library's map + bin order from oracle statistics and oracle bin totals, as count_reads computes them from GPU ones."""
    import kmc_b200
    c = json.load(open(STAGE1_GOLDEN))["cases"][case]
    h = c["header"]
    k, m, n_bins = h["k"], h["sig_len"], len(c["bins"])
    batch = batch_of(case_reads(case))
    mapper = kmc_b200.signature_map(oracle_signature_stats(batch, k, m), m, n_bins)
    sp = s1.split(batch, k, m, np.maximum(mapper, 0).astype(np.uint32), n_bins)
    kx = oracle_kxmer_totals(sp, h["both"])
    pos = kmc_b200.stage2_bin_order(sp.frags[:, 1], sp.frags[:, 2], kx, k, h["cmin"], h["cmax"], c["counter_max"], h["p"])
    return mapper, pos


@pytest.mark.parametrize("case", sorted(STAGE1_CASES))
def test_map_and_bin_order_reproduce_the_reference_kmc_pre(s1, case):
    mapper, pos = mapper_and_order(s1, case)
    assert sorted(pos.tolist()) == list(range(pos.size))
    assert np.array_equal(file_position_map(mapper, pos), load_map(case))


def test_map_invariants_and_refusals():
    import kmc_b200
    for m, n_bins, seed in ((5, 64, 1), (7, 512, 2), (9, 2000, 3), (11, 4096, 4), (9, 64, 5)):
        rng = np.random.default_rng(seed)
        counts = (rng.pareto(1.2, (1 << (2 * m)) + 1) * 50).astype(np.uint32)
        mp = kmc_b200.signature_map(counts, m, n_bins)
        allowed = np.array([is_allowed(x, m) for x in range(1 << (2 * m))] + [False])
        assert np.array_equal(mp >= 0, allowed | (np.arange(mp.size) == mp.size - 1))
        assert mp.max() < n_bins and mp[-1] == mp.max()
        assert np.array_equal(mp, kmc_b200.signature_map(counts, m, n_bins))
    zeros = np.zeros((1 << 14) + 1, np.uint32)
    for m, n_bins in ((4, 64), (12, 64), (7, 1), (7, 0), (7, 4097)):
        with pytest.raises(kmc_b200.KmcB200Error) as ei:
            kmc_b200.signature_map(np.zeros((1 << (2 * m)) + 1, np.uint32) if m != 12 else zeros, m, n_bins)
        assert ei.value.code == kmc_b200.ERR_INVALID
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        kmc_b200.stage2_bin_order([1, 2], [1, 2], None, 29, 2, 255, 255, 5)      # k = 29 sorts (k+x)-mers: their counts are needed
    assert ei.value.code == kmc_b200.ERR_INVALID
    # k % 32 == 0: plain k-mers, the largest need first
    assert list(kmc_b200.stage2_bin_order([0, 3000, 30, 10 ** 6], [0, 1000, 10, 10 ** 5], None, 32, 2, 255, 255, 8)) == [3, 1, 2, 0]


def is_allowed(x, m):
    """mmer.h:40-63 symbol by symbol: no AA after the first symbol, no ACA prefix, no TT? or TGT suffix"""
    s = [(x >> (2 * (m - 1 - i))) & 3 for i in range(m)]
    if any(s[i] == 0 and s[i + 1] == 0 for i in range(1, m - 1)):
        return False
    return s[:3] != [0, 1, 0] and s[m - 3:m - 1] != [3, 3] and s[m - 3:] != [3, 2, 3]
