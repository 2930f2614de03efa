"""CPU: the sequential stage-1 oracle (oracle/stage1_oracle.c) against the definition of a split and against stored results of the
unmodified reference CLI (tests/golden/stage1_reference.json, written by tests/golden/make_stage1_reference.py)."""
import json
import os

import numpy as np
import pytest

from stage1_testlib import (PACK_WINDOW, STAGE1_GOLDEN, Stage1Oracle, batch_of, expected_kmer_bins, kmer_signature, make_reads, random_map,
                            records)


@pytest.fixture(scope="module")
def s1():
    return Stage1Oracle()


def check_split(s1, batch, k, m, n_bins, seed=0):
    """Per bin: the multiset of k-mers is {k-mer : map[min norm m-mer]}; every record is consecutive k-mers of one signature, at most
    256 of them; packs are <= 64 KiB, non-empty, end on record boundaries and follow the s / 65408 rule."""
    sig_map = random_map(seed, m, n_bins)
    norm = s1.norm_table(m)
    sp = s1.split(batch, k, m, sig_map)
    exp = expected_kmer_bins(batch, k, m, sig_map, norm)
    assert int(sp.frags[:, 1].sum()) == sp.out.size and int(sp.frags[:, 5].sum()) == sp.pack_bytes.size
    for b in range(n_bins):
        f = sp.frags[b]
        recs = records(sp.bin_data(b), k)
        assert len(recs) == int(f[3]) and sum(a + 1 for a, _ in recs) == int(f[2])
        got = []
        for a, sym in recs:
            assert a + 1 <= 256
            sigs = {kmer_signature(sym[t:t + k], m, norm) for t in range(a + 1)}
            assert len(sigs) == 1 and int(sig_map[sigs.pop()]) == b
            got += ["".join("ACGT"[x] for x in sym[t:t + k]) for t in range(a + 1)]
        assert sorted(got) == exp.get(b, [])
        packs = sp.bin_packs(b)
        assert int(packs.sum()) == int(f[1]) and np.all(packs > 0) and np.all(packs <= 65536)
        starts, pos = [], 0
        for a, _ in recs:
            starts.append(pos)
            pos += 1 + (a + k + 3) // 4
        ends = np.cumsum(packs.astype(np.int64))
        pack_of = np.array([s // PACK_WINDOW for s in starts])
        first = [0] + [int(e) for e in ends[:-1]] if packs.size else []
        assert set(first) <= set(starts)
        for i, s in enumerate(starts):
            assert int(np.searchsorted(ends, s, side="right")) == len(np.unique(pack_of[:i + 1])) - 1
    return sp


@pytest.mark.parametrize("k,m", [(17, 5), (31, 9), (6, 5), (33, 11), (64, 7), (128, 5), (128, 11)])
def test_oracle_against_brute_force(s1, k, m):
    reads = make_reads(k * 7 + m, "short", n_reads=40, read_len=220) + make_reads(k + m, "n_dense", n_reads=20, read_len=300)
    check_split(s1, batch_of(reads), k, m, 37, seed=k)


@pytest.mark.parametrize("m", range(5, 12))
def test_every_signature_length(s1, m):
    reads = make_reads(100 + m, "short", n_reads=30, read_len=180)
    check_split(s1, batch_of(reads), 2 * m + 3, m, 16, seed=m)


def test_edge_inputs(s1):
    k, m = 21, 7
    rng = np.random.default_rng(5)
    rnd = lambda n: bytes(np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)])
    reads = [rnd(k - 1), rnd(k), rnd(k + 1), b"", b"N" + rnd(40), rnd(3) + b"N" + rnd(50), rnd(30).lower(), b"ACGTRYKMSWBDHVN" * 4,
             rnd(k) + b"N" + rnd(k), b"A" * 900, b"T" * 700, b"AC" * 600, b"ACGTTGCA" * 150, b"GATTACA" * 200 + rnd(60)]
    sp = check_split(s1, batch_of(reads), k, m, 9)
    assert max(a for b in range(9) for a, _ in records(sp.bin_data(b), k)) == 255      # runs of more than 256 k-mers are cut
    # k = m + 1, reads of exactly m + 1 symbols
    check_split(s1, batch_of([rnd(m + 1) for _ in range(30)] + [rnd(m) for _ in range(5)]), m + 1, m, 5)
    # low-complexity reads: poly-A k-mers have no allowed orientation, their signature is the special one (4^m, the map's last bin)
    sp = check_split(s1, batch_of(make_reads(3, "low_complexity", n_reads=12, read_len=2000)), 31, 9, 64)
    assert int(sp.frags[63][2]) > 1000


def test_identity_map_gives_signature_counts(s1):
    reads = make_reads(8, "short", n_reads=50)
    batch = batch_of(reads)
    cnt = s1.signature_counts(batch, 25, 7)
    norm = s1.norm_table(7)
    exp = expected_kmer_bins(batch, 25, 7, np.arange((1 << 14) + 1), norm)
    assert cnt.size == (1 << 14) + 1
    assert {s: int(c) for s, c in enumerate(cnt) if c} == {s: len(v) for s, v in exp.items()}


def test_batches_concatenate(s1):
    from stage1_testlib import concat_splits
    reads = make_reads(11, "long", n_reads=30, read_len=3000) + make_reads(12, "low_complexity", n_reads=5, read_len=3000)
    sig_map = random_map(3, 9, 50)
    whole = s1.split(batch_of(reads), 31, 9, sig_map)
    cuts = [0, 1, 5, 6, 17, 30, 33, 35]
    parts = concat_splits([s1.split(batch_of(reads[a:b]), 31, 9, sig_map, 50) for a, b in zip(cuts[:-1], cuts[1:])])
    for b in range(50):
        assert np.array_equal(parts.bin_data(b), whole.bin_data(b))
        assert np.array_equal(parts.frags[b][1:4], whole.frags[b][1:4])


# ----------------------------------------------------------------------------- against the reference CLI's stored results
def _golden():
    with open(STAGE1_GOLDEN) as f:
        return json.load(f)


def _cases():
    if not os.path.exists(STAGE1_GOLDEN):
        return []
    return sorted(_golden()["cases"])


@pytest.mark.parametrize("case", _cases())
def test_oracle_against_reference_cli(s1, case, oracle):
    """oracle split -> oracle stage 2 -> per file-bin payload / LUT digests equal the reference database's; the records add up to the
    reference's #Total_super-k-mers (short reads: the reference does not cut them into parts)."""
    from stage1_testlib import case_reads, load_map
    from kmc_testlib import Params, digest
    c = _golden()["cases"][case]
    reads = case_reads(case)
    sig_map = load_map(case)
    h = c["header"]
    n_bins = len(c["bins"])
    sp = s1.split(batch_of(reads), h["k"], h["sig_len"], sig_map, n_bins)
    p = Params(k=h["k"], both_strands=h["both"], cutoff_min=h["cmin"], cutoff_max=h["cmax"], counter_max=c["counter_max"], lut_prefix_len=h["p"])
    for b in range(n_bins):
        r = oracle.process_bin(sp.to_bin(b), p)
        assert {"payload": digest(r.payload), "lut": digest(np.asarray(r.lut, dtype=np.uint64))} == c["bins"][b], "bin %d" % b
    assert int(sp.frags[:, 2].sum()) == c["total_kmers"]
    if c["total_super_kmers"] is not None:
        assert int(sp.frags[:, 3].sum()) == c["total_super_kmers"]
