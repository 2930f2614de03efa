"""The second partition level's width and the leaf kernel of one-word bins (choose_b2, kL2SevenBitsMaxMean, kLeafCtaMinMean) on bins
just either side of every size where one of them changes, on a bin whose leaves need split table rounds, and on a bin with a dominant
k-mer: byte for byte the oracle's payload, LUT and statistics, and the width and kernel each bin takes (Stage2Context.leaf_plan).

The sizes where the plan changes (k = 31, mean leaf = k-mers / 2^(8 + bits)):
  * 2^25: the last bin with ~1 K-record leaves in 7 bits; above it 7 bits stay (8 bits before kL2SevenBitsMaxMean);
  * 1280 x 2^15: 7-bit leaves of more than kLeafCtaMinMean = 1280 records go to leaf_hash_cta_kernel;
  * 5120 x 2^15: the last bin of 7 bits (mean leaf 5 K records: its largest leaves are split rounds); above it 8 bits."""
import numpy as np
import pytest

from kmc_testlib import Bin, Oracle, Params, fast_bin, pack_superkmers

pytestmark = pytest.mark.gpu

P = Params(k=31, cutoff_min=2, lut_prefix_len=7)


def _run(p: Params, b: Bin):
    """kmcb200_process_bin on a fresh context (the environment is read when it is created): the result and the leaf plan of the bin."""
    import kmc_b200
    ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(p.k, p.both_strands, p.cutoff_min, p.cutoff_max, p.counter_max, p.lut_prefix_len), device=0, n_slots=1)
    r = ctx.process_bin(kmc_b200.SuperKmerBin(data=b.data, n_rec=b.n_rec, pack_bytes=b.pack_bytes, n_super_kmers=b.n_super_kmers, kmer_len=b.k))
    plan = ctx.leaf_plan(0)
    ctx.close()
    return r, plan


def _check(p: Params, b: Bin, bits, kernel):
    got, plan = _run(p, b)
    assert plan == (bits, kernel)
    want = Oracle().process_bin(b, p)
    assert tuple(got.stats) == tuple(want.stats)
    assert np.array_equal(got.lut, want.lut)
    assert got.payload.tobytes() == want.payload


@pytest.mark.parametrize("n,bits,kernel", [
    (1 << 25, 7, "hash"), ((1 << 25) + 4096, 7, "hash"),
    (1280 << 15, 7, "hash"), ((1280 << 15) + 4096, 7, "cta"),
    (5120 << 15, 7, "cta"), ((5120 << 15) + 4096, 8, "cta"),
])
def test_width_and_kernel_at_the_thresholds(n, bits, kernel):
    b = fast_bin(6100 + n % 997, 31, n)
    assert b.n_rec == n
    _check(P, b, bits, kernel)


def test_split_rounds_at_seven_bits(monkeypatch):
    """48 Mi k-mers in 7 bits (mean leaf 1.5 K records: the CTA kernel) with a 1024-slot CTA table: nearly every leaf is split."""
    monkeypatch.setenv("KMCB200_LEAF_CTA", "4:10")
    _check(P, fast_bin(6200, 31, 48 << 20), 7, "cta")


def test_dominant_kmer_at_seven_bits():
    """A 40 Mi-k-mer bin (7 bits, 8 before) plus 3 x 10^5 copies of poly-A: that leaf is beyond kLwHeavy and goes to the heavy launch."""
    rng = np.random.default_rng(62)
    k = 31
    base = fast_bin(6300, k, 40 << 20)
    heavy = pack_superkmers(k, [np.zeros(k, dtype=np.uint8)] * 300_000 + [rng.integers(0, 4, k + 60).astype(np.uint8) for _ in range(2000)])
    b = Bin(data=np.concatenate([base.data, heavy.data]), n_rec=base.n_rec + heavy.n_rec, n_super_kmers=base.n_super_kmers + heavy.n_super_kmers,
            pack_bytes=np.concatenate([base.pack_bytes, heavy.pack_bytes]).astype(np.uint64),
            pack_recs=np.concatenate([base.pack_recs, heavy.pack_recs]).astype(np.uint64), k=k)
    p = Params(k=k, cutoff_min=1, counter_max=2 ** 24 - 1, lut_prefix_len=7)
    _check(p, b, 7, "cta")
