"""leaf_hash_cta_kernel (one hash table per CTA; KMCB200_LEAF_KERNEL=cta forces it on bins of any leaf size) against leaf_hash_kernel (one table per
warp, KMCB200_LEAF_KERNEL=hash) on the same seeded bins: the same payload, LUT and 8 result words, and neither took the LSD fallback."""
import numpy as np
import pytest

from kmc_testlib import Bin, Params, fast_bin, pack_superkmers

pytestmark = pytest.mark.gpu

CTA_CONFIGS = ["4:12", "4:10"]                          # KMCB200_LEAF_CTA: warps per CTA : log2(table slots)


def _ctx(p: Params):
    import kmc_b200
    return kmc_b200.Stage2Context(kmc_b200.Stage2Params(p.k, p.both_strands, p.cutoff_min, p.cutoff_max, p.counter_max, p.lut_prefix_len), device=0, n_slots=1)


def _dev_run(p: Params, b: Bin):
    """kmcb200_dev_process_bin on a fresh context (the environment is read when it is created): (payload bytes, LUT, the 8 result words)."""
    import torch
    ctx = _ctx(p)
    d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device="cuda")
    d_bin[:b.size] = torch.from_numpy(np.ascontiguousarray(b.data)).cuda()
    cap = ctx.out_capacity(b.n_rec) + 64
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device="cuda")
    d_res = torch.zeros(8, dtype=torch.int64, device="cuda")
    ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, b.n_rec, b.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    res = [int(x) for x in d_res.cpu().numpy().view(np.uint64)]
    out = d_out[:res[4] * ctx.out_rec_bytes].cpu().numpy().tobytes()
    lut = d_lut.cpu().numpy().view(np.uint64).copy()
    ctx.close()
    return out, lut, res


def _host_run(p: Params, b: Bin):
    """kmcb200_process_bin (the host path, which also counts oversized bins in key blocks): (payload bytes, LUT, the four statistics)."""
    import kmc_b200
    ctx = _ctx(p)
    r = ctx.process_bin(kmc_b200.SuperKmerBin(data=b.data, n_rec=b.n_rec, pack_bytes=b.pack_bytes, n_super_kmers=b.n_super_kmers, kmer_len=b.k))
    ctx.close()
    return r.payload.tobytes(), r.lut.copy(), list(r.stats)


def _check(monkeypatch, p: Params, b: Bin, env=None, cta="4:12", run=_dev_run):
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("KMCB200_LEAF_KERNEL", "hash")
    want = run(p, b)
    monkeypatch.setenv("KMCB200_LEAF_KERNEL", "cta")          # (by default only bins of large leaves take it)
    monkeypatch.setenv("KMCB200_LEAF_CTA", cta)
    got = run(p, b)
    if run is _dev_run:
        assert want[2][7] == 0 and got[2][7] == 0, "the LSD fallback took the bin"
    assert got[2] == want[2]
    assert np.array_equal(got[1], want[1])
    assert got[0] == want[0]
    return got


@pytest.mark.parametrize("cta", CTA_CONFIGS)
@pytest.mark.parametrize("coverage", ["30x", "2x", "distinct"])
def test_coverages(monkeypatch, cta, coverage):
    """2^20 k-mers: a 2-bit second level (leaves of ~1 K records) and a forced 1-bit one (~2 K records)."""
    n = 1 << 20
    genome = {"30x": n // 30, "2x": n // 2, "distinct": 4 * n}[coverage]
    b = fast_bin(4242, 31, n, genome_len=genome, err_ppm=0 if coverage == "distinct" else 10000)
    p = Params(k=31, cutoff_min=2 if coverage == "30x" else 1, lut_prefix_len=7)
    _check(monkeypatch, p, b, cta=cta)
    _check(monkeypatch, p, b, {"KMCB200_L2_BITS": "1"}, cta=cta)


@pytest.mark.parametrize("cta", ["4:12", "4:10"])
@pytest.mark.parametrize("env", [{"KMCB200_LEAF_RATIO0": "8"}, {"KMCB200_LEAF_FILL_PCT": "10"}, {"KMCB200_LEAF_RATIO0": "256", "KMCB200_LEAF_FILL_PCT": "85"}])
def test_split_and_predicated_rounds(monkeypatch, cta, env):
    """Rounds planned far too large (the shared table fills up: every warp stops, the round is split on the next bit) and far too small
    (many predicated rounds over one leaf), on leaves of ~8 K records (a 1-bit second level on 2^22 k-mers)."""
    n = 1 << 22
    b = fast_bin(777, 31, n, genome_len=n // 4)
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    _check(monkeypatch, p, b, dict(env, KMCB200_L2_BITS="1"), cta=cta)


def test_dominant_kmer_goes_the_heavy_way(monkeypatch):
    """A k-mer with 3 x 10^5 copies: its leaf is beyond kLwHeavy and is counted by the HEAVY launch of leaf_warp_kernel."""
    rng = np.random.default_rng(38)
    k = 31
    one = np.zeros(k, dtype=np.uint8)                     # poly-A
    lists = [one] * 300_000 + [rng.integers(0, 4, k + 60) for _ in range(4000)]
    p = Params(k=k, both_strands=True, cutoff_min=1, counter_max=2 ** 24 - 1, lut_prefix_len=7)
    _check(monkeypatch, p, pack_superkmers(k, lists))


@pytest.mark.parametrize("cmin,cmax,cntmax", [(1, 10 ** 9, 255), (2, 3, 255), (1, 1, 255), (3, 2, 255), (2, 2 ** 32 - 1, 100), (5, 100, 65535)])
def test_general_cutoffs(monkeypatch, cmin, cmax, cntmax):
    """The general instance: cutoff_min = 1, a reachable cutoff_max, cutoff_max < cutoff_min, counter_max below the counts."""
    b = fast_bin(99, 31, 1 << 20)
    p = Params(k=31, cutoff_min=cmin, cutoff_max=cmax, counter_max=cntmax, lut_prefix_len=7)
    _check(monkeypatch, p, b)


@pytest.mark.parametrize("p_len", [3, 7, 11])
def test_lut_prefix_longer_and_shorter_than_the_leaf(monkeypatch, p_len):
    """2^20 k-mers, 8 + 2 partition bits: a LUT prefix of 3 symbols is shared by a leaf (one_prefix), 7 and 11 are not."""
    b = fast_bin(1234, 31, 1 << 20)
    p = Params(k=31, cutoff_min=2, lut_prefix_len=p_len)
    _check(monkeypatch, p, b)


def test_oversized_bin_in_key_blocks(monkeypatch):
    """A bin counted key block by key block: the leaves carry the block's prefix (leaf_prefix != 0)."""
    b = fast_bin(31337, 31, 1_300_000)
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    _check(monkeypatch, p, b, {"KMCB200_MAX_BLOCK_RECORDS": "150000"}, run=_host_run)


@pytest.mark.parametrize("cta", CTA_CONFIGS)
def test_leaves_of_exact_sizes(monkeypatch, cta):
    """-b mode, k = 31, 8 + 2 partition bits: a leaf is the first 5 symbols.  Filler k-mers never start with A; the leaves AAAAA .. AAACA hold
    exactly 0, 1, 32 (8 k-mers x 4), 4096 (1024 x 4) and 4096 distinct records (more than 7/8 of a 4096-slot table: split)."""
    rng = np.random.default_rng(5)
    k = 31

    def kmers(prefix, n):
        return [np.concatenate([np.array(prefix, dtype=np.uint8), rng.integers(0, 4, k - len(prefix)).astype(np.uint8)]) for _ in range(n)]

    lists = [rng.integers(1, 4, k + 99).astype(np.uint8) for _ in range(1500)]          # 150 000 filler k-mers
    lists += kmers([0, 0, 0, 0, 1], 1)
    lists += kmers([0, 0, 0, 0, 2], 8) * 4
    lists += kmers([0, 0, 0, 0, 3], 1024) * 4
    lists += kmers([0, 0, 0, 1, 0], 4096)
    order = rng.permutation(len(lists))
    b = pack_superkmers(k, [lists[i] for i in order])
    p = Params(k=k, both_strands=False, cutoff_min=1, lut_prefix_len=7)
    _check(monkeypatch, p, b, {"KMCB200_L2_BITS": "2"}, cta=cta)
