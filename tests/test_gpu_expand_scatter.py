"""The level 1 of a bin of one-word records on the MSD path: a counting expansion (expand_kernel<kExpandCells>) and an expansion that writes
every k-mer straight into its level-1 bucket (expand_kernel<kExpandPartition>, the `expand_scatter_L1` interval).  Each case is compared
with the sequence that writes the records in tile order and partitions them afterwards (dev_expand -> dev_sort(hist_ready) -> dev_count,
which keeps expand_kernel<kExpandAll> + msd_partition_kernel) and with the oracle: the same payload, LUT and result words."""
import numpy as np
import pytest

from kmc_testlib import Bin, Params, bin_extras, fast_bin, pack_superkmers

pytestmark = pytest.mark.gpu

P_LEN = {17: 5, 31: 7, 32: 8}


def _ctx(p: Params, n_slots=1):
    import kmc_b200
    return kmc_b200.Stage2Context(kmc_b200.Stage2Params(p.k, p.both_strands, p.cutoff_min, p.cutoff_max, p.counter_max, p.lut_prefix_len), device=0, n_slots=n_slots)


def _dev_bin(b: Bin):
    import torch
    d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device="cuda")
    d_bin[:b.size] = torch.from_numpy(np.ascontiguousarray(b.data)).cuda()
    return d_bin


def _outputs(ctx, n_rec):
    import torch
    cap = ctx.out_capacity(n_rec) + 64
    return (torch.zeros(cap, dtype=torch.uint8, device="cuda"), torch.zeros(ctx.lut_entries, dtype=torch.int64, device="cuda"),
            torch.zeros(8, dtype=torch.int64, device="cuda"), cap)


def _words(ctx, d_out, d_lut, d_res):
    res = [int(x) for x in d_res.cpu().numpy().view(np.uint64)]
    return d_out[:res[4] * ctx.out_rec_bytes].cpu().numpy().tobytes(), d_lut.cpu().numpy().view(np.uint64).copy(), res


def _new_path(ctx, b: Bin, n_rec=None):
    """kmcb200_dev_process_bin: (payload, LUT, the 8 result words, the sort's interval names)."""
    import torch
    n_rec = b.n_rec if n_rec is None else n_rec
    d_bin = _dev_bin(b)
    d_out, d_lut, d_res, cap = _outputs(ctx, max(n_rec, 1))
    ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, n_rec, b.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return _words(ctx, d_out, d_lut, d_res) + (ctx.stage_times(0)["pass_names"],)


def _old_path(ctx, b: Bin):
    """dev_expand (records in tile order) -> dev_sort(hist_ready) (msd_partition_kernel at level 1) -> dev_count."""
    import torch
    st = torch.cuda.current_stream().cuda_stream
    n = b.n_rec
    d_bin = _dev_bin(b)
    d_recs = torch.zeros(n + 8, dtype=torch.int64, device="cuda")
    d_tmp = torch.zeros(n + 8, dtype=torch.int64, device="cuda")
    d_out, d_lut, d_res, cap = _outputs(ctx, n)
    ctx.dev_expand(0, d_bin.data_ptr(), b.size, n, b.pack_bytes, d_recs.data_ptr(), None, st)
    where = ctx.dev_sort(0, d_recs.data_ptr(), d_tmp.data_ptr(), n, hist_ready=True, stream=st)
    names = ctx.stage_times(0)["pass_names"]
    ctx.dev_count(0, (d_tmp if where == 1 else d_recs).data_ptr(), n, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(), st)
    torch.cuda.synchronize()
    return _words(ctx, d_out, d_lut, d_res) + (names,)


def _check(oracle, p: Params, b: Bin, scatter=True, fallback=0):
    """New path == old path == oracle.  scatter: the bin takes the new level 1 (else the sort sees no MSD path: both run msd_partition or
    the LSD passes).  fallback: the new path's result[7] (the LSD fallback sorted the bin from the level-1 output); the old path's
    dev_count reports no fallback, so word 7 is compared only when it is 0."""
    e = oracle.process_bin(b, p)
    ctx = _ctx(p)
    new = _new_path(ctx, b)
    old = _old_path(ctx, b)
    ctx.close()
    assert ("expand_scatter_L1" in new[3]) == scatter, new[3]
    assert "expand_scatter_L1" not in old[3]
    if scatter:
        assert "msd_partition_L1" in old[3] and "msd_partition_L1" not in new[3]
    assert new[2][7] == fallback
    assert new[2][:7] == old[2][:7]
    if fallback == 0:
        assert new[2] == old[2]
    assert np.array_equal(new[1], old[1]) and np.array_equal(new[1], e.lut)
    assert new[0] == old[0] and new[0] == e.payload
    assert tuple(new[2][:4]) == tuple(e.stats)
    return new


@pytest.mark.parametrize("both", [True, False], ids=["ci", "b"])
@pytest.mark.parametrize("k", [17, 31, 32])
def test_widths_and_strands(oracle, k, both):
    """One-word k-mers whose top digit starts at bit 26, 54 and 56; canonical and -b mode."""
    p = Params(k=k, both_strands=both, cutoff_min=2, lut_prefix_len=P_LEN[k])
    _check(oracle, p, fast_bin(60 + k + both, k, 600_000))


@pytest.mark.parametrize("n", [65_535, 65_536, 70_001])
def test_around_the_msd_threshold(oracle, n):
    """Below 2^16 records the sort is the plain LSD passes: the bin keeps the single expansion into tile order."""
    p = Params(k=31, cutoff_min=1, lut_prefix_len=7)
    _check(oracle, p, fast_bin(n, 31, n, genome_len=n // 3), scatter=n >= 1 << 16)


@pytest.mark.parametrize("mean_extra", [0.3, 2.0, 200.0])
def test_staged_and_unstaged_tiles(oracle, mean_extra):
    """~1.3 k-mers per super-k-mer: a tile of 4096 k-mers spans more than 12 KB of the bin and more than 1024 super-k-mers, so its k-mers
    are extracted from global memory (the unstaged branch); ~3 per super-k-mer mixes both kinds; ~200 has few super-k-mers per tile.
    Every pack's last tile is partial."""
    p = Params(k=31, cutoff_min=1, lut_prefix_len=7)
    b = fast_bin(int(mean_extra * 10) + 3, 31, 400_000, genome_len=150_000, mean_extra=mean_extra)
    _check(oracle, p, b)


def test_all_distinct(oracle):
    n = 1 << 20
    p = Params(k=31, cutoff_min=1, lut_prefix_len=7)
    _check(oracle, p, fast_bin(4711, 31, n, genome_len=4 * n, err_ppm=0))


def test_dominant_poly_a(oracle):
    """2000 poly-A super-k-mers of k + 255 symbols: 512 000 copies of one k-mer, whole tiles whose every k-mer has digit 0."""
    k = 31
    rng = np.random.default_rng(11)
    lists = [np.zeros(k + 255, dtype=np.uint8)] * 2000 + [rng.integers(0, 4, k + 60).astype(np.uint8) for _ in range(4000)]
    p = Params(k=k, both_strands=True, cutoff_min=1, counter_max=2 ** 24 - 1, lut_prefix_len=7)
    _check(oracle, p, pack_superkmers(k, lists))


def test_skewed_bin_takes_the_lsd_fallback(oracle):
    """A poly-A leaf of more than 2^22 records is beyond what the leaf kernels stream: the LSD fallback sorts the bin, starting from the
    buffer the level-1 partition expansion wrote."""
    k = 31
    rng = np.random.default_rng(12)
    lists = [np.zeros(k + 255, dtype=np.uint8)] * 16_500 + [rng.integers(0, 4, k + 80).astype(np.uint8) for _ in range(3000)]
    p = Params(k=k, both_strands=True, cutoff_min=1, counter_max=2 ** 32 - 1, lut_prefix_len=7)
    _check(oracle, p, pack_superkmers(k, lists), fallback=1)


@pytest.mark.parametrize("delta", [1, -1])
def test_malformed_bin_stops_on_the_device(oracle, delta):
    """n_rec one more / one less than the bin holds: the pack scan stops the bin before the counting expansion writes a cell, the
    partition expansion and everything behind it return at once, nothing is emitted.  A good bin on the same context is then right."""
    import kmc_b200
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    b = fast_bin(5, 31, 300_000)
    ctx = _ctx(p)
    out, lut, res, names = _new_path(ctx, b, n_rec=b.n_rec + delta)
    assert res[6] != 0 and res[4] == 0 and not lut.any()
    assert "expand_scatter_L1" in names
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        ctx.process_bin(kmc_b200.SuperKmerBin(data=b.data, n_rec=b.n_rec + delta, pack_bytes=b.pack_bytes, n_super_kmers=b.n_super_kmers, kmer_len=b.k))
    assert ei.value.code == kmc_b200.ERR_BIN_FORMAT
    e = oracle.process_bin(b, p)
    got = _new_path(ctx, b)
    ctx.close()
    assert got[0] == e.payload and np.array_equal(got[1], e.lut) and tuple(got[2][:4]) == tuple(e.stats) and got[2][6] == 0


@pytest.mark.parametrize("indexed", [False, True], ids=["walk", "indexed"])
def test_submitted_bins_in_two_slots(oracle, indexed):
    """submit_bin / submit_bin_indexed (the length bytes instead of the walk) into two slots, waited in reverse order."""
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    bins = [fast_bin(70 + j, 31, 500_000 + 1000 * j) for j in range(2)]
    exp = [oracle.process_bin(b, p) for b in bins]
    ctx = _ctx(p, n_slots=2)
    held = []
    for slot, b in enumerate(bins):
        data = np.ascontiguousarray(b.data)
        packs = np.ascontiguousarray(b.pack_bytes, dtype=np.uint64)
        out = np.zeros(ctx.out_capacity(b.n_rec) + 64, dtype=np.uint8)
        lut = np.zeros(ctx.lut_entries, dtype=np.uint64)
        if indexed:
            extras, psk = bin_extras(b)
            ctx.submit_bin_indexed(slot, data.ctypes.data, data.size, b.n_rec, packs, extras, psk, out.ctypes.data, out.size, lut.ctypes.data)
        else:
            ctx.submit_bin(slot, data.ctypes.data, data.size, b.n_rec, packs, out.ctypes.data, out.size, lut.ctypes.data)
        held.append((data, out, lut))
    for slot in (1, 0):
        nb, stats = ctx.wait_bin(slot)
        _, out, lut = held[slot]
        assert "expand_scatter_L1" in ctx.stage_times(slot)["pass_names"]
        assert stats == exp[slot].stats and out[:nb].tobytes() == exp[slot].payload and np.array_equal(lut, exp[slot].lut)
    ctx.close()
