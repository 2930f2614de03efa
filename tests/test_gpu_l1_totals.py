"""Level 1 of a bin of one-word records on the MSD path from the pack walk's digit totals: the walk counts the level-1 digit of every
k-mer into 256 totals, msd_bounds_kernel makes them the bucket boundaries, and the one expansion of the bin (expand_kernel<kExpandPartition>,
the `expand_scatter_L1` interval) reserves every tile's run inside each bucket with a global atomicAdd.  The order of the records inside a
level-1 bucket therefore varies from run to run; what the bin emits must not.  Every case is compared with the oracle."""
import numpy as np
import pytest

from kmc_testlib import Bin, Params, fast_bin, pack_superkmers

pytestmark = pytest.mark.gpu


def _run(ctx, b: Bin):
    """kmcb200_dev_process_bin: (payload, LUT, the 8 result words, the sort's interval names)."""
    import torch
    d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device="cuda")
    d_bin[:b.size] = torch.from_numpy(np.ascontiguousarray(b.data)).cuda()
    cap = ctx.out_capacity(b.n_rec) + 64
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device="cuda")
    d_res = torch.zeros(8, dtype=torch.int64, device="cuda")
    ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, b.n_rec, np.ascontiguousarray(b.pack_bytes, dtype=np.uint64), d_out.data_ptr(), cap,
                        d_lut.data_ptr(), d_res.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    res = [int(x) for x in d_res.cpu().numpy().view(np.uint64)]
    return (d_out[:res[4] * ctx.out_rec_bytes].cpu().numpy().tobytes(), d_lut.cpu().numpy().view(np.uint64).copy(), res,
            ctx.stage_times(0)["pass_names"])


def _ctx(p: Params):
    import kmc_b200
    return kmc_b200.Stage2Context(kmc_b200.Stage2Params(p.k, p.both_strands, p.cutoff_min, p.cutoff_max, p.counter_max, p.lut_prefix_len), device=0)


def _same_as_oracle(got, e):
    out, lut, res, _ = got
    assert res[6] == 0, res
    assert out == e.payload and np.array_equal(lut, e.lut) and tuple(res[:4]) == tuple(e.stats)


def test_packs_over_64k_are_counted_by_the_warp_walker(oracle):
    """Packs of ~128 KiB (two collector flushes each) are left to the exact warp walker, whose lanes count the digits of the super-k-mers
    they index: the bin still takes the level-1 partition expansion."""
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    b = fast_bin(91, 31, 1 << 18)
    pb = np.asarray(b.pack_bytes, dtype=np.uint64)
    pr = np.asarray(b.pack_recs, dtype=np.uint64)
    if pb.size % 2:
        pb, pr = np.append(pb, np.uint64(0)), np.append(pr, np.uint64(0))
    big = Bin(data=b.data, n_rec=b.n_rec, n_super_kmers=b.n_super_kmers, pack_bytes=pb[0::2] + pb[1::2], pack_recs=pr[0::2] + pr[1::2], k=31)
    assert big.pack_bytes.max() > 1 << 16 and big.n_rec >= 1 << 16
    ctx = _ctx(p)
    got = _run(ctx, big)
    ctx.close()
    assert "expand_scatter_L1" in got[3] and "msd_partition_L1" not in got[3], got[3]
    _same_as_oracle(got, oracle.process_bin(b, p))


def test_repeated_runs_emit_the_same(oracle):
    """The same bin five times on one context: the runs inside the level-1 buckets land in another order each time, the payload, the
    LUT and the 8 result words do not change."""
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    b = fast_bin(92, 31, 1 << 20)
    ctx = _ctx(p)
    runs = [_run(ctx, b) for _ in range(5)]
    ctx.close()
    assert "expand_scatter_L1" in runs[0][3]
    for r in runs[1:]:
        assert r[0] == runs[0][0] and np.array_equal(r[1], runs[0][1]) and r[2] == runs[0][2]
    _same_as_oracle(runs[0], oracle.process_bin(b, p))


@pytest.mark.parametrize("both", [True, False], ids=["ci", "b"])
def test_smallest_k_of_the_msd_path(oracle, both):
    """k = 12 (2k = 24 bits, the least the MSD path takes): the forward window (symbols 0-3) and the reverse one (symbols 8-11) of a k-mer
    are closest together."""
    p = Params(k=12, both_strands=both, cutoff_min=1, lut_prefix_len=4)
    b = fast_bin(93 + both, 12, 300_000)
    ctx = _ctx(p)
    got = _run(ctx, b)
    ctx.close()
    assert "expand_scatter_L1" in got[3], got[3]
    _same_as_oracle(got, oracle.process_bin(b, p))


@pytest.mark.parametrize("both", [True, False], ids=["ci", "b"])
def test_one_top_digit_takes_nearly_all(oracle, both):
    """Super-k-mers of 31 A's and 27 random symbols: every one of their k-mers starts with AAAA, so ~97 % of the bin has level-1 digit 0
    (in both strand modes) and nearly every tile's reservation goes to the same cursor."""
    k = 31
    rng = np.random.default_rng(14)
    lists = [np.concatenate([np.zeros(k, dtype=np.uint8), rng.integers(0, 4, 27).astype(np.uint8)]) for _ in range(3000)]
    lists += [rng.integers(0, 4, k + 40).astype(np.uint8) for _ in range(60)]
    p = Params(k=k, both_strands=both, cutoff_min=1, counter_max=65535, lut_prefix_len=7)
    b = pack_superkmers(k, lists)
    assert b.n_rec >= 1 << 16
    ctx = _ctx(p)
    got = _run(ctx, b)
    ctx.close()
    assert "expand_scatter_L1" in got[3], got[3]
    _same_as_oracle(got, oracle.process_bin(b, p))


def test_dominant_kmer_found_in_any_record_order(oracle):
    """A poly-A k-mer with 3 x 10^5 copies behind 4000 random super-k-mers: the first record of its leaf is seldom a poly-A one now that
    level-1 runs arrive in no fixed order, and the heavy launch must still find the dominant k-mer (no LSD fallback)."""
    k = 31
    rng = np.random.default_rng(39)
    lists = [rng.integers(0, 4, k + 60).astype(np.uint8) for _ in range(4000)] + [np.zeros(k, dtype=np.uint8)] * 300_000
    p = Params(k=k, both_strands=True, cutoff_min=1, counter_max=2 ** 24 - 1, lut_prefix_len=7)
    b = pack_superkmers(k, lists)
    ctx = _ctx(p)
    got = _run(ctx, b)
    ctx.close()
    assert got[2][7] == 0, "the LSD fallback took the bin"
    _same_as_oracle(got, oracle.process_bin(b, p))
