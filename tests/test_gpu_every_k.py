"""GPU: every k-mer length from 5 to 128 against the oracles.  Much of the device code extracts bits at positions that depend on k: the
level-1 digit totals of one-word records on k mod 4, the level-1 and level-2 digits, the 12-bit key-block prefix and the LUT prefix of
wide records on where they fall relative to a 64-bit word, stage 1's (k+x)-mer counts on k mod 32.  Each stage-2 case is compared with
the oracle byte for byte (payload, LUT, the four statistics) and asserts the path it claims to take, so that a case that falls back to
another path fails.  tests/test_oracle_every_k.py pins the oracle to the unmodified reference at the same (k, strand, p, counter width).
  * the stage-2 sweep: every k in both strand modes, two bins of 1.5 - 2.5 x 10^5 k-mers on one context (k >= 12: the MSD partition and
    the counted leaves; k < 12: the LSD passes), the LUT prefix and the counter width rotated across k;
  * the expansion at every k, on bins whose padding symbols are garbage, before a sort can hide a wrong record;
  * a forced level 2 whose digit [2k-8-b2, 2k-8) spans two words, for every k mod 32 class that has one and every wide record width;
  * key blocks (both flows) and one bin over several contexts at the k whose 12-bit prefix [2k-12, 2k) spans two words, and around them;
  * stage 1 with (k+x)-mer counts and stage 0's signature statistics for every k from m + 1 to 128."""
import numpy as np
import pytest

from kmc_testlib import Bin, Params, synth_bin
from test_oracle_every_k import EVERY_K, sweep_params

pytestmark = pytest.mark.gpu


def _ctx(p: Params, n_slots=1):
    import kmc_b200
    return kmc_b200.Stage2Context(kmc_b200.Stage2Params(p.k, p.both_strands, p.cutoff_min, p.cutoff_max, p.counter_max, p.lut_prefix_len), device=0, n_slots=n_slots)


def _skb(b: Bin):
    import kmc_b200
    return kmc_b200.SuperKmerBin(data=b.data, n_rec=b.n_rec, pack_bytes=b.pack_bytes, n_super_kmers=b.n_super_kmers, kmer_len=b.k)


def _same(r, e):
    """r: kmc_b200.BinResult, e: the oracle's."""
    assert r.stats == e.stats
    assert np.array_equal(r.lut, e.lut)
    assert r.payload.tobytes() == e.payload


def _dev_run(ctx, b: Bin):
    """kmcb200_dev_process_bin on device copies of the bin: (BinResult, the 8 result words)."""
    import torch
    import kmc_b200
    d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device="cuda")
    d_bin[:b.size] = torch.from_numpy(np.ascontiguousarray(b.data)).cuda()
    cap = ctx.out_capacity(b.n_rec) + 64
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device="cuda")
    d_res = torch.zeros(8, dtype=torch.int64, device="cuda")
    ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, b.n_rec, b.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(),
                        torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    res = [int(x) for x in d_res.cpu().numpy().view(np.uint64)]
    return kmc_b200.BinResult(d_out[:res[4] * ctx.out_rec_bytes].cpu().numpy(), d_lut.cpu().numpy().view(np.uint64), *res[:4]), res


def concat_bins(*bins):
    """One bin holding the records of several (their collector packs one after the other)."""
    return Bin(data=np.concatenate([b.data for b in bins]), n_rec=sum(b.n_rec for b in bins), n_super_kmers=sum(b.n_super_kmers for b in bins),
               pack_bytes=np.concatenate([b.pack_bytes for b in bins]).astype(np.uint64), pack_recs=np.concatenate([b.pack_recs for b in bins]).astype(np.uint64),
               k=bins[0].k)


def sweep_bin(seed, k, scale=1.0):
    """~1.9 x 10^5 k-mers at scale 1: a 30x part plus a part whose k-mers occur ~2000 times (counts beyond one byte, clamped by the
    1-byte counters)."""
    n1, n2 = int(8000 * scale), int(9000 * scale)
    return concat_bins(synth_bin(seed, k, n1, genome_len=3000, err=0.01), synth_bin(seed + 1, k, n2, genome_len=k + 45, max_extra=20, err=0.0))


def assert_bin_path(names, k):
    """k >= 12 (2k >= 24 bits) and >= 2^16 k-mers: the MSD path with counted leaves, one-word records expanded straight into their level-1
    buckets from the pack walk's digit totals, wider ones partitioned after a tile-order expansion; k < 12: the LSD passes alone."""
    if k >= 12:
        assert "leaf_count" in names, names
        assert ("expand_scatter_L1" in names) == (k <= 32), names
        assert ("msd_partition_L1" in names) == (k > 32), names
        assert "lsd_sort(all passes)" not in names, names
    else:
        assert "lsd_sort(all passes)" in names and "leaf_count" not in names, names


# ---------------------------------------------------------------------------------------------------------------------- stage 2 at every k
SWEEP = [(k, both) for k in EVERY_K for both in (True, False)]


@pytest.mark.parametrize("k,both", SWEEP, ids=["k%d-%s" % (k, "ci" if both else "b") for k, both in SWEEP])
def test_stage2_every_k(oracle, k, both):
    """One context, two different bins one after the other: the first through process_bin, the second through dev_process_bin, whose
    result words must report no bin error and (on the MSD path) no LSD fallback."""
    p = sweep_params(k, both)
    ctx = _ctx(p)
    for i, (seed, scale) in enumerate(((7000 + 2 * k + both, 1.0), (9000 + 2 * k + both, 1.15))):
        b = sweep_bin(seed, k, scale)
        assert 150_000 <= b.n_rec <= 250_000, b.n_rec
        e = oracle.process_bin(b, p)
        if i == 0:
            _same(ctx.process_bin(_skb(b)), e)
        else:
            r, res = _dev_run(ctx, b)
            _same(r, e)
            assert res[6] == 0 and res[7] == 0, res
        assert_bin_path(ctx.stage_times()["pass_names"], k)
    ctx.close()


@pytest.mark.parametrize("k", EVERY_K)
def test_expand_every_k(oracle, k):
    """dev_expand's records (tile order = stream order) equal the oracle's expansion, in both strand modes; the unused low symbols of every
    record's last byte are random."""
    import torch
    for both in (True, False):
        p = sweep_params(k, both)
        b = synth_bin(11000 + 2 * k + both, k, 3000, genome_len=4000, pad_garbage=True)
        ctx = _ctx(p)
        d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device="cuda")
        d_bin[:b.size] = torch.from_numpy(b.data).cuda()
        d_recs = torch.zeros((b.n_rec + 8) * p.words, dtype=torch.int64, device="cuda")
        d_res = torch.zeros(8, dtype=torch.int64, device="cuda")
        ctx.dev_expand(0, d_bin.data_ptr(), b.size, b.n_rec, b.pack_bytes, d_recs.data_ptr(), d_res.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        got = d_recs.cpu().numpy().view(np.uint64)[:b.n_rec * p.words].reshape(b.n_rec, p.words)
        assert int(d_res[6]) == 0
        assert np.array_equal(got, oracle.expand(b, p)), "k=%d both=%s" % (k, both)
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------- level 2 across words
def l2_crossing_pairs():
    """Every (k, b2), b2 = 1 .. 10, k = 33 .. 128, whose level-2 digit [2k-8-b2, 2k-8) spans a multiple of 64."""
    return [(k, b2) for k in range(33, 129) for b2 in range(1, 11) if (2 * k - 8 - b2) // 64 != (2 * k - 9) // 64]


def l2_cases():
    """A seeded, fixed selection: one crossing b2 for every k mod 32 class that has one (5 .. 8) in every wide record width (2 .. 4 words),
    the strand mode alternating."""
    rng = np.random.default_rng(2027)
    pairs = l2_crossing_pairs()
    cases = []
    for words in (2, 3, 4):
        for cls in (5, 6, 7, 8):
            cand = [(k, b2) for k, b2 in pairs if (k + 31) // 32 == words and k % 32 == cls]
            k, b2 = cand[int(rng.integers(len(cand)))]
            cases.append((k, b2, len(cases) % 2 == 0))
    return cases


L2_CASES = l2_cases()


def test_level2_crossings_are_the_chosen_classes():
    pairs = l2_crossing_pairs()
    assert {k % 32 for k, _ in pairs} == {5, 6, 7, 8}
    assert {(k % 32, (k + 31) // 32) for k, _, _ in L2_CASES} == {(c, w) for c in (5, 6, 7, 8) for w in (2, 3, 4)}
    assert all((k, b2) in pairs for k, b2, _ in L2_CASES)


@pytest.mark.parametrize("k,b2,both", L2_CASES, ids=["k%d-b2_%d-%s" % (k, b2, "ci" if both else "b") for k, b2, both in L2_CASES])
def test_level2_digit_across_words(oracle, monkeypatch, k, b2, both):
    """KMCB200_L2_BITS forces the second partition level on a bin that would have none."""
    monkeypatch.setenv("KMCB200_L2_BITS", str(b2))
    p = sweep_params(k, both)
    ctx = _ctx(p)
    b = sweep_bin(13000 + k + b2, k)
    _same(ctx.process_bin(_skb(b)), oracle.process_bin(b, p))
    names = ctx.stage_times()["pass_names"]
    assert "msd_count_L2" in names and "msd_partition_L2" in names and "leaf_count" in names, names
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------------- key blocks and several contexts
# the 12-bit prefix [2k-12, 2k) of one-word records around k = 12, and of wide records where it spans two words (k mod 32 = 1 .. 5) and next to that
BLOCK_KS = [12, 13, 14] + list(range(33, 38)) + list(range(65, 70)) + list(range(97, 102)) + [128]
MAX_BLOCK = 20_000


def block_bin(k):
    """~3.6 x 10^5 k-mers at ~18x coverage."""
    return synth_bin(17000 + k, k, 30000, genome_len=20000, err=0.01)


@pytest.mark.parametrize("flow", ["scatter", "filter"])
@pytest.mark.parametrize("k", BLOCK_KS)
def test_key_blocks_every_prefix_position(oracle, monkeypatch, flow, k):
    """An oversized bin (KMCB200_MAX_BLOCK_RECORDS below its k-mers, bytes in several chunks) counted key block by key block equals the
    oracle.  Every block costs at least three launches (sort, count, accumulate): far more than the same bin in one piece."""
    p = sweep_params(k, k % 2 == 0)
    b = block_bin(k)
    e = oracle.process_bin(b, p)
    ctx = _ctx(p)
    l0 = ctx.kernel_launches()
    _same(ctx.process_bin(_skb(b)), e)
    one_piece = ctx.kernel_launches() - l0
    ctx.close()
    monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", str(MAX_BLOCK))
    monkeypatch.setenv("KMCB200_MAX_CHUNK_BYTES", str(1 << 18))
    monkeypatch.setenv("KMCB200_KEY_BLOCKS", flow)
    ctx = _ctx(p)
    l0 = ctx.kernel_launches()
    _same(ctx.process_bin(_skb(b)), e)
    blocks = ctx.kernel_launches() - l0
    ctx.close()
    assert blocks >= 3 * (b.n_rec // MAX_BLOCK) and blocks > one_piece, (blocks, one_piece)


@pytest.mark.parametrize("k", BLOCK_KS)
def test_several_contexts_every_prefix_position(oracle, monkeypatch, k):
    """process_bin_multi with two or three contexts on device 0: key ranges cut on the 12-bit prefix, every context's range in several key
    blocks; every context launches kernels of its own."""
    import kmc_b200
    p = sweep_params(k, k % 2 == 1)
    b = block_bin(k)
    monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", str(b.n_rec // 7))
    sp = kmc_b200.Stage2Params(p.k, p.both_strands, p.cutoff_min, p.cutoff_max, p.counter_max, p.lut_prefix_len)
    ctxs = [kmc_b200.Stage2Context(sp, device=0, n_slots=1) for _ in range(2 + k % 2)]
    l0 = [c.kernel_launches() for c in ctxs]
    r = kmc_b200.Stage2Context.process_bin_multi(ctxs, _skb(b))
    _same(r, oracle.process_bin(b, p))
    assert all(c.kernel_launches() > l for c, l in zip(ctxs, l0))
    for c in ctxs:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------- stage 1 and stage 0
PROFILES = {"short": (40, 150), "long": (6, 10_000), "n_dense": (60, 200), "low_complexity": (8, 3000)}
SIGNATURE_LENS = range(5, 12)


def stage1_runs():
    """(k, m, both_strands) for every k from 6 to 128, each k in both strand modes; within every k mod 32 class the signature lengths
    m < k are dealt out in turn, smallest k first, so that every m meets every class (one run more where a class has only three k)."""
    runs = []
    for c in range(32):
        slots = [(k, both) for k in range(6, 129) if k % 32 == c for both in (True, False)]
        while len(slots) < len(SIGNATURE_LENS):
            slots.append((slots[-1][0], len(slots) % 2 == 0))
        todo = []
        for k, both in slots:
            if not any(m < k for m in todo):
                todo += [m for m in SIGNATURE_LENS if m not in todo]
            m = min(m for m in todo if m < k)
            todo.remove(m)
            runs.append((k, m, both))
    return sorted(runs)


STAGE1_RUNS = stage1_runs()


def test_stage1_runs_meet_every_class():
    assert {k for k, _, _ in STAGE1_RUNS} == set(range(6, 129))
    assert all(5 <= m < k and m <= 11 for k, m, _ in STAGE1_RUNS)
    assert {(k % 32, m) for k, m, _ in STAGE1_RUNS} == {(c, m) for c in range(32) for m in SIGNATURE_LENS}
    assert {(k, both) for k, _, both in STAGE1_RUNS} == {(k, both) for k in range(6, 129) for both in (True, False)}


@pytest.mark.parametrize("k", range(6, 129))
def test_stage1_and_stage0_every_k(k):
    """Splitter with count_kxmers against the sequential oracle (bins byte for byte) and the collector's (k+x)-mer rule (max_x = 0 .. 3 by
    k mod 32); SignatureStats of the same batch against the oracle's CalcStats."""
    import kmc_b200
    from stage0_testlib import max_x_of, oracle_kxmer_totals, oracle_signature_stats
    from stage1_testlib import Stage1Oracle, batch_of, make_reads, random_map
    s1 = Stage1Oracle()
    for k_, m, both in STAGE1_RUNS:
        if k_ != k:
            continue
        seed = 1000 * k + 10 * m + both
        n_bins = (64, 512, 4096)[(k + m) % 3]
        reads = []
        for j, (prof, (n, ln)) in enumerate(PROFILES.items()):
            reads += make_reads(seed + j, prof, n_reads=n, read_len=ln)
        batch = batch_of(reads)
        sig_map = random_map(seed, m, n_bins)
        sp = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=len(batch))
        sp.count_kxmers(both)
        out, packs, frags = sp.split_raw(batch)
        fr = np.array([[f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs] for f in frags], dtype=np.uint64)
        exp = s1.split(batch, k, m, sig_map, n_bins)
        assert np.array_equal(fr, exp.frags) and out.tobytes() == exp.out.tobytes() and np.array_equal(packs, exp.pack_bytes), (k, m, both)
        kx = sp.kxmer_totals()
        assert np.array_equal(kx, oracle_kxmer_totals(exp, both)), (k, m, both)
        assert (int(kx.sum()) > 0) == bool(max_x_of(k))
        sp.close()
        st = kmc_b200.SignatureStats(k, m, max_batch_bytes=len(batch))
        st.add(batch)
        assert st.kernel_launches() == 1
        assert np.array_equal(st.read(), oracle_signature_stats(batch, k, m)), (k, m)
        st.close()
