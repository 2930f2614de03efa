"""GPU: the skewed bins of tests/test_skewed_bins_model.py through the two stage-2 flows that take the biggest bins of a real run, each
case against the oracle (payload, LUT, the four statistics):
  * key blocks (run_oversized_bin: count_top12 -> bisect_blocks -> run_key_blocks, scatter and filter -> sort_count_block), reached by
    lowering KMCB200_MAX_BLOCK_RECORDS: a dominant k-mer in a heavy leaf of a block whose prefix is not 0 (leaf_warp_kernel rebuilds its
    k-mers from leaf_prefix), poly-A / poly-T in the first and the last block, one 12-bit bucket larger than the block limit, a leaf no leaf
    kernel can count inside a later block (the LSD fallback sorts the block in its region and appends behind the earlier blocks);
  * one bin over several contexts (kmcb200_process_bin_multi): key ranges left empty by a lopsided bin, one GPU owning every block, the
    thresholds below which the bin is not split, a share of zero-byte packs, packs over 64 KiB, a malformed pack in the last share, an
    output buffer one record short;
  * the database path: an oversized bin through submit_bin + wait_bin_scanned, and count_reads on reads with poly-A tails and a satellite.
Every case shows that it took the intended path: an oversized bin launches more kernels than its one-shot run, a context whose key range
is empty launches its two expansions and no sort, an unsplit bin runs on the first context alone."""
import os

import numpy as np
import pytest

from kmc_testlib import fast_bin
from test_gpu_corners import repack
from test_skewed_bins_model import (BLOCK_LIMIT, MSD_MIN_RECORDS, MULTI_GENS, hist12, key_blocks, make_bin, multi_blocks, multi_shares,
                                    params, threshold_bin, zero_byte_share_packs)

pytestmark = pytest.mark.gpu

# kmcb200_process_bin_multi on a context with an empty key range and a share in collector packs (one chunk): the counting and the
# scattering expansion (stage_expand: init + walk, pack scan, tile table, the expansion kernel) and four zero fills (the histogram, the two
# totals, the block counters)
EMPTY_RANGE_LAUNCHES = 2 * 5 + 4


def _ctx(p, device=0, n_slots=1):
    import kmc_b200
    return kmc_b200.Stage2Context(kmc_b200.Stage2Params(p.k, p.both_strands, p.cutoff_min, p.cutoff_max, p.counter_max, p.lut_prefix_len),
                                  device=device, n_slots=n_slots)


def _skb(b):
    import kmc_b200
    return kmc_b200.SuperKmerBin(data=b.data, n_rec=b.n_rec, pack_bytes=b.pack_bytes, n_super_kmers=b.n_super_kmers, kmer_len=b.k)


def _same(r, e):
    assert r.stats == e.stats
    assert np.array_equal(r.lut, e.lut)
    assert r.payload.tobytes() == e.payload


_bins, _expected, _layout = {}, {}, {}


def skewed(gen, k, both):
    if (gen, k, both) not in _bins:
        _bins[(gen, k, both)] = make_bin(gen, k, both)[0]
    return _bins[(gen, k, both)]


def expected(oracle, key, b, p):
    """The oracle's result, kept for the other flows of the same bin and parameters."""
    pk = (key, p.k, p.both_strands, p.cutoff_min, p.cutoff_max, p.counter_max, p.lut_prefix_len)
    if pk not in _expected:
        _expected[pk] = oracle.process_bin(b, p)
    return _expected[pk]


def top12_hist(oracle, key, b, p):
    if (key, p.both_strands) not in _layout:
        _layout[(key, p.both_strands)] = hist12(oracle.expand(b, p), p.k)
    return _layout[(key, p.both_strands)]


# ---------------------------------------------------------------------------------------------------------------------- key blocks
KB_CASES = [("dominant", 31, True, {}, "hash"), ("dominant", 31, True, {}, "cta"), ("dominant", 31, False, dict(p=3, cmin=1), "hash"),
            ("dominant", 31, True, dict(cmax=30_000), "cta"), ("dominant", 31, True, dict(cmin=1, cntmax=65535), "hash"),
            ("polyat", 31, True, {}, "hash"), ("polyat", 31, False, dict(cmin=1), "cta"),
            ("one_prefix_bg", 31, True, {}, "hash"), ("one_prefix_bg", 55, True, dict(cmin=1), None),
            ("overfull", 31, True, {}, "hash"), ("overfull", 31, True, {}, "cta"), ("overfull", 31, False, dict(p=3, cmin=1), "hash"),
            ("overfull", 55, True, {}, None), ("overfull", 55, True, dict(p=3, cmin=1), None)]


def _kb_id(c):
    return "%s-k%d-%s%s-%s" % (c[0], c[1], "ci" if c[2] else "b", "".join("-%s%d" % kv for kv in sorted(c[3].items())), c[4] or "wide")


@pytest.mark.parametrize("flow", ["scatter", "filter"])
@pytest.mark.parametrize("gen,k,both,pkw,leaf", KB_CASES, ids=[_kb_id(c) for c in KB_CASES])
def test_skewed_bin_in_key_blocks(oracle, monkeypatch, flow, gen, k, both, pkw, leaf):
    """The bin once in one shot (the control), then key block by key block: the same bytes.  The block run launches at least three kernels
    per block more than the one-shot run, and its last block's leaves were counted by the leaf kernel asked for."""
    p = params(k, both, **pkw)
    b = skewed(gen, k, both)
    e = expected(oracle, (gen, k, both), b, p)
    if leaf:
        monkeypatch.setenv("KMCB200_LEAF_KERNEL", leaf)
    ctx = _ctx(p)
    l0 = ctx.kernel_launches()
    _same(ctx.process_bin(_skb(b)), e)
    one_shot = ctx.kernel_launches() - l0
    ctx.close()
    monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", str(BLOCK_LIMIT))
    monkeypatch.setenv("KMCB200_KEY_BLOCKS", flow)
    blocks = key_blocks(top12_hist(oracle, (gen, k, both), b, p), BLOCK_LIMIT)
    ctx = _ctx(p)
    l0 = ctx.kernel_launches()
    _same(ctx.process_bin(_skb(b)), e)
    launched = ctx.kernel_launches() - l0
    assert launched - one_shot >= 3 * (len(blocks) - 1), (launched, one_shot, len(blocks))
    if blocks[-1][2] >= MSD_MIN_RECORDS:
        assert ctx.leaf_plan()[1] == (leaf if k <= 32 else "wide")
    _same(ctx.process_bin(_skb(b)), e)          # again on the same context: nothing of the first run may stay behind
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------------- several contexts
def _ctxs(p, n_ctx):
    import torch
    n_dev = torch.cuda.device_count()
    return [_ctx(p, device=g % n_dev) for g in range(n_ctx)]


def _multi(ctxs, b, out=None):
    """process_bin_multi; returns (result, kernel launches of every context)."""
    import kmc_b200
    l0 = [c.kernel_launches() for c in ctxs]
    r = kmc_b200.Stage2Context.process_bin_multi(ctxs, _skb(b), out=out)
    return r, [c.kernel_launches() - x for c, x in zip(ctxs, l0)]


def assert_multi_shape(launched, per):
    """A context whose key range is empty expands its share twice (counting, scattering) and sorts nothing; every other one sorts and
    counts each of its blocks (at least three launches each) on top of that."""
    for g, blocks in enumerate(per):
        if blocks:
            assert launched[g] >= EMPTY_RANGE_LAUNCHES + 3 * len(blocks), (g, launched)
        else:
            assert launched[g] == EMPTY_RANGE_LAUNCHES, (g, launched)


MULTI_PARAMS = {("dominant", 31, True, 2): {}, ("dominant", 31, True, 3): dict(cmin=1), ("dominant", 31, True, 4): dict(cmax=30_000),
                ("dominant", 31, False, 3): dict(p=3, cmin=1), ("polyat", 31, False, 2): {}, ("lopsided", 31, True, 3): {},
                ("lopsided", 31, True, 4): dict(p=3), ("one_prefix", 31, True, 2): {}, ("one_prefix", 31, True, 4): dict(cmin=1),
                ("overfull", 31, True, 3): {}, ("overfull", 55, True, 2): dict(cmin=1)}
assert sorted(MULTI_PARAMS) == sorted(MULTI_GENS)
MULTI_CASES = [c + (MULTI_PARAMS[c],) for c in MULTI_GENS]


@pytest.mark.parametrize("gen,k,both,n_ctx,pkw", MULTI_CASES, ids=[_kb_id(c[:3] + (c[4], "%dctx" % c[3])) for c in MULTI_CASES])
def test_skewed_bin_over_several_contexts(oracle, monkeypatch, gen, k, both, n_ctx, pkw):
    """A uniform bin first, so that every context holds totals of its own range; then the skewed bin, whose key ranges may be empty (their
    totals must be zeros again) or hold a block above the limit, a heavy leaf or a leaf that takes the LSD fallback."""
    monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", str(BLOCK_LIMIT))
    p = params(k, both, **pkw)
    ctxs = _ctxs(p, n_ctx)
    warm = fast_bin(900 + k, k, 600_000)
    r, launched = _multi(ctxs, warm)
    _same(r, expected(oracle, ("warm", k), warm, p))
    assert all(launched)
    b = skewed(gen, k, both)
    r, launched = _multi(ctxs, b)
    _same(r, expected(oracle, (gen, k, both), b, p))
    per = multi_blocks(top12_hist(oracle, (gen, k, both), b, p), n_ctx, BLOCK_LIMIT)
    assert_multi_shape(launched, per)
    for c in ctxs:
        c.close()


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("what", ["n_rec", "n_packs"])
@pytest.mark.parametrize("n_ctx", [2, 3, 4])
def test_split_thresholds(oracle, n_ctx, what, split):
    """4096 n_ctx - 1 k-mers or n_ctx - 1 packs: the first context counts the bin alone; 4096 n_ctx k-mers in n_ctx packs: every context
    takes part."""
    p = params(31, True, 7, 2)
    ctxs = _ctxs(p, n_ctx)
    b = threshold_bin(n_ctx, what, split)
    r, launched = _multi(ctxs, b)
    _same(r, oracle.process_bin(b, p))
    assert launched[0] > 0 and (all(launched[1:]) if split else not any(launched[1:])), launched
    for c in ctxs:
        c.close()


@pytest.mark.parametrize("layout", ["zero_byte_share", "packs_300k", "alternating_64k_300k"])
def test_pack_layouts_over_three_contexts(oracle, monkeypatch, layout):
    """The dominant-k-mer bin over 3 contexts in packs [0.7 S, 0, 0, the rest] (the second context's share is one zero-byte pack: its
    counting and scattering expansions run on 0 bytes, its key range still holds blocks), and in packs over 64 KiB."""
    monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", str(BLOCK_LIMIT))
    p = params(31, True)
    b = skewed("dominant", 31, True)
    b = {"zero_byte_share": zero_byte_share_packs, "packs_300k": lambda x: repack(x, 300 << 10),
         "alternating_64k_300k": lambda x: repack(x, [1 << 16, 300 << 10])}[layout](b)
    if layout == "zero_byte_share":
        assert multi_shares(b.pack_bytes, 3)[1][2] == 0
    ctxs = _ctxs(p, 3)
    r, launched = _multi(ctxs, b)
    _same(r, expected(oracle, ("dominant", 31, True), b, p))
    assert_multi_shape(launched, multi_blocks(top12_hist(oracle, ("dominant", 31, True), b, p), 3, BLOCK_LIMIT))
    for c in ctxs:
        c.close()


def test_errors_over_several_contexts(oracle, monkeypatch):
    """A pack that ends 3 bytes inside a record in the last context's share: ERR_BIN_FORMAT.  An output buffer one record short:
    ERR_CAPACITY.  After each, every context still counts a bin correctly, alone and together."""
    import kmc_b200
    monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", str(BLOCK_LIMIT))
    p = params(31, True)
    b = skewed("dominant", 31, True)
    e = expected(oracle, ("dominant", 31, True), b, p)
    small = fast_bin(5, 31, 200_000)
    e_small = oracle.process_bin(small, p)
    ctxs = _ctxs(p, 3)
    pack0, n_packs, _ = multi_shares(b.pack_bytes, 3)[2]
    assert n_packs >= 2
    bad = b.pack_bytes.copy()
    bad[pack0 + n_packs // 2] -= 3
    bad[pack0 + n_packs // 2 + 1] += 3
    assert multi_shares(bad, 3)[2][:2] == (pack0, n_packs)
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        kmc_b200.Stage2Context.process_bin_multi(ctxs, kmc_b200.SuperKmerBin(data=b.data, n_rec=b.n_rec, pack_bytes=bad, kmer_len=31))
    assert ei.value.code == kmc_b200.ERR_BIN_FORMAT
    for c in ctxs:
        _same(c.process_bin(_skb(small)), e_small)
    _same(_multi(ctxs, b)[0], e)
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        _multi(ctxs, b, out=np.empty(len(e.payload) - p.out_rec_bytes, dtype=np.uint8))
    assert ei.value.code == kmc_b200.ERR_CAPACITY
    _same(_multi(ctxs, b, out=np.empty(len(e.payload), dtype=np.uint8))[0], e)
    for c in ctxs:
        _same(c.process_bin(_skb(small)), e_small)
        c.close()


# ---------------------------------------------------------------------------------------------------------------------- the database path
def test_oversized_bin_with_scanned_lut(oracle, monkeypatch):
    """submit_bin + wait_bin_scanned(slot, lut_base) on a bin above the block limit (finished inside submit_bin, its LUT prefix-summed on
    the host): the LUT is lut_base plus the exclusive prefix sum of the oracle's; the same as from a context that counts the bin in one
    shot (lut_scan_kernel).  Then a small bin through the same slot."""
    from test_gpu_corners import _submit_wait
    p = params(31, True)
    b = skewed("dominant", 31, True)
    e = expected(oracle, ("dominant", 31, True), b, p)
    small = fast_bin(6, 31, 50_000)
    e_small = oracle.process_bin(small, p)
    base = 987_654_321
    scanned = base + np.concatenate([[0], np.cumsum(e.lut)[:-1]]).astype(np.uint64)
    launched = {}
    for oversized in (False, True):
        if oversized:
            monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", str(BLOCK_LIMIT))
        ctx = _ctx(p, n_slots=2)
        l0 = ctx.kernel_launches()
        data, out, lut = _submit_wait(ctx, 1, b)
        nb, stats = ctx.wait_bin_scanned(1, base)
        launched[oversized] = ctx.kernel_launches() - l0
        assert stats == e.stats and out[:nb].tobytes() == e.payload and np.array_equal(lut, scanned)
        data, out, lut = _submit_wait(ctx, 1, small)
        nb, stats = ctx.wait_bin_scanned(1, 5)
        assert stats == e_small.stats and out[:nb].tobytes() == e_small.payload
        assert np.array_equal(lut, 5 + np.concatenate([[0], np.cumsum(e_small.lut)[:-1]]).astype(np.uint64))
        ctx.close()
    assert launched[True] > launched[False]


def _repeat_reads(seed):
    """Reads of a random genome, reads that end in poly-A (and, on the other strand, start in poly-T), and reads of a 171-base satellite
    repeat."""
    from stage1_testlib import make_reads
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    unit = acgt[rng.integers(0, 4, 171)].tobytes()
    sat = unit * 3
    genome = make_reads(seed, "short", 20000, 150, genome_len=300_000)
    poly = [r[:90] + b"A" * 60 for r in genome[:3000]] + [b"T" * 50 + r[:100] for r in genome[3000:5000]]
    return genome + poly + [sat[o:o + 150] for o in rng.integers(0, 171, 3000)]


def test_count_reads_with_key_blocks(tmp_path, monkeypatch):
    """count_reads with KMCB200_MAX_BLOCK_RECORDS lowered, so that the largest bins (poly-A, the satellite) are counted key block by key
    block inside submit_bin: .kmc_pre and .kmc_suf byte for byte those of the same call without it, and, where the reference CLI is built,
    those of kmc -sr1."""
    import kmc_b200
    from kmc_b200 import reads
    from stage1_testlib import kmc_pre_bins, write_fastq_reads
    from test_gpu_kmc_files import KMC_REF, KMC_TOOLS, count, md5
    limit = 50_000
    fq = str(tmp_path / "reads.fq")
    write_fastq_reads(fq, _repeat_reads(41))
    k, m, p = 31, 9, 7
    sig_map, n_bins, ref_db = None, None, None
    if os.path.exists(KMC_REF) and os.path.exists(KMC_TOOLS):
        ref_db, _ = count(KMC_REF, str(tmp_path), "ref", fq, k, ("-p%d" % m, "-ci2", "-sr1"))
        h, _, _, raw = kmc_pre_bins(ref_db + ".kmc_pre", ref_db + ".kmc_suf")
        m, sig_map = reads.signature_map_from_kmc_pre(ref_db + ".kmc_pre")
        p, n_bins = h["p"], raw.shape[0]
    submitted = []

    class Recording(kmc_b200.Stage2Context):
        def submit_bin(self, slot, data_ptr, size, n_rec, *a, **kw):
            submitted.append(n_rec)
            return super().submit_bin(slot, data_ptr, size, n_rec, *a, **kw)

    monkeypatch.setattr(reads, "Stage2Context", Recording)
    files = {}
    for knob in (False, True):
        if knob:
            monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", str(limit))
        out = str(tmp_path / ("db_%d" % knob))
        reads.count_reads([fq], out, k, m, sig_map, p, 2, 10 ** 9, 255, True, batch_bytes=1 << 21, n_bins=n_bins)
        files[knob] = [open(out + ext, "rb").read() for ext in (".kmc_pre", ".kmc_suf")]
    assert max(submitted) > limit
    assert files[True] == files[False]
    if ref_db:
        assert md5(str(tmp_path / "db_1.kmc_suf")) == md5(ref_db + ".kmc_suf")
        assert md5(str(tmp_path / "db_1.kmc_pre")) == md5(ref_db + ".kmc_pre")
