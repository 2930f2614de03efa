"""GPU corners: stage 2 on inputs the rest of the suite never gives it, each case byte for byte against the oracle (payload, LUT, the four
statistics).
  * pack layouts a caller may hand over: the whole bin as one pack, packs beyond 64 KiB (the warp-per-pack walker), both kinds mixed, one
    record per pack, empty packs; through every entry point (process_bin, two slots, the indexed form, dev_process_bin);
  * every record width (k = 5 .. 128, including k = 65 / 97 where the top symbols start a fresh word) against every counter width (0 .. 4
    bytes), through every leaf / sort variant, and counts that fill the third and fourth counter byte;
  * the staged device calls (dev_expand -> dev_sort(hist_ready) -> dev_count), which sort the leaves of wide records, and the knobs no
    other test sets."""
import numpy as np
import pytest

from kmc_testlib import Bin, Params, bin_extras, fast_bin, pack_superkmers, synth_bin

pytestmark = pytest.mark.gpu

WALK_CHUNK = 1 << 16          # packs up to this size are walked by walk_packs_parallel_kernel, larger ones by walk_packs_kernel


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


def _env(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


# ---------------------------------------------------------------------------------------------------------------------- bins and pack layouts
def record_sizes(b: Bin):
    """Byte length of every record of the bin, in stream order (a walk over the length bytes)."""
    d, k = bytes(b.data), b.k
    sizes, pos = [], 0
    while pos < len(d):
        n = 1 + (d[pos] + k + 3) // 4
        sizes.append(n)
        pos += n
    assert pos == len(d)
    return sizes


def with_packs(b: Bin, pack_bytes):
    packs = np.array(pack_bytes, dtype=np.uint64)
    assert packs.size == 0 or int(packs.sum()) == b.size          # (no packs: the whole bin is one pack)
    return Bin(data=b.data, n_rec=b.n_rec, n_super_kmers=b.n_super_kmers, pack_bytes=packs, pack_recs=np.zeros(packs.size, np.uint64), k=b.k)


def repack(b: Bin, target_bytes):
    """The bin's whole records regrouped into packs of at most target_bytes (a list: the targets of consecutive packs, cycled); a record
    larger than the target is a pack of its own."""
    targets = list(target_bytes) if isinstance(target_bytes, (list, tuple)) else [target_bytes]
    packs, acc = [], 0
    for s in record_sizes(b):
        if acc and acc + s > targets[len(packs) % len(targets)]:
            packs.append(acc)
            acc = 0
        acc += s
    if acc:
        packs.append(acc)
    return with_packs(b, packs)


def concat_bins(*bins):
    """One bin holding the records of several (their collector packs one after the other)."""
    return Bin(data=np.concatenate([b.data for b in bins]), n_rec=sum(b.n_rec for b in bins), n_super_kmers=sum(b.n_super_kmers for b in bins),
               pack_bytes=np.concatenate([b.pack_bytes for b in bins]).astype(np.uint64), pack_recs=np.concatenate([b.pack_recs for b in bins]).astype(np.uint64),
               k=bins[0].k)


def exact_pack_bin(k, first_pack):
    """A bin whose first pack holds exactly first_pack bytes (records of 64 bytes and one of 64 + first_pack % 64), then ~100 KB in
    collector packs."""
    rng = np.random.default_rng(first_pack)
    genome = rng.integers(0, 4, 3000)
    lens = [4 * 63 - 3] * (first_pack // 64 - 1) + [4 * (63 + first_pack % 64) - 3]          # 1 + ceil(n / 4) bytes
    lists = [genome[s:s + n] for s, n in zip(rng.integers(0, 3000 - 260, len(lens)), lens)]
    rest = [genome[s:s + n] for s, n in zip(rng.integers(0, 3000 - 260, 8000), k + rng.integers(0, 40, 8000))]
    first = pack_superkmers(k, lists)
    assert first.size == first_pack
    return with_packs(pack_superkmers(k, lists + rest), [first_pack] + [int(x) for x in pack_superkmers(k, rest).pack_bytes])


def _base_bin(k, big):
    # ~250 KB (collector packs of 64 KiB) or ~2 MB of bin bytes, 30x coverage
    n_sk = {True: 2_000_000, False: 250_000}[big] // (1 + (k + 14) // 4)
    return synth_bin(300 + k + big, k, n_sk, genome_len=n_sk * 12 // 30 + 500, err=0.01)


def layout_bin(layout, k):
    """(bin with the layout's packs, the same bin in collector packs)."""
    if layout == "whole_bin_small":            # n_packs = 0: the whole bin is one pack of < 64 KiB
        b = synth_bin(400 + k, k, 40_000 // (1 + (k + 14) // 4), genome_len=3000)
        assert b.size < WALK_CHUNK
        return with_packs(b, []), b
    if layout == "exact_65536":
        b = exact_pack_bin(k, WALK_CHUNK)
        return b, repack(b, WALK_CHUNK)
    if layout == "exact_65537":
        b = exact_pack_bin(k, WALK_CHUNK + 1)
        return b, repack(b, WALK_CHUNK)
    if layout == "one_record_per_pack":         # ~10^5 k-mers in ~3 * 10^4 packs
        b = synth_bin(500 + k, k, 30000, genome_len=5000, mean_extra=2.0)
        return with_packs(b, record_sizes(b)), b
    big = layout in ("whole_bin_2mb", "packs_1m", "packs_200k", "alternating_64k_300k", "empty_packs_big")
    b = _base_bin(k, big)
    if layout == "whole_bin_2mb":
        assert b.size > 30 * WALK_CHUNK
        return with_packs(b, []), b
    if layout == "packs_200k":
        return repack(b, 200 << 10), b
    if layout == "packs_1m":
        return repack(b, 1 << 20), b
    if layout == "alternating_64k_300k":
        return repack(b, [WALK_CHUNK, 300 << 10]), b
    if layout == "empty_packs":                 # zero-byte packs between collector packs, at the start and at the end
        pb = [int(x) for x in b.pack_bytes]
        return with_packs(b, [0] + [x for p in pb for x in (p, 0, 0)][:-1] + [0]), b
    if layout == "empty_packs_big":             # ... and between packs of 300 KiB
        pb = [int(x) for x in repack(b, 300 << 10).pack_bytes]
        return with_packs(b, [x for p in pb for x in (0, p)] + [0]), b
    raise ValueError(layout)


def big_packs(b: Bin):
    """Does the bin reach the warp walker (a pack of more than 64 KiB, or no packs and more than 64 KiB)?"""
    return int(b.pack_bytes.max()) > WALK_CHUNK if b.pack_bytes.size else b.size > WALK_CHUNK


LAYOUT_CASES = ([(lay, k) for lay in ("whole_bin_small", "whole_bin_2mb") for k in (9, 31, 128)]
                + [(lay, 31) for lay in ("packs_200k", "packs_1m", "alternating_64k_300k", "exact_65536", "exact_65537", "one_record_per_pack",
                                         "empty_packs", "empty_packs_big")]
                + [("packs_1m", 128), ("alternating_64k_300k", 55), ("one_record_per_pack", 97), ("empty_packs", 5)])
LAYOUT_P = {5: 1, 9: 5, 31: 7, 55: 7, 97: 5, 128: 8}


def _dev_run(ctx, b: Bin, pack_bytes=None):
    """kmcb200_dev_process_bin on device copies of the bin; returns (BinResult-like, the 8 result words)."""
    import torch
    import kmc_b200
    d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device="cuda")
    if b.size:
        d_bin[:b.size] = torch.from_numpy(np.ascontiguousarray(b.data)).cuda()
    cap = ctx.out_capacity(b.n_rec) + 64
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device="cuda")
    d_res = torch.zeros(8, dtype=torch.int64, device="cuda")
    packs = b.pack_bytes if pack_bytes is None else pack_bytes
    ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, b.n_rec, packs, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    res = [int(x) for x in d_res.cpu().numpy().view(np.uint64)]
    r = kmc_b200.BinResult(d_out[:res[4] * ctx.out_rec_bytes].cpu().numpy(), d_lut.cpu().numpy().view(np.uint64), *res[:4])
    return r, res


def _submit_wait(ctx, slot, b: Bin, pack_bytes=None, indexed=False):
    """submit_bin (or submit_bin_indexed) into `slot`; returns (out, lut) - the caller waits."""
    data = np.ascontiguousarray(b.data)
    packs = np.ascontiguousarray(b.pack_bytes if pack_bytes is None else pack_bytes, dtype=np.uint64)
    out = np.zeros(ctx.out_capacity(b.n_rec) + 64, dtype=np.uint8)
    lut = np.zeros(ctx.lut_entries, dtype=np.uint64)
    if indexed:
        if packs.size == 0:
            packs = np.array([b.size], dtype=np.uint64)           # (the indexed form takes no empty pack list: one pack holding the whole bin)
        extras, psk = bin_extras(with_packs(b, packs))
        ctx.submit_bin_indexed(slot, data.ctypes.data, data.size, b.n_rec, packs, extras, psk, out.ctypes.data, out.size, lut.ctypes.data)
    else:
        ctx.submit_bin(slot, data.ctypes.data, data.size, b.n_rec, packs, out.ctypes.data, out.size, lut.ctypes.data)
    return data, out, lut


@pytest.mark.parametrize("path", ["process_bin", "two_slots", "indexed", "dev"])
@pytest.mark.parametrize("layout,k", LAYOUT_CASES, ids=["%s-k%d" % c for c in LAYOUT_CASES])
def test_pack_layouts(oracle, layout, k, path):
    """Caller-made pack layouts through every entry point.  Where the layout takes the warp-per-pack walker, process_bin launches exactly
    one kernel more than for the same bin in collector packs."""
    b, collector = layout_bin(layout, k)
    p = Params(k=k, cutoff_min=2 if k > 20 else 1, lut_prefix_len=LAYOUT_P[k])
    e = oracle.process_bin(b, p)
    if path == "process_bin":
        ref_ctx = _ctx(p)
        l0 = ref_ctx.kernel_launches()
        _same(ref_ctx.process_bin(_skb(collector)), e)
        l_collector = ref_ctx.kernel_launches() - l0
        l0 = ref_ctx.kernel_launches()
        _same(ref_ctx.process_bin(_skb(b)), e)
        l_layout = ref_ctx.kernel_launches() - l0
        assert l_layout - l_collector == (1 if big_packs(b) else 0)
        ref_ctx.close()
        return
    ctx = _ctx(p, n_slots=2)
    if path == "two_slots":              # the layout in slot 1 while slot 0 holds the same bin in collector packs
        d0, out0, lut0 = _submit_wait(ctx, 0, collector)
        d1, out1, lut1 = _submit_wait(ctx, 1, b)
        for slot, out, lut in ((1, out1, lut1), (0, out0, lut0)):
            nb, stats = ctx.wait_bin(slot)
            assert stats == e.stats and out[:nb].tobytes() == e.payload and np.array_equal(lut, e.lut)
    elif path == "indexed":
        d, out, lut = _submit_wait(ctx, 0, b, indexed=True)
        nb, stats = ctx.wait_bin(0)
        assert stats == e.stats and out[:nb].tobytes() == e.payload and np.array_equal(lut, e.lut)
        if b.pack_bytes.size > 1:          # and one pack holding the whole bin
            d, out, lut = _submit_wait(ctx, 1, b, pack_bytes=np.array([b.size], dtype=np.uint64), indexed=True)
            nb, stats = ctx.wait_bin(1)
            assert stats == e.stats and out[:nb].tobytes() == e.payload and np.array_equal(lut, e.lut)
    else:
        r, res = _dev_run(ctx, b)
        assert res[6] == 0
        _same(r, e)
    ctx.close()


def test_big_pack_ending_inside_a_record_is_a_format_error(oracle):
    """A pack of 300 KiB that ends 3 bytes before its last record does (the next one starts there): the warp walker finds pos != end.
    The context then still counts a good bin - in big packs and in collector packs - correctly."""
    import kmc_b200
    k = 31
    p = Params(k=k, cutoff_min=2, lut_prefix_len=7)
    good, collector = layout_bin("alternating_64k_300k", k)
    bad = repack(collector, 300 << 10).pack_bytes.copy()
    bad[0] -= 3
    bad[1] += 3
    ctx = _ctx(p)
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        ctx.process_bin(_skb(with_packs(collector, bad)))
    assert ei.value.code == kmc_b200.ERR_BIN_FORMAT
    r, res = _dev_run(ctx, collector, pack_bytes=bad)
    assert res[6] != 0
    e = oracle.process_bin(good, p)
    _same(ctx.process_bin(_skb(good)), e)
    _same(ctx.process_bin(_skb(collector)), e)
    ctx.close()


@pytest.mark.parametrize("flow", ["scatter", "filter"])
@pytest.mark.parametrize("target", [300 << 10, 1 << 20, [WALK_CHUNK, 300 << 10]], ids=["300k", "1m", "alternating"])
def test_oversized_bin_in_big_packs(oracle, monkeypatch, flow, target):
    """An oversized bin (counted key block by key block) in caller-made packs of more than 64 KiB: the counting, scattering and filtering
    expansions walk them with the warp walker.  Without packs the bin cannot be cut into chunks: ERR_INVALID, and the context stays usable."""
    import kmc_b200
    monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", "150000")
    monkeypatch.setenv("KMCB200_MAX_CHUNK_BYTES", str(1 << 21))
    monkeypatch.setenv("KMCB200_KEY_BLOCKS", flow)
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    b = fast_bin(31337, 31, 1_300_000)
    e = oracle.process_bin(b, p)
    ctx = _ctx(p)
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        ctx.process_bin(_skb(with_packs(b, [])))
    assert ei.value.code == kmc_b200.ERR_INVALID
    _same(ctx.process_bin(_skb(repack(b, target))), e)
    _same(ctx.process_bin(_skb(b)), e)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------------- record x counter width
K_P = {5: 1, 8: 4, 12: 4, 31: 7, 32: 4, 33: 5, 55: 7, 64: 8, 65: 5, 96: 8, 97: 5, 127: 11, 128: 8}
WIDTHS = {"cw0": (1, 10 ** 9), "cw1": (255, 10 ** 9), "cw2": (65535, 10 ** 9), "cw3": (2 ** 24 - 1, 10 ** 9), "cw4": (2 ** 32 - 1, 10 ** 9),
          "cw1_by_cutoff_max": (2 ** 32 - 1, 200)}          # (counter_max, cutoff_max)
KERNELS = {"default": {}, "lsd": {"KMCB200_SORT": "lsd"}}


def width_matrix():
    """A fixed, seeded selection of (kernel, k, counter width, both_strands): every kernel meets every k once and every width at least twice.
    The rows drawn second and third belonged to retired leaf paths.  They are still drawn, so that the other kernels' rows stay what they
    were, and the oracle's corner test (test_oracle_golden) still takes their combinations."""
    rng = np.random.default_rng(2026)
    names = list(WIDTHS)
    cases = []
    for kern in ("default", "retired", "leaf_sort", "lsd"):
        off = int(rng.integers(len(names)))
        for i, k in enumerate(rng.permutation(list(K_P))):
            cases.append((kern, int(k), names[(i + off) % len(names)], bool(rng.integers(2))))
    return cases


WIDTH_CASES = [c for c in width_matrix() if c[0] in KERNELS]


def width_params(k, width, both, p_len=None):
    cntmax, cmax = WIDTHS[width]
    return Params(k=k, both_strands=both, cutoff_min=1, cutoff_max=cmax, counter_max=cntmax, lut_prefix_len=K_P[k] if p_len is None else p_len)


def width_bin(seed, k, scale=1.0):
    """~1.7 x 10^5 k-mers (the hybrid sort and the leaf kernels for k >= 12): a 30x part plus a part where k-mers occur ~2000 times
    (counts beyond one byte, clamped by counter_max = 255 and above cutoff_max = 200)."""
    n1, n2 = int(6000 * scale), int(8000 * scale)
    return concat_bins(synth_bin(seed, k, n1, genome_len=2500, err=0.01), synth_bin(seed + 1, k, n2, genome_len=k + 45, max_extra=20, err=0.0))


@pytest.mark.parametrize("kern,k,width,both", WIDTH_CASES, ids=["%s-k%d-%s-%s" % (c[0], c[1], c[2], "ci" if c[3] else "b") for c in WIDTH_CASES])
def test_record_and_counter_widths(oracle, monkeypatch, kern, k, width, both):
    """One context, two different bins one after the other: stale bytes of the first in the leaves' padded records or the output buffer
    would show in the second."""
    _env(monkeypatch, KERNELS[kern])
    p = width_params(k, width, both)
    assert p.counter_bytes == {"cw0": 0, "cw1": 1, "cw2": 2, "cw3": 3, "cw4": 4, "cw1_by_cutoff_max": 1}[width]
    ctx = _ctx(p)
    for seed, scale in ((k, 1.0), (k + 1000, 0.6)):
        b = width_bin(seed, k, scale)
        _same(ctx.process_bin(_skb(b)), oracle.process_bin(b, p))
    ctx.close()


def test_prefix_15_with_wide_records(oracle):
    """p = 15 (a LUT of 4^15 entries, 8 GiB) with 4-word records and 2-byte counters; two bins on one context."""
    p = Params(k=127, both_strands=True, cutoff_min=1, counter_max=65535, lut_prefix_len=15)
    ctx = _ctx(p)
    lut = np.empty(ctx.lut_entries, dtype=np.uint64)
    for seed, scale in ((15, 1.0), (16, 0.5)):
        b = width_bin(seed, 127, scale)
        r = ctx.process_bin(_skb(b), lut=lut)
        e = oracle.process_bin(b, p)
        assert r.stats == e.stats and r.payload.tobytes() == e.payload and np.array_equal(r.lut, e.lut)
        del e
    ctx.close()


def _dominant_bin(k, copies, seed):
    """`copies` records of exactly one k-mer (plus its reverse complement half the time) among 4000 random super-k-mers."""
    rng = np.random.default_rng(seed)
    one = rng.integers(0, 4, k).astype(np.uint8)
    rc = (3 - one[::-1]).astype(np.uint8)
    lists = [one if i % 2 else rc for i in range(copies)] + [rng.integers(0, 4, k + 60) for _ in range(4000)]
    return pack_superkmers(k, lists)


@pytest.mark.parametrize("kern", ["default", "lsd"])
@pytest.mark.parametrize("k,copies,cntmax,fallback", [(31, 300_000, 2 ** 24 - 1, 0), (31, 300_000, 100_000, 0), (55, 100_000, 2 ** 24 - 1, 1), (65, 100_000, 70_000, 1)])
def test_counts_in_the_third_counter_byte(oracle, monkeypatch, kern, k, copies, cntmax, fallback):
    """A k-mer with 10^5 .. 3 x 10^5 copies and 3-byte counters, unclamped or clamped between 2^16 and the count.  One-word records count it
    inside the leaf kernel (dominant-k-mer path, result[7] = 0); wider leaves of more than 65534 records take the LSD fallback (result[7] = 1)."""
    _env(monkeypatch, KERNELS[kern])
    p = Params(k=k, both_strands=True, cutoff_min=1, counter_max=cntmax, lut_prefix_len=K_P[k])
    assert p.counter_bytes == 3
    b = _dominant_bin(k, copies, 7 + k)
    e = oracle.process_bin(b, p)
    assert max(int.from_bytes(e.payload[i + p.out_rec_bytes - 3:i + p.out_rec_bytes], "little") for i in range(0, len(e.payload), p.out_rec_bytes)) >= 1 << 16
    ctx = _ctx(p)
    _same(ctx.process_bin(_skb(b)), e)
    r, res = _dev_run(ctx, b)
    _same(r, e)
    if kern == "default":
        assert res[7] == fallback
    ctx.close()


@pytest.mark.parametrize("cntmax", [2 ** 32 - 1, 2 ** 24 + 5])
def test_counts_in_the_fourth_counter_byte(oracle, cntmax):
    """Poly-A super-k-mers of k + 255 symbols: one k-mer with more than 2^24 copies, 4-byte counters (unclamped / clamped just above 2^24).
    Its leaf is beyond what the leaf kernel streams (kLwMaxHeavyLeaf): the LSD fallback sorts the bin and count_emit_kernel writes it."""
    k = 31
    rng = np.random.default_rng(24)
    lists = [np.zeros(k + 255, dtype=np.uint8)] * 65600 + [rng.integers(0, 4, k + 80) for _ in range(3000)]
    b = pack_superkmers(k, lists)
    p = Params(k=k, both_strands=True, cutoff_min=1, counter_max=cntmax, lut_prefix_len=7)
    assert p.counter_bytes == 4
    e = oracle.process_bin(b, p)
    assert e.payload[p.out_rec_bytes - 1] == 1                      # the poly-A k-mer sorts first; its count's fourth byte is 1
    ctx = _ctx(p)
    _same(ctx.process_bin(_skb(b)), e)
    r, res = _dev_run(ctx, b)
    _same(r, e)
    assert res[7] == 1
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------------- staged device calls
STAGED_CASES = [(n, k) for n in (20_000, 150_000) for k in (9, 31, 55, 128)] + [(150_000, k) for k in (33, 65, 97)]


@pytest.mark.parametrize("n,k", STAGED_CASES, ids=["index-n%d-k%d" % c for c in STAGED_CASES])
def test_staged_device_calls(oracle, n, k):
    """dev_expand -> dev_sort(hist_ready=True) -> dev_count: the sort takes the level-1 cells the expansion left (per expand tile); below
    2^16 records or k < 12 it is the plain LSD sort on the ZeroBlock the expansion zeroed.  The sorted records must be where dev_sort's
    return value says.  Records of 2..4 words take msd_local_sort_kernel on key_bits = 2k (not a multiple of 8), including k = 33 / 65 /
    97 where the top symbol starts a fresh word."""
    import torch
    p = Params(k=k, both_strands=True, cutoff_min=2, lut_prefix_len=LAYOUT_P[k] if k in LAYOUT_P else K_P[k])
    b = fast_bin(4000 + k + n, k, n)
    exp_sorted = oracle.sort(oracle.expand(b, p), (k + 3) // 4)
    exp = oracle.compact(exp_sorted, p)
    e = oracle.process_bin(b, p)
    assert exp.stats == e.stats and exp.payload == e.payload
    ctx = _ctx(p)
    st = torch.cuda.current_stream().cuda_stream
    d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device="cuda")
    d_bin[:b.size] = torch.from_numpy(b.data).cuda()
    w = p.words
    for rep in range(2):              # twice: the second chain must not see the first one's state
        d_recs = torch.zeros((n + 8) * w, dtype=torch.int64, device="cuda")
        d_tmp = torch.zeros((n + 8) * w, dtype=torch.int64, device="cuda")
        d_res = torch.zeros(8, dtype=torch.int64, device="cuda")
        ctx.dev_expand(0, d_bin.data_ptr(), b.size, n, b.pack_bytes, d_recs.data_ptr(), d_res.data_ptr(), st)
        where = ctx.dev_sort(0, d_recs.data_ptr(), d_tmp.data_ptr(), n, hist_ready=True, stream=st)
        assert where in (0, 1)
        srt = d_tmp if where == 1 else d_recs
        torch.cuda.synchronize()
        assert int(d_res[6]) == 0
        got = srt.cpu().numpy().view(np.uint64)[:n * w].reshape(n, w)
        assert np.array_equal(got, exp_sorted), "records not sorted in the buffer dev_sort named (%d)" % where
        cap = ctx.out_capacity(n) + 64
        d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device="cuda")
        d_res2 = torch.zeros(8, dtype=torch.int64, device="cuda")
        ctx.dev_count(0, srt.data_ptr(), n, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res2.data_ptr(), st)
        torch.cuda.synchronize()
        res = [int(x) for x in d_res2.cpu().numpy()]
        assert tuple(res[:4]) == exp.stats
        assert d_out[:res[4] * ctx.out_rec_bytes].cpu().numpy().tobytes() == exp.payload
        assert np.array_equal(d_lut.cpu().numpy().view(np.uint64), exp.lut)
        names = ctx.stage_times()["pass_names"]
        hybrid = n >= 1 << 16 and 2 * k >= 24
        assert ("msd_local_sort" in names) == hybrid and (("lsd_sort(all passes)" in names) != hybrid)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------------- knobs
def test_pipelined_slots_with_overlapped_walk(oracle):
    """The index kernels of a submitted bin run on its slot's copy stream, next to the kernels of the bin before it on the compute stream;
    bins of different sizes and pack layouts through two slots (submit / wait), buffers reused and regrown."""
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    ctx = _ctx(p, n_slots=2)
    bins = [synth_bin(100 + i, 31, n, genome_len=max(2000, n), err=0.01) for i, n in enumerate([3000, 50, 40000, 0, 7000, 1, 20000])]
    bins[2] = repack(bins[2], 300 << 10)
    bins[6] = with_packs(bins[6], [])
    pending = {}                  # slot -> (bin index, host buffers of the bin in flight: data, out, lut)
    res = [None] * len(bins)
    for i, b in enumerate(bins):
        slot = i % 2
        if slot in pending:
            j, (_, out, lut) = pending.pop(slot)
            res[j] = (ctx.wait_bin(slot), out, lut)
        pending[slot] = (i, _submit_wait(ctx, slot, b))
    for slot, (j, (_, out, lut)) in sorted(pending.items(), key=lambda x: x[1][0]):
        res[j] = (ctx.wait_bin(slot), out, lut)
    for b, ((nb, stats), out, lut) in zip(bins, res):
        e = oracle.process_bin(b, p)
        assert stats == e.stats and out[:nb].tobytes() == e.payload and np.array_equal(lut, e.lut)
    ctx.close()


def test_key_block_records(oracle, monkeypatch):
    """KMCB200_KEY_BLOCK_RECORDS: 1024 plans far more than 512 blocks for one scattering expansion, so the host bisects again with the block
    limit (the same blocks, hence the same launches, as without the knob); 20000 gives 65 or more small scattered blocks instead of <= 16,
    each with at least three launches of its own (sort, count, accumulate)."""
    monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", "150000")
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    b = fast_bin(2718, 31, 1_300_000)
    e = oracle.process_bin(b, p)
    launches = {}
    for kbr in (None, "1024", "20000"):
        if kbr:
            monkeypatch.setenv("KMCB200_KEY_BLOCK_RECORDS", kbr)
        ctx = _ctx(p)
        l0 = ctx.kernel_launches()
        _same(ctx.process_bin(_skb(b)), e)
        launches[kbr] = ctx.kernel_launches() - l0
        ctx.close()
    assert launches["1024"] == launches[None]
    assert launches["20000"] - launches[None] >= 3 * 40
