"""Stage 2 at the sizes it runs at, every case against the oracle (payload, LUT, the four statistics):
  * the benchmark's own bins: the 2^28-k-mer pool bin bench.py times and the 96 Mi one, through dev_process_bin on a non-default stream
    with the bin resident in HBM (as bench.py counts them) and through process_bin, against one oracle run on the whole bin;
  * one sort near the context's block limit (0.6 x free HBM / bytes per record): a k = 31 bin of ~1.5e9 k-mers whose payload passes
    4 GiB, counted in one shot at the default limits, then in key blocks of ~5e8 records (filter) and of the default 2^28 (scatter);
  * a k = 128 bin of 4 GiB or more (size >= 4 x the default 1 GiB expansion chunk): key blocks by bytes, through process_bin and through
    submit_bin + wait_bin_scanned on two slots;
  * LUT offsets past 2^32: wait_bin_scanned with lut_base above 2^32, one shot and in key blocks.
A plain oracle run on a 1.5e9-k-mer bin would take minutes, so those expected outputs are built from oracle runs on the bin's pieces:
a composite bin repeats pieces (r copies of piece i), and a k-mer's count in it is sum(r_i c_i) over the pieces that hold it, merged
exactly in numpy.  Each case reads the free HBM and the host's MemAvailable first and skips, naming both, when it cannot reach its size."""
import math
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from kmc_testlib import (Bin, Params, brute_force_counts, emit_rows, expected_from_arrays, expected_from_counts, fast_bin, raw_counts,
                         raw_rows)
from test_skewed_bins_model import key_blocks

GiB = 1 << 30
PIECE = 1 << 24                    # k-mers per piece of the composite bins
THREADS = max(1, min(16, os.cpu_count() or 1))


# ---------------------------------------------------------------------------------------------------------------------- budgets
def per_record_bytes(k, p: Params):
    """kmcb200_create's HBM per record of one sort: two record buffers, the leaves' 8-byte padded output, ~2 bytes of tables."""
    words = (k + 31) // 32
    return 2 * 8 * words + ((((k - p.lut_prefix_len) // 4) + p.counter_bytes + 7) // 8) * 8 + 2


def block_limit(free, k, p: Params, n_slots=1):
    """The context's max_block_records for `free` bytes of free HBM: the largest bin it counts in one sort."""
    fit = int(0.6 * free) // per_record_bytes(k, p) // n_slots
    return max(1 << 24, min(fit, (1 << 32) - (1 << 24)))


def free_hbm():
    import torch
    torch.cuda.empty_cache()
    return int(torch.cuda.mem_get_info(0)[0])


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def need_host(nbytes, what):
    have = mem_available()
    if have < nbytes:
        pytest.skip("%s needs %.1f GB of host memory, MemAvailable is %.1f GB" % (what, nbytes / 1e9, have / 1e9))


def need_hbm(nbytes, free, what):
    if free < nbytes:
        pytest.skip("%s needs %.1f GB of free HBM, %.1f GB are free" % (what, nbytes / 1e9, free / 1e9))


def slot_bytes(size, n_rec, p: Params, out_capacity):
    """What one slot allocates for a bin (kSlotSlack: an eighth more than it needs)."""
    return int(1.125 * (size + out_capacity + n_rec * per_record_bytes(p.k, p))) + (256 << 20)


def _ctx(p: Params, n_slots=1):
    import kmc_b200
    return kmc_b200.Stage2Context(kmc_b200.Stage2Params(p.k, p.both_strands, p.cutoff_min, p.cutoff_max, p.counter_max, p.lut_prefix_len),
                                  n_slots=n_slots)


def _skb(b: Bin):
    import kmc_b200
    return kmc_b200.SuperKmerBin(data=b.data, n_rec=b.n_rec, pack_bytes=b.pack_bytes, n_super_kmers=b.n_super_kmers, kmer_len=b.k)


def _report(name, **kv):
    print("\n[%s] %s" % (name, " ".join("%s=%s" % (k, v) for k, v in kv.items())))


# ---------------------------------------------------------------------------------------------------------------------- composite bins
def composite_bin(parts):
    """parts: [(Bin, r)] -> one bin holding r copies of every piece, packs and all (a pack never straddles two pieces)."""
    k = parts[0][0].k
    rep = [b for b, r in parts for _ in range(r)]
    return Bin(data=np.concatenate([b.data for b in rep]), n_rec=sum(b.n_rec for b in rep), n_super_kmers=sum(b.n_super_kmers for b in rep),
               pack_bytes=np.concatenate([b.pack_bytes for b in rep]), pack_recs=np.concatenate([b.pack_recs for b in rep]), k=k)


def merge_counts(parts):
    """parts: [(keys ascending, counts, r)] -> (distinct keys ascending, sum of r * count per key)."""
    keys = np.concatenate([kk for kk, _, _ in parts])
    counts = np.concatenate([c * np.uint64(r) for _, c, r in parts])
    order = np.argsort(keys, kind="stable")
    keys, counts = keys[order], counts[order]
    if keys.size == 0:
        return keys, counts
    start = np.flatnonzero(np.concatenate([[True], keys[1:] != keys[:-1]]))
    return keys[start], np.add.reduceat(counts, start)


def composite_expected(parts, p: Params, pool, n_ranges=64):
    """The expected output of a composite bin, merged range by range of the key space in parallel: (payload chunks in key order, lut,
    stats, top-12-bit histogram of its k-mers)."""
    big = max((kk for kk, _, _ in parts), key=lambda a: a.size)
    edges = np.unique(np.concatenate([[0], big[(np.arange(1, n_ranges) * big.size) // n_ranges]])).astype(np.uint64)
    cuts = [np.concatenate([np.searchsorted(kk, edges, side="left"), [kk.size]]) for kk, _, _ in parts]

    def one(i):
        keys, counts = merge_counts([(kk[c[i]:c[i + 1]], cc[c[i]:c[i + 1]], r) for (kk, cc, r), c in zip(parts, cuts)])
        hist = np.bincount((keys >> np.uint64(2 * p.k - 12)).astype(np.int64), weights=counts.astype(np.float64), minlength=4096)
        return expected_from_arrays(keys, counts, p), hist

    res = list(pool.map(one, range(edges.size)))
    lut = np.sum([e[1] for e, _ in res], axis=0).astype(np.uint64)
    stats = tuple(int(sum(e[2][j] for e, _ in res)) for j in range(4))
    hist = np.rint(np.sum([h for _, h in res], axis=0)).astype(np.int64)
    return [e[0] for e, _ in res], lut, stats, hist


def scaled_expected(oracle, piece: Bin, r, p: Params):
    """The expected output of r copies of one bin at any k: the oracle's raw rows with every counter times r, then the cutoffs."""
    suffix, prefixes, counts = raw_rows(oracle, piece, p.both_strands, p.lut_prefix_len)
    return emit_rows(suffix, prefixes, counts * np.uint64(r), p)


def same_chunks(payload, chunks):
    """payload (uint8 array) is the concatenation of chunks (bytes)."""
    assert payload.size == sum(len(c) for c in chunks), (payload.size, sum(len(c) for c in chunks))
    off = 0
    for i, c in enumerate(chunks):
        assert np.array_equal(payload[off:off + len(c)], np.frombuffer(c, dtype=np.uint8)), "payload differs in key range %d" % i
        off += len(c)


# ---------------------------------------------------------------------------------------------------------------------- the helpers, without a GPU
@pytest.mark.parametrize("prm", [Params(31, True, 2, 1_000_000_000, 255, 7), Params(31, False, 1, 6, 4, 3), Params(19, True, 3, 70_000, 300, 11),
                                 Params(15, True, 1, 2 ** 32 - 1, 2 ** 32 - 1, 3), Params(23, True, 2, 70_000, 70_000, 7)],
                         ids=["k31-ci2-cs255", "k31-b-cx6-cs4", "k19-2byte", "k15-4byte", "k23-3byte"])
def test_expected_from_arrays_equals_expected_from_counts(prm):
    """The vectorised expected output equals the loop over a dict of counts, with k-mers cut by both cutoffs and counters clamped."""
    b = fast_bin(11, prm.k, 4000, genome_len=600)
    b = composite_bin([(b, 3), (fast_bin(12, prm.k, 3000, genome_len=20_000), 1)])
    cnt = brute_force_counts(b, prm)
    keys = np.array(sorted(cnt), dtype=np.uint64)
    counts = np.array([cnt[int(x)] for x in keys], dtype=np.uint64)
    payload, lut, stats = expected_from_arrays(keys, counts, prm)
    e_payload, e_lut, e_stats = expected_from_counts(cnt, prm)
    assert stats == e_stats and np.array_equal(lut, e_lut) and payload == e_payload
    assert stats[1] + stats[2] > 0 or prm.cutoff_min == 1


def test_composite_expected_equals_oracle_on_the_whole_bin(oracle):
    """Raw counts of the pieces, merged with their multiplicities range by range, give what the oracle computes on the composite bin."""
    prm = Params(31, True, 2, 40, 30, 7)
    pieces = [(fast_bin(21, 31, 200_000), 3), (fast_bin(22, 31, 150_000, genome_len=600_000, err_ppm=0), 1),
              (fast_bin(23, 31, 100_000), 2), (fast_bin(21, 31, 200_000), 1)]          # the same piece twice: keys shared across parts
    parts = [raw_counts(oracle, b, True, prm.lut_prefix_len) + (r,) for b, r in pieces]
    whole = composite_bin(pieces)
    e = oracle.process_bin(whole, prm)
    with ThreadPoolExecutor(4) as pool:
        chunks, lut, stats, hist = composite_expected(parts, prm, pool, n_ranges=7)
    assert len(chunks) == 7
    assert stats == e.stats and np.array_equal(lut, e.lut) and b"".join(chunks) == e.payload
    assert int(hist.sum()) == whole.n_rec and stats[1] > 0 and stats[2] > 0


def test_scaled_expected_equals_oracle_at_k128(oracle):
    """r copies of one k = 128 bin: the oracle's raw rows scaled by r equal the oracle on the repeated bin, cutoffs included."""
    piece = fast_bin(31, 128, 20_000, mean_extra=0.3, genome_len=2_000)
    for r, prm in ((3, Params(128, True, 7, 60, 50, 8)), (2, Params(128, False, 2, 255, 255, 4))):
        e = oracle.process_bin(composite_bin([(piece, r)]), prm)
        payload, lut, stats = scaled_expected(oracle, piece, r, prm)
        assert stats == e.stats and np.array_equal(lut, e.lut) and payload == e.payload


# ---------------------------------------------------------------------------------------------------------------------- 1. the benchmark's bins
@pytest.mark.gpu
@pytest.mark.parametrize("pool_index", [0, 5])
def test_bench_pool_bin_vs_oracle(oracle, pool_index):
    """bench.py's pool bin (seed 4000 + index) with bench's parameters, counted as bench.py counts it (dev_process_bin on a non-default
    stream, the bin resident in HBM, a context of E2E_SLOTS slots) and through process_bin: both equal one oracle run on the whole bin."""
    import torch
    import bench
    t0 = time.time()
    n = bench.pool_sizes(1)[pool_index]
    prm = Params(bench.K, True, bench.CUTOFF_MIN, bench.CUTOFF_MAX, bench.COUNTER_MAX, bench.LUT_P)
    need_host(int(n * 24) + 2 * GiB, "the %d-k-mer bench bin and its oracle run" % n)
    with ThreadPoolExecutor(THREADS) as pool:
        b = bench.gen_bin(4000 + pool_index, bench.K, n, pool)
    free = free_hbm()
    ctx_cap = prm.out_capacity(n) + 64
    need = max(slot_bytes(b.size, n, prm, ctx_cap), math.ceil(n * per_record_bytes(prm.k, prm) * bench.E2E_SLOTS / 0.6))
    need_hbm(need, free, "the %d-k-mer bench bin in one sort on a %d-slot context" % (n, bench.E2E_SLOTS))
    with ThreadPoolExecutor(1) as one:
        fut = one.submit(oracle.process_bin, b, prm)          # (ctypes releases the GIL: the GPU runs meanwhile)
        ctx = _ctx(prm, n_slots=bench.E2E_SLOTS)
        cap = ctx.out_capacity(n) + 64
        dev = torch.device("cuda", 0)
        d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device=dev)
        d_bin[:b.size] = torch.from_numpy(b.data).to(dev)
        d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
        d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device=dev)
        d_res = torch.zeros(8, dtype=torch.int64, device=dev)
        stream = torch.cuda.Stream(device=dev)
        assert stream.cuda_stream != 0
        torch.cuda.synchronize()
        ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, b.n_rec, b.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(),
                            stream.cuda_stream)
        stream.synchronize()
        res = [int(x) for x in d_res.cpu().numpy().view(np.uint64)]
        dev_payload = d_out[:res[4] * ctx.out_rec_bytes].cpu().numpy()
        dev_lut = d_lut.cpu().numpy().view(np.uint64).copy()
        del d_bin, d_out, d_lut, d_res
        r = ctx.process_bin(_skb(b))
        ctx.close()
        torch.cuda.empty_cache()
        e = fut.result()
    assert res[5] == 0 and res[6] == 0, res
    assert tuple(res[:4]) == e.stats
    assert np.array_equal(dev_lut, e.lut)
    assert dev_payload.tobytes() == e.payload
    assert r.stats == e.stats and np.array_equal(r.lut, e.lut) and r.payload.tobytes() == e.payload
    _report("bench bin %d" % pool_index, n=n, bin_bytes=b.size, payload_bytes=len(e.payload), path="one sort",
            free_hbm_gb="%.1f" % (free / 1e9), wall_s="%.1f" % (time.time() - t0))


# ---------------------------------------------------------------------------------------------------------------------- 2. one sort near the limit
DISTINCT_PIECES = 38               # ~1.48e7 distinct k-mers each: with ci = 1 more than 2^32 / 8 records are emitted
MULTIPLICITIES = (20, 13, 11, 7, 5, 3, 2, 1)
TARGET_KMERS = 1_500_000_000


def near_limit_units(n_max):
    """How many 2^24-k-mer units fit below n_max, and the multiplicities of the 30x pieces that fill what the distinct pieces leave."""
    units = n_max // PIECE
    left, mults = units - DISTINCT_PIECES, []
    for m in MULTIPLICITIES:
        if m <= left:
            mults.append(m)
            left -= m
    return units, mults


def test_near_limit_composition():
    """The composite bin below on an empty card: ~1.5e9 k-mers, more than 2^30, 38 all-distinct pieces and 30x pieces at 20, 13, 11, 7."""
    units, mults = near_limit_units(TARGET_KMERS)
    assert units * PIECE <= TARGET_KMERS < (units + 1) * PIECE
    assert mults == [20, 13, 11, 7] and units * PIECE > 2 ** 30


@pytest.mark.gpu
def test_one_sort_near_the_block_limit_payload_past_4gib(oracle, monkeypatch):
    """A k = 31 bin of up to 1.5e9 k-mers (at most 0.85 x the context's block limit), ci = 1, 2-byte counters: more than 2^30 k-mers in one
    sort and more than 4 GiB of payload.  Then the same bin in key blocks: filter with KMCB200_MAX_BLOCK_RECORDS = n / 3, and scatter with
    the same limit and the default 2^28-record preferred block.  Every run gives the expected bytes."""
    import torch
    t0 = time.time()
    prm = Params(31, True, 1, 1_000_000_000, 65535, 7)
    for v in ("KMCB200_MAX_BLOCK_RECORDS", "KMCB200_KEY_BLOCKS", "KMCB200_KEY_BLOCK_RECORDS", "KMCB200_MAX_CHUNK_BYTES"):
        monkeypatch.delenv(v, raising=False)
    free = free_hbm()
    limit = block_limit(free, 31, prm)
    units, mults = near_limit_units(min(TARGET_KMERS, int(0.85 * limit)))
    if sum(mults) + DISTINCT_PIECES <= 2 ** 30 // PIECE:
        pytest.skip("more than 2^30 k-mers in one sort need %.1f GB of free HBM, %.1f GB are free"
                    % ((2 ** 30 + PIECE) * per_record_bytes(31, prm) / 0.6 / 0.85 / 1e9, free / 1e9))
    need_host(28 * GiB, "the %d-unit composite bin, its expected output and its results" % units)

    specs = [(("distinct", 5000 + i), 1) for i in range(DISTINCT_PIECES)] + [(("30x", 6000 + i), m) for i, m in enumerate(mults)]

    def piece(spec):
        kind, seed = spec
        b = fast_bin(seed, 31, PIECE, genome_len=4 * PIECE, err_ppm=0) if kind == "distinct" else fast_bin(seed, 31, PIECE)
        return b, raw_counts(oracle, b, True, prm.lut_prefix_len)

    with ThreadPoolExecutor(THREADS) as pool:
        got = list(pool.map(piece, [s for s, _ in specs]))
        b = composite_bin([(g[0], r) for g, (_, r) in zip(got, specs)])
        parts = [g[1] + (r,) for g, (_, r) in zip(got, specs)]
        del got
        chunks, lut, stats, hist = composite_expected(parts, prm, pool)
        del parts
    n = b.n_rec
    payload_bytes = sum(len(c) for c in chunks)
    t_expected = time.time() - t0
    assert n > 2 ** 30 and n <= 0.85 * limit and payload_bytes > 4 * GiB, (n, limit, payload_bytes)
    assert stats[3] == n and int(hist.sum()) == n
    cap = prm.out_capacity(n) + 64
    need_hbm(slot_bytes(b.size, n, prm, cap), free, "the %d-k-mer bin" % n)

    def run(env):
        for kk, v in env.items():
            monkeypatch.setenv(kk, v)
        ctx = _ctx(prm)
        try:
            l0 = ctx.kernel_launches()
            r = ctx.process_bin(_skb(b))
            launched = ctx.kernel_launches() - l0
        finally:
            ctx.close()
            torch.cuda.empty_cache()
        assert r.stats == stats
        assert np.array_equal(r.lut, lut)
        same_chunks(r.payload, chunks)
        return launched

    one_shot = run({})
    blocks = key_blocks(hist, n // 3)
    assert len(blocks) >= 3 and max(x[2] for x in blocks) > 2 ** 28
    launched = {}
    for flow in ("filter", "scatter"):
        launched[flow] = run({"KMCB200_MAX_BLOCK_RECORDS": str(n // 3), "KMCB200_KEY_BLOCKS": flow})
        assert launched[flow] - one_shot >= 3 * (len(blocks) - 1), (flow, launched[flow], one_shot, len(blocks))
    _report("near limit", n=n, units=units, multiplicities=mults, bin_bytes=b.size, payload_bytes=payload_bytes, block_limit=limit,
            one_sort_launches=one_shot, key_blocks=len(blocks), largest_block=max(x[2] for x in blocks), launches=launched,
            free_hbm_gb="%.1f" % (free / 1e9), expected_s="%.1f" % t_expected, wall_s="%.1f" % (time.time() - t0))


# ---------------------------------------------------------------------------------------------------------------------- 3. a 4 GiB bin at k = 128
@pytest.mark.gpu
def test_k128_bin_of_4gib_at_the_default_chunk_size(oracle, monkeypatch):
    """r copies of one k = 128 bin, at least 4 GiB in all: the key-block path by bytes (size >= 4 x max_chunk_bytes) with the default
    1 GiB expansion chunks, through process_bin and through submit_bin + wait_bin_scanned on two slots at once."""
    import torch
    t0 = time.time()
    prm = Params(128, True, 2, 1_000_000_000, 255, 8)
    for v in ("KMCB200_MAX_BLOCK_RECORDS", "KMCB200_KEY_BLOCKS", "KMCB200_KEY_BLOCK_RECORDS", "KMCB200_MAX_CHUNK_BYTES"):
        monkeypatch.delenv(v, raising=False)
    piece = fast_bin(7128, 128, 1 << 22, mean_extra=0.3)
    r = 4 * GiB // piece.size + 1
    size = r * piece.size
    n = r * piece.n_rec
    assert size >= 4 * GiB
    free = free_hbm()
    cap = prm.out_capacity(n) + 64
    # both slots hold the bin's buffers at once, and the bin stays below the two-slot block limit (one block: oversized by bytes only)
    need = max(2 * slot_bytes(size, n, prm, cap), math.ceil(2 * n * per_record_bytes(128, prm) / 0.6))
    need_hbm(need, free, "a %d-byte k = 128 bin on two slots" % size)
    need_host(size + 4 * GiB, "the %d-byte k = 128 bin" % size)
    b = composite_bin([(piece, r)])
    e_payload, e_lut, e_stats = scaled_expected(oracle, piece, r, prm)
    assert e_stats[3] == n and n <= block_limit(free, 128, prm, n_slots=2)
    ctx = _ctx(prm, n_slots=2)
    try:
        res = ctx.process_bin(_skb(b))
        assert res.stats == e_stats and np.array_equal(res.lut, e_lut) and res.payload.tobytes() == e_payload
        del res
        data = np.ascontiguousarray(b.data)
        packs = np.ascontiguousarray(b.pack_bytes, dtype=np.uint64)
        bases = (0, (1 << 32) + 1)
        outs = [(np.empty(cap, dtype=np.uint8), np.zeros(ctx.lut_entries, dtype=np.uint64)) for _ in bases]
        for slot, (out, lut) in enumerate(outs):
            ctx.submit_bin(slot, data.ctypes.data, b.size, n, packs, out.ctypes.data, cap, lut.ctypes.data)
        excl = np.concatenate([[0], np.cumsum(e_lut)[:-1]]).astype(np.uint64)
        for slot, (out, lut) in enumerate(outs):
            nb, stats = ctx.wait_bin_scanned(slot, bases[slot])
            assert stats == e_stats and nb == len(e_payload)
            assert np.array_equal(lut, np.uint64(bases[slot]) + excl)
            assert out[:nb].tobytes() == e_payload
    finally:
        ctx.close()
        torch.cuda.empty_cache()
    _report("k128 4 GiB", n=n, copies=r, bin_bytes=size, payload_bytes=len(e_payload), path="key blocks by bytes (one block, 1 GiB chunks)",
            free_hbm_gb="%.1f" % (free / 1e9), wall_s="%.1f" % (time.time() - t0))


# ---------------------------------------------------------------------------------------------------------------------- 4. LUT offsets past 2^32
@pytest.mark.gpu
@pytest.mark.parametrize("p", [7, 11])
def test_scanned_lut_past_2_32(oracle, monkeypatch, p):
    """wait_bin_scanned(slot, lut_base) with lut_base = 2^32 - 5, 2^32 + 7 and 2^40 + 3 on two slots: the LUT is lut_base plus the
    exclusive prefix sum of the oracle's, in 64 bits.  Once for a bin counted in one sort (the scan runs on the GPU), once for the same
    bin in key blocks (finished inside submit_bin, the scan runs on the host); the key-block run launches more kernels."""
    prm = Params(31, True, 2, 1_000_000_000, 255, p)
    b = fast_bin(4100 + p, 31, 1_000_000)
    e = oracle.process_bin(b, prm)
    excl = np.concatenate([[0], np.cumsum(e.lut)[:-1]]).astype(np.uint64)
    data = np.ascontiguousarray(b.data)
    packs = np.ascontiguousarray(b.pack_bytes, dtype=np.uint64)
    launched = []
    for blocks in (False, True):
        if blocks:
            monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", "250000")
        ctx = _ctx(prm, n_slots=2)
        try:
            cap = ctx.out_capacity(b.n_rec) + 64
            l0 = ctx.kernel_launches()
            for i, base in enumerate(((1 << 32) - 5, (1 << 32) + 7, (1 << 40) + 3)):
                out, lut = np.zeros(cap, dtype=np.uint8), np.zeros(ctx.lut_entries, dtype=np.uint64)
                ctx.submit_bin(i % 2, data.ctypes.data, b.size, b.n_rec, packs, out.ctypes.data, cap, lut.ctypes.data)
                nb, stats = ctx.wait_bin_scanned(i % 2, base)
                assert stats == e.stats and out[:nb].tobytes() == e.payload, (blocks, base)
                assert np.array_equal(lut, np.uint64(base) + excl), (blocks, base)
            launched.append(ctx.kernel_launches() - l0)
        finally:
            ctx.close()
    assert launched[1] > launched[0], launched
