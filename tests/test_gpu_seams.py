"""GPU: the batch kernels where their work is divided.  Stage 1, stage 0, small k, the estimator, the reads-text parser and homopolymer
compression each split a batch into tiles and thread spans and carry state across them (a halo, a carry or a scan).  Every case here puts
events (separators, lower-case switches, homopolymer edges, signature run starts and ends) at s - 1, s and s + 1 of such seams s, checks
on the reference that it hit them, and compares the GPU with that reference: the stage-1 oracle byte for byte, the stage-0 oracle, the
small-k model, the estimator oracle's full counter tables, the parser model and the homopolymer-compression model."""
import numpy as np
import pytest

from estimate_testlib import SparseCounters, oracle_increments
from hc_testlib import homopolymer_compress, padded
from seam_testlib import (FASTX_SPAN, FASTX_TILE, PACK_WINDOW, REC_TILE, SCAN_BLOCK, TILE, WARP, SeamBatch, check_line_ends, kmer_signatures,
                          norm_table, offsets, records_batch, runs, sampled_kmers, seam_anchors, sizes_to, super_kmers, text_with_line_ends,
                          tiled)
from stage0_testlib import oracle_kxmer_totals, oracle_signature_stats
from stage1_testlib import Split, Stage1Oracle, random_map
from test_fastx_model import FASTA, FASTQ, parse_chunk, records_of
from test_small_k_model import counts

pytestmark = pytest.mark.gpu

KM = [(k, m) for m in (5, 9, 11) for k in sorted({m + 1, 31, 32, 33, 128})]


@pytest.fixture(scope="module")
def s1():
    return Stage1Oracle()


def gpu_split(sp, batch) -> Split:
    out, packs, frags = sp.split_raw(batch)
    fr = np.array([[f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs] for f in frags], dtype=np.uint64)
    return Split(out.copy(), packs.copy(), fr, sp.kmer_len)


def assert_same(got: Split, exp: Split):
    assert np.array_equal(got.frags, exp.frags)
    assert got.out.tobytes() == exp.out.tobytes()
    assert np.array_equal(got.pack_bytes, exp.pack_bytes)


def assert_model_is_oracle(sig, exp: Split):
    """the numpy record model agrees with the oracle on the batch (so its starts and ends are what the oracle wrote)"""
    s, e = super_kmers(sig)
    assert int(exp.frags[:, 3].sum()) == s.size and int(exp.frags[:, 2].sum()) == int((e - s + 1).sum())
    return s, e


# ----------------------------------------------------------------------------- stage-1 seam batches
def run_start_batch(k, m, n_tiles=40):
    """signature runs that start at s - 1, s, s + 1 of every thread seam that is a multiple of 256 (warp and tile seams among them), the
    first half of them in lower case from the run start on.  -> (batch, run starts)"""
    b = SeamBatch(n_tiles * TILE + 77, seed=1000 * k + m)
    starts = []
    for j, a in seam_anchors(len(b), 256, margin=2):
        t = a + offsets(j + j // 16)
        if t + k + 2 >= len(b):
            continue
        b.plant_run(t, k, m)
        if j % 2:
            b.lower(t, t + 100)
        starts.append(t)
    return b, starts


def separator_batch(k, n_tiles=40):
    """a separator on the first base of a k-mer at s - 1, s, s + 1 (a record starts there) and on the last base of one (a record ends
    just before it), alternately, at every multiple of 256.  -> (batch, record starts, record ends)"""
    b = SeamBatch(n_tiles * TILE + 5, seed=77 + k, alphabet=b"CG")
    rec_starts, rec_ends = [], []
    for j, a in seam_anchors(len(b), 256, margin=2):
        t = a + offsets(j + j // 16)
        if t + k + 2 >= len(b):
            continue
        if j % 2 == 0:
            b.sep(t - 1, b"N" if j % 4 else b"\n")
            rec_starts.append(t)
        else:
            b.sep(t + k - 1)                                                  # k-mer t is the first that holds it: t - 1 ends a record
            rec_ends.append(t - 1)
    return b, rec_starts, rec_ends


def long_run_batch(k):
    """runs of 255, 256, 257, 511, 512, 513 special-signature k-mers ending at s - 1, s, s + 1 of successive tile seams.  -> (batch,
    [(first, last)])"""
    lens = (255, 256, 257, 511, 512, 513)
    b = SeamBatch((3 * len(lens) + 2) * TILE, seed=3 + k)
    want = []
    for i in range(3 * len(lens)):
        n = lens[i % len(lens)]
        last = (i + 1) * TILE + offsets(i // len(lens))
        b.poly_a(last - n + 1, n, k)
        want.append((last - n + 1, last))
    return b, want


def stage1_batches(k, m, norm):
    """the three seam batches of (k, m), each checked against the model: it holds the runs and records it was built for"""
    b1, starts = run_start_batch(k, m)
    sig = kmer_signatures(b1.a, k, m, norm)
    rs, re = runs(sig)
    w = k - m + 1
    got = dict(zip(rs.tolist(), re.tolist()))
    assert all(got.get(t) == t + w - 1 for t in starts)
    b2, rec_starts, rec_ends = separator_batch(k)
    s, e = super_kmers(kmer_signatures(b2.a, k, m, norm))
    assert set(rec_starts) <= set(s.tolist()) and set(rec_ends) <= set(e.tolist())
    b3, want = long_run_batch(k)
    s, e = super_kmers(kmer_signatures(b3.a, k, m, norm))
    ss, es = set(s.tolist()), set(e.tolist())
    for lo, hi in want:
        assert all(t in ss for t in range(lo, hi + 1, 256)) and hi in es
    return [b1.tobytes(), b2.tobytes(), b3.tobytes()]


@pytest.mark.parametrize("k,m", KM)
def test_split_runs_separators_and_long_runs_on_seams(s1, k, m):
    import kmc_b200
    norm = norm_table(m)
    n_bins = 64
    sig_map = random_map(k * 7 + m, m, n_bins)
    both = (k + m) % 2 == 0
    for batch in stage1_batches(k, m, norm):
        sp = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=len(batch))
        sp.count_kxmers(both)
        got = gpu_split(sp, batch)
        exp = s1.split(batch, k, m, sig_map, n_bins)
        assert_model_is_oracle(kmer_signatures(np.frombuffer(batch, np.uint8), k, m, norm), exp)
        assert_same(got, exp)
        assert np.array_equal(sp.kxmer_totals(), oracle_kxmer_totals(exp, both))
        sp.close()


@pytest.mark.parametrize("n,k,m", [((1 << 24) + (1 << 20), 31, 9), ((1 << 24) + (1 << 20), 128, 11), (1 << 26, 31, 9), (1 << 26, 128, 11)])
def test_split_poly_a_run_across_the_scan_block_seam(s1, n, k, m):
    """A poly-A run of several tiles that starts in tile 4093 and goes past position 2^24: the tiles after 2^24 take the run start and
    the 256-k-mer cut from the second CTA of the tile scans (split_scan_top_kernel)."""
    import kmc_b200
    seam = TILE * SCAN_BLOCK                                                  # 2^24 positions
    b = SeamBatch(n, seed=n % 1000 + k)
    lo = seam - 3 * TILE + 77
    b.poly_a(lo, 5 * TILE + 300, k)
    if n == 1 << 26:
        b.poly_a(2 * seam - 2 * TILE + 1, 3 * TILE, k)
    batch = b.tobytes()
    # the target: records start at lo + 256 j on both sides of the seam, and a run start never falls in tiles 4094 .. 4096
    exc = slice(lo - 1, lo + 5 * TILE + 300 + k)
    s, _ = super_kmers(kmer_signatures(b.a[exc], k, m, norm_table(m)))
    s = s + exc.start
    assert s[0] == lo and np.all(np.diff(s) == 256) and s[0] < seam - 2 * TILE and s[-1] > seam + TILE
    assert (seam - lo) % 256 not in (0, 255)
    sig_map = random_map(k + m, m, 256)
    sp = kmc_b200.Splitter(k, m, sig_map, 256, max_batch_bytes=n)
    got = gpu_split(sp, batch)
    sp.close()
    assert_same(got, s1.split(batch, k, m, sig_map, 256))


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_split_records_on_pack_window_seams(s1, delta):
    """One bin, k = 128: records of 33..97 bytes arranged so that, at every pack window seam 65408 j, a record ends exactly there and the
    next starts there (delta 0), or one record starts one byte before it (-1) or ends one byte after it (+1)."""
    import kmc_b200
    k, m = 128, 5
    sizes, off = [], 0
    for j in range(1, 5):
        seam = j * PACK_WINDOW
        target = seam + (delta if delta != 1 else 0) - (0 if delta != 1 else 60)
        sizes += sizes_to(target - off, 33)
        off = target
        if delta == 1:
            sizes.append(61)                                                  # [seam - 60, seam + 1)
            off += 61
        sizes += sizes_to(1000, 33)
        off += 1000
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    ends = starts + np.array(sizes)
    for j in range(1, 5):
        seam = j * PACK_WINDOW
        if delta == 0:
            assert seam in set(ends.tolist()) and seam in set(starts.tolist())
        elif delta == -1:
            assert seam - 1 in set(starts.tolist())
        else:
            assert seam + 1 in set(ends.tolist())
    batch = records_batch(sizes, k)
    sig_map = np.zeros(4 ** m + 1, np.uint32)
    exp = s1.split(batch, k, m, sig_map, 1)
    assert int(exp.frags[0][3]) == len(sizes) and int(exp.frags[0][1]) == sum(sizes)
    sp = kmc_b200.Splitter(k, m, sig_map, 1, max_batch_bytes=len(batch))
    got = gpu_split(sp, batch)
    sp.close()
    assert_same(got, exp)
    assert np.all(got.pack_bytes <= 65504)


def round_patterns(n_rec, n_bins, seed):
    """bins for n_rec records, 32 at a time: all one bin, two bins alternating, 32 different bins, random"""
    rng = np.random.default_rng(seed)
    out = []
    for r in range(0, n_rec, 32):
        kind = (r // 32) % 4
        if kind == 0:
            rb = np.full(32, rng.integers(0, n_bins))
        elif kind == 1:
            rb = np.where(np.arange(32) % 2, *rng.choice(n_bins, 2, replace=False))
        elif kind == 2:
            rb = rng.permutation(n_bins)[:32]
        else:
            rb = rng.integers(0, n_bins, 32)
        out.append(rb)
    return np.concatenate(out)[:n_rec]


@pytest.mark.parametrize("n_rec", [REC_TILE - 1, REC_TILE, REC_TILE + 1, 2 * REC_TILE + 1])
@pytest.mark.parametrize("k", [31, 128])
def test_split_record_tiles_and_match_any_rounds(s1, n_rec, k):
    """n_rec one-k-mer records whose bins follow round_patterns: every round of the rank kernel's match.any is one bin, two alternating
    bins, 32 bins or random, and the last round and tile are partial."""
    import kmc_b200
    m, n_bins = 9, 64
    sig_map = random_map(n_rec + k, m, n_bins)
    norm = norm_table(m)
    pool = tiled(4 * n_rec * k, b"ACGT", seed=n_rec, block=4 * n_rec * k).reshape(-1, k)      # untiled: every row drawn on its own
    sig = kmer_signatures((np.concatenate([pool, np.full((pool.shape[0], 1), ord("N"), np.uint8)], axis=1)).reshape(-1), k, m, norm)
    pool_bins = sig_map[sig[::k + 1]]
    by_bin = {b: list(np.flatnonzero(pool_bins == b)) for b in range(n_bins)}
    want = round_patterns(n_rec, n_bins - 1, seed=k)                          # the special signature's bin (n_bins - 1) is rare here
    pick = np.array([by_bin[int(b)].pop() for b in want])
    batch = np.concatenate([pool[pick], np.full((n_rec, 1), ord("\n"), np.uint8)], axis=1).reshape(-1).tobytes()
    exp = s1.split(batch, k, m, sig_map, n_bins)
    assert int(exp.frags[:, 3].sum()) == n_rec and np.array_equal(exp.frags[:, 3].astype(np.int64), np.bincount(want, minlength=n_bins))
    sp = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=len(batch))
    got = gpu_split(sp, batch)
    sp.close()
    assert_same(got, exp)


# ----------------------------------------------------------------------------- stage 0
def lane_batch(k, m):
    """stage 0's own seams: planted runs of exactly 16 positions on a thread's span (k = m + 15), runs that start at lane 0 and at
    lane 31 of a warp, and special-signature runs over one and two whole warps, a whole tile and more than a tile.  -> (batch, runs)"""
    b = SeamBatch(24 * TILE + 300, seed=k + 5 * m)
    want = []
    w = k - m + 1
    for j, a in seam_anchors(12 * TILE, WARP, margin=2):
        if j % 2:
            continue
        t = a + (0 if j % 4 == 0 else 31 * 16 + offsets(j // 4))          # lane 0, or lane 31 and the positions either side of it
        b.plant_run(t, k, m)
        want.append((t, t + w - 1))
    for i, n in enumerate((WARP, 2 * WARP, TILE, TILE + WARP + 3)):
        t = (13 + 3 * i) * TILE
        b.poly_a(t, n, k)
        want.append((t, t + n - 1))
    return b, want


@pytest.mark.parametrize("k,m", KM + [(20, 5), (24, 9), (26, 11)])
def test_sigstats_runs_on_thread_warp_and_tile_seams(k, m):
    import torch
    import kmc_b200
    norm = norm_table(m)
    batches = stage1_batches(k, m, norm)
    lb, want = lane_batch(k, m)
    rs, re = runs(kmer_signatures(lb.a, k, m, norm))
    got_runs = dict(zip(rs.tolist(), re.tolist()))
    assert all(got_runs.get(lo) == hi for lo, hi in want)
    if k == m + 15:                                                           # runs of exactly one thread's 16 positions
        assert sum(hi - lo + 1 == 16 and lo % 16 == 0 for lo, hi in want) >= 30
    batches.append(lb.tobytes())
    L = max(len(x) for x in batches)
    st = kmc_b200.SignatureStats(k, m, max_batch_bytes=L)
    d = torch.empty(L, dtype=torch.uint8, device="cuda")
    for batch in batches:
        want_counts = oracle_signature_stats(batch, k, m)
        st.reset()
        st.add(batch)
        assert np.array_equal(st.read(), want_counts)
        st.reset()
        d[:len(batch)] = torch.from_numpy(np.frombuffer(batch, np.uint8).copy()).cuda()
        st.dev_add(d.data_ptr(), len(batch))
        torch.cuda.synchronize()
        assert np.array_equal(st.read(), want_counts)
    st.close()


# ----------------------------------------------------------------------------- small k
def small_k_batch(n, k, seed):
    """random ACGT with, at s - 1, s, s + 1 of every multiple of 64 (thread spans, tile seams among them): a homopolymer run edge, a
    separator k - 1 bases before the seam, a value change; runs of 40 equal bases that start and end on thread seams"""
    b = SeamBatch(n, seed=seed, alphabet=b"ACGT")
    for j, a in seam_anchors(n, 64, margin=k + 2):
        d = offsets(j + j // 64)
        kind = j % 4
        if kind == 0:
            b.sep(a - (k - 1) + d, b"N" if j % 8 else b"\n")
        elif kind == 1 and a + d + 41 < n:
            b.homopolymer(a + d, a + d + 40, b"ACGT"[j % 8 // 2:j % 8 // 2 + 1])
        elif kind == 2 and a + d + 20 < n:
            b.homopolymer(a + d - 20, a + d, b"T")
        elif kind == 3:
            b.lower(a + d, a + d + 30)
    return b.tobytes()


@pytest.mark.parametrize("k", [1, 4, 7, 8, 11, 13])
@pytest.mark.parametrize("both", [True, False])
def test_small_k_seams_and_batch_lengths(k, both):
    import kmc_b200
    base = small_k_batch(8 * TILE + 1, k, seed=k)
    sk = kmc_b200.SmallKCounter(k, both_strands=both, max_batch_bytes=8 * TILE + 1)
    for n in (TILE - 1, TILE, TILE + 1, 4 * TILE - 1, 4 * TILE, 4 * TILE + 1, 8 * TILE + 1):   # the last one is exactly max_batch_bytes
        batch = base[:n]
        sk.reset()
        sk.add(batch)
        assert np.array_equal(sk.read(), counts(np.frombuffer(batch, np.uint8), k, both)), n
    sk.close()


@pytest.mark.parametrize("k", [1, 4, 7, 8, 11, 13])
def test_small_k_persistent_grid_takes_several_tiles(k):
    """2^24 bases: 4096 tiles, more than three per CTA of the shared-memory kernel's persistent grid"""
    import kmc_b200
    n = 1 << 24
    batch = np.frombuffer(small_k_batch(1 << 18, k, seed=40 + k), np.uint8)
    batch = np.tile(batch, n // batch.size)
    sk = kmc_b200.SmallKCounter(k, both_strands=k % 2 == 1, max_batch_bytes=n)
    sk.add(batch)
    assert np.array_equal(sk.read(), counts(batch, k, k % 2 == 1))
    sk.close()


# ----------------------------------------------------------------------------- the estimator
@pytest.mark.parametrize("k", [1, 31, 32, 33, 64, 65, 128, 255, 256])
def test_estimator_sampled_kmers_end_on_seams(k):
    """k-mers the oracle samples, placed so that they end on t0 - 1, t0, t0 + 1 of tile and thread seams t0, with a separator k or
    k + 1 bases before their end: a hash rolled wrongly at a seam changes a counter the tables show."""
    import kmc_b200
    s = 7
    kms = sampled_kmers(k, s, 8, seed=k)
    n_tiles = 24
    b = SeamBatch(n_tiles * TILE + 3, seed=k, alphabet=b"ACGT")
    placed = []
    if kms:
        for j, a in seam_anchors(len(b), TILE // 2, margin=2 * k + 4):
            t0 = a + (16 * (j % 7) if j % 2 else 0)                          # tile seams, and thread seams inside a tile
            end = t0 + offsets(j // 2)
            km = kms[j % len(kms)]
            b.a[end - k + 1:end + 1] = np.frombuffer(km, np.uint8)
            b.sep(end - k - (j // 2) % 2)                                     # right before the k-mer, or one base further
            placed.append((end, km))
    else:
        assert k == 1                                                         # neither canonical 1-mer is sampled
    batch = b.tobytes()
    for end, km in placed:
        assert batch[end - k + 1:end + 1] == km
        assert oracle_increments(km, k, s).size
    assert len(placed) >= (40 if k < 256 else 20) or k == 1
    est = kmc_b200.HistogramEstimator(k, s, max_batch_bytes=len(batch))
    est.add(batch)
    got = SparseCounters.from_dense(est.read().reshape(-1))
    est.close()
    exp = SparseCounters(oracle_increments(batch, k, s))
    assert np.array_equal(got.index, exp.index) and np.array_equal(got.value, exp.value)


# ----------------------------------------------------------------------------- parser and homopolymer compression
def seam_text(fmt, n_tiles=8, seed=1):
    """text whose '\\n', '\\r\\n' and (FASTA) header starts lie on the last and first byte of 64-byte spans and 16 KiB tiles"""
    targets = []
    kinds = ("lf", "crlf", "hdr") if fmt == "fasta" else ("lf", "crlf")
    for j, a in seam_anchors(n_tiles * FASTX_TILE, FASTX_SPAN * 5, margin=8):
        targets.append((kinds[j % len(kinds)], a - 1 + (j // len(kinds)) % 2))
    for t in range(1, n_tiles):
        targets.append((kinds[t % len(kinds)], t * FASTX_TILE - 1 + (t // len(kinds)) % 2))
    text, placed = text_with_line_ends(fmt, targets, n_tiles * FASTX_TILE, seed)
    check_line_ends(text, placed)
    on_tile = [p for _, p in placed if p % FASTX_TILE in (0, FASTX_TILE - 1)]
    assert len(placed) >= 0.9 * len(targets) and len(on_tile) >= n_tiles - 1
    return text


def unaligned_copies(data, offsets_=range(1, 16)):
    """one device buffer per offset o, the data at a pointer o bytes past a 16-byte boundary"""
    import torch
    buf = torch.zeros(len(data) + 64, dtype=torch.uint8, device="cuda")
    src = torch.from_numpy(np.frombuffer(data, np.uint8).copy()).cuda()
    for o in offsets_:
        buf.zero_()
        buf[o:o + len(data)] = src
        assert (buf.data_ptr() + o) % 16 == o
        yield o, buf, buf.data_ptr() + o


@pytest.mark.parametrize("fmt", ["fastq", "fasta"])
def test_parser_line_ends_on_span_and_tile_seams(fmt):
    import torch
    import kmc_b200
    text = seam_text(fmt)
    p = kmc_b200.FastxParser(fmt, max_chunk_bytes=len(text))
    fmt = FASTQ if fmt == "fastq" else FASTA                                  # what the model takes
    for end, final in ((len(text), True), (len(text) - 5000, False), (3 * FASTX_TILE + 1, False)):
        raw = text[:end]
        want, wc = parse_chunk(raw, fmt, final)
        seq, c = p.parse(raw, final)
        assert c == wc and seq.tobytes() == want.tobytes(), (end, final)
    # the device twin at pointers 1..15 bytes past a 16-byte boundary, so every load is byte-wise, and at an aligned one
    want, wc = parse_chunk(text, fmt, True)
    d_seq = torch.zeros(len(text) + 1, dtype=torch.uint8, device="cuda")
    d_res = torch.zeros(4, dtype=torch.int64, device="cuda")
    for o, _, ptr in unaligned_copies(text, range(0, 16)):
        d_seq.fill_(0xAB)
        p.dev_parse(ptr, len(text), True, None, d_seq.data_ptr(), d_seq.numel(), d_res.data_ptr(), None)
        torch.cuda.synchronize()
        assert list(d_res.cpu().numpy()) == [wc, want.size, records_of(text, fmt, wc), 0], o
        assert d_seq[:want.size].cpu().numpy().tobytes() == want.tobytes(), o
    p.close()


def hc_seam_batch(n, seed):
    """homopolymer runs whose edges lie at s - 1, s, s + 1 of every 64-byte span, case switches inside some, separators between"""
    b = SeamBatch(n, seed=seed, alphabet=b"ACGT")
    for j, a in seam_anchors(n, FASTX_SPAN, margin=40):
        d = offsets(j + j // 256)
        base = b"ACGT"[j % 4:j % 4 + 1]
        if j % 3 == 0:
            b.homopolymer(a + d - 30, a + d, base)                            # ends at the seam
        elif j % 3 == 1:
            b.homopolymer(a + d, a + d + 30, base)                            # starts there
        else:
            b.homopolymer(a + d - 10, a + d + 10, base)                       # straddles it
            b.lower(a + d, a + d + 5)
        if j % 16 == 5:
            b.sep(a + d + 25, b"\n")
    return b.tobytes()


def test_homopolymer_compression_at_unaligned_pointers_and_span_seams(s1):
    """split, statistics and small-k counts with compression on: host batches, the device twins at pointers 1..15 bytes past a 16-byte
    boundary, and the aligned device twin all equal the uncompressed handles (and the oracle) on the compressed batch"""
    import torch
    import kmc_b200
    batch = hc_seam_batch(3 * FASTX_TILE + 13, seed=9)
    comp = homopolymer_compress(batch)
    raw = np.frombuffer(batch, np.uint8)
    runs_cut = int(np.sum((raw[1:] == raw[:-1])[np.arange(1, raw.size) % FASTX_SPAN == 0]))
    assert runs_cut > 100                                                      # runs that go on across a span seam
    k, m, nb = 31, 9, 32
    sig_map = random_map(2, m, nb)
    model = padded(batch).tobytes()
    exp = s1.split(comp.tobytes(), k, m, sig_map, nb)
    sp = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=len(batch), homopolymer_compressed=True)
    assert_same(gpu_split(sp, batch), exp)
    want_stats = oracle_signature_stats(comp.tobytes(), k, m)
    want_k = {kk: counts(comp, kk) for kk in (3, 9)}
    st = kmc_b200.SignatureStats(k, m, max_batch_bytes=len(batch), homopolymer_compressed=True)
    sks = {kk: kmc_b200.SmallKCounter(kk, max_batch_bytes=len(batch), homopolymer_compressed=True) for kk in want_k}
    cap = exp.out.size + 64
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_packs = torch.zeros(exp.pack_bytes.size + 8, dtype=torch.int64, device="cuda")
    d_frags = torch.zeros(nb * 5, dtype=torch.int64, device="cuda")
    d_res = torch.zeros(8, dtype=torch.int64, device="cuda")
    for o, buf, ptr in unaligned_copies(batch, range(0, 16)):
        before = buf.clone()
        sp.dev_split(ptr, len(batch), d_out.data_ptr(), cap, d_packs.data_ptr(), d_packs.numel(), d_frags.data_ptr(), d_res.data_ptr())
        st.reset()
        st.dev_add(ptr, len(batch))
        for sk in sks.values():
            sk.reset()
            sk.dev_add(ptr, len(batch))
        torch.cuda.synchronize()
        res = d_res.cpu().numpy()
        assert res[2] == 0 and res[0] == exp.out.size and d_out[:res[0]].cpu().numpy().tobytes() == exp.out.tobytes(), o
        assert np.array_equal(d_packs[:res[1]].cpu().numpy().view(np.uint64), exp.pack_bytes), o
        assert np.array_equal(st.read(), want_stats), o
        for kk, sk in sks.items():
            assert np.array_equal(sk.read(), want_k[kk]), (o, kk)
        assert torch.equal(buf, before)
    # and the uncompressed handles on the padded model batch say the same
    plain = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=len(batch))
    assert_same(gpu_split(plain, model), exp)
    for h in [sp, st, plain] + list(sks.values()):
        h.close()
