"""Skewed bins for stage 2's key-block and multi-GPU flows, and host checks (no GPU) that every generator makes what it claims.

The biggest bins of a real run are where repeats collect (poly-A / poly-T, satellites, low-complexity minimizers), and only those bins
are cut into key blocks (run_oversized_bin) or split over several GPUs (kmcb200_process_bin_multi).  The generators below make such
bins, seeded; a numpy restatement of the host-side layout (the top-12-bit histogram, bisect_blocks, the multi-GPU key ranges and pack
shares, the level-2 bits of a block, a block's leaves) says where their k-mers land.  The checks here pin that layout for the very
cases tests/test_gpu_skewed_blocks.py runs: a dominant k-mer in a heavy leaf of a block whose prefix is not 0, a leaf too large for the
leaf kernels inside a later block, a single 12-bit bucket above the block limit, key ranges left empty, a pack share of zero-byte packs.
They also pin the oracle itself on small skewed bins against the brute-force counter."""
import numpy as np
import pytest

from kmc_testlib import Bin, Params, _make_packs, brute_force_counts, expected_from_counts, fast_bin
from test_gpu_corners import concat_bins, record_sizes, with_packs

# kmc_b200/csrc/leaf_warp.cuh, kmc_b200.cu, expand.cuh
LW_HEAVY = 16384               # kLwHeavy: a one-word leaf beyond this is counted by leaf_warp_kernel (dominant-k-mer path)
LW_MAX_LEAF = 65534            # kLwMaxLeaf: what a warp-counted leaf (or its rest, after the dominant k-mer) may hold
LW_MAX_HEAVY_LEAF = 1 << 22    # kLwMaxHeavyLeaf
MSD_MIN_RECORDS = 1 << 16      # msd_path: smaller sorts (and key blocks) take the plain LSD passes, without leaves
MAX_BLOCKS = 512               # kExpandMaxBlocks
L2_SEVEN_BITS_MAX_MEAN = 5120  # kL2SevenBitsMaxMean

BLOCK_LIMIT = 250_000          # KMCB200_MAX_BLOCK_RECORDS of the GPU cases
N_BG = 1_200_000               # k-mers of a 30x background
COPIES = 40_000                # copies of a dominant k-mer: above LW_HEAVY, and more than a quarter of its leaf
MID_BUCKET = 0x900             # "GAAA.." + ...: a middle key block of one GPU, the last GPU's range of 2-4 canonical ones
ONE_PREFIX = (1, 2, 0, 3, 1, 0)                      # CGATCA: bucket 1588
OVERFULL_PREFIX = ONE_PREFIX + (2, 1, 3, 0, 0, 1)    # 12 shared symbols: one leaf for any block of <= 16 bits and level 2 of <= 8


# ---------------------------------------------------------------------------------------------------------------------- generators
def sym6(bucket):
    """The first 6 symbols of the k-mers whose top 12 key bits are `bucket`."""
    return np.array([(bucket >> (10 - 2 * i)) & 3 for i in range(6)], dtype=np.uint8)


def revcomp(s):
    return (3 - np.asarray(s)[..., ::-1]).astype(np.uint8)


def force_canonical(rows):
    """Rows of k symbols whose first symbol is A, C or G get a last symbol below 3 - first: the reverse complement then starts with a larger
    symbol, so every row is its own canonical k-mer."""
    assert np.all(rows[:, 0] <= 2)
    rows[:, -1] = rows[:, -1] % (3 - rows[:, 0])
    return rows


def kmer_records(k, rows):
    """One bin record per row of symbols (rows: [n, L], k <= L <= k + 255), in collector packs of <= 64 KiB."""
    rows = np.asarray(rows, dtype=np.uint8)
    n, L = rows.shape
    nb = (L + 3) // 4
    pad = np.zeros((n, nb * 4), dtype=np.uint8)
    pad[:, :L] = rows
    q = pad.reshape(n, nb, 4)
    body = (q[:, :, 0] << 6) | (q[:, :, 1] << 4) | (q[:, :, 2] << 2) | q[:, :, 3]
    data = np.concatenate([np.full((n, 1), L - k, dtype=np.uint8), body.astype(np.uint8)], axis=1).reshape(-1)
    pb, pr, pf = _make_packs(np.full(n, 1 + nb, dtype=np.int64), np.full(n, L - k + 1, dtype=np.int64))
    return Bin(data=data, n_rec=n * (L - k + 1), n_super_kmers=n, pack_bytes=pb, pack_recs=pr, k=k, extras=np.full(n, L - k, dtype=np.int64),
               pack_first=pf)


def dominant_kmer(k, bucket, both, seed):
    """A k-mer whose top 12 key bits are `bucket`; canonical when both."""
    rng = np.random.default_rng(seed)
    one = np.concatenate([sym6(bucket), rng.integers(0, 4, k - 6)]).astype(np.uint8)
    return force_canonical(one[None])[0] if both else one


def dominant_bin(k, copies, bucket, both, n_bg=N_BG, seed=1):
    """A 30x background of n_bg k-mers plus `copies` copies of one k-mer (dominant_kmer); with both, every second copy is its reverse
    complement."""
    one = dominant_kmer(k, bucket, both, seed)
    rows = np.repeat(one[None], copies, axis=0)
    if both:
        rows[1::2] = revcomp(one)
    return concat_bins(fast_bin(seed, k, n_bg), kmer_records(k, rows))


def prefix_rows(k, prefix, n, both, rng, pool=None):
    """n k-mers that all start with `prefix`, their tails drawn from a pool of `pool` tails (all-distinct tails when pool is None); with both,
    every second one is written as its reverse complement."""
    prefix = np.asarray(prefix, dtype=np.uint8)
    tails = rng.integers(0, 4, (n if pool is None else pool, k - prefix.size)).astype(np.uint8)
    rows = np.concatenate([np.repeat(prefix[None], tails.shape[0], axis=0), tails], axis=1)
    if both:
        rows = force_canonical(rows)
    if pool is not None:
        rows = rows[rng.integers(0, pool, n)]
    if both:
        rows[1::2] = revcomp(rows[1::2])
    return rows


def one_prefix_bin(k, n, both, n_bg=0, seed=2):
    """n k-mers that share their first 6 symbols (ONE_PREFIX: one 12-bit bucket), ~4 copies of each tail; plus a 30x background of n_bg."""
    b = kmer_records(k, prefix_rows(k, ONE_PREFIX, n, both, np.random.default_rng(seed), pool=max(n // 4, 1)))
    return concat_bins(fast_bin(seed, k, n_bg), b) if n_bg else b


def lopsided_bin(k, frac, both, n=N_BG, seed=3):
    """frac of n k-mers in one 12-bit bucket (one_prefix_bin), the rest a 30x background."""
    m = int(frac * n)
    return one_prefix_bin(k, m, both, n_bg=n - m, seed=seed)


def overfull_leaf_bin(k, both, n_bg=1_000_000, n_leaf=80_000, seed=4):
    """n_leaf all-distinct k-mers sharing their first 12 symbols (OVERFULL_PREFIX) in a 30x background: under the key-block layout they are
    one leaf of more than LW_MAX_LEAF records with no dominant k-mer, inside a block whose prefix is not 0."""
    rows = prefix_rows(k, OVERFULL_PREFIX, n_leaf, both, np.random.default_rng(seed))
    return concat_bins(fast_bin(seed, k, n_bg), kmer_records(k, rows))


def polyat_bin(k, copies, n_bg=N_BG, seed=5):
    """A 30x background plus poly-A and poly-T super-k-mers of k + 255 symbols, `copies` k-mers of each (rounded up to whole records).
    Canonical: both are the all-A k-mer (key 0).  -b: key 0 and the all-ones key, the first and the last bucket."""
    n_sk = -(-copies // 256)
    tails = kmer_records(k, np.concatenate([np.zeros((n_sk, k + 255), np.uint8), np.full((n_sk, k + 255), 3, np.uint8)]))
    return concat_bins(fast_bin(seed, k, n_bg), tails)


# ---------------------------------------------------------------------------------------------------------------------- host-side layout
def top_bits(recs, k, nbits):
    """The top nbits (<= 40) of every k-mer of an expanded record array [n, W] (the k-mer in the low 2k bits, word 0 least significant)."""
    w = recs.shape[1]
    shift = 2 * k - nbits
    base = 64 * (w - 1)
    assert shift >= base
    return recs[:, w - 1] >> np.uint64(shift - base)


def kmer_words(syms, both):
    """One k-mer (symbols) as the expanded record's words."""
    s = np.asarray(syms)
    if both and tuple(revcomp(s)) < tuple(s):
        s = revcomp(s)
    v = 0
    for x in s:
        v = (v << 2) | int(x)
    return np.array([(v >> (64 * i)) & ((1 << 64) - 1) for i in range((s.size + 31) // 32)], dtype=np.uint64)


def hist12(recs, k):
    return np.bincount(top_bits(recs, k, 12).astype(np.int64), minlength=4096)


def bisect_blocks(hist, lo, hi, limit):
    """kmc_b200.cu bisect_blocks: aligned prefixes inside [lo, hi), ascending, each with at most `limit` k-mers unless it is one bucket.
    Returns [(prefix, bits, n)]."""
    cover, p = [], lo
    while p < hi:
        ln = 1
        while ln < 4096 and p % (2 * ln) == 0 and p + 2 * ln <= hi:
            ln *= 2
        cover.append((p, ln))
        p += ln
    csum = np.concatenate([[0], np.cumsum(hist)])
    todo, blocks = cover[::-1], []
    while todo:
        q, ln = todo.pop()
        cnt = int(csum[q + ln] - csum[q])
        if cnt == 0:
            continue
        if cnt <= limit or ln == 1:
            lg = ln.bit_length() - 1
            blocks.append((q >> lg, 12 - lg, cnt))
        else:
            todo += [(q + ln // 2, ln // 2), (q, ln // 2)]
    return blocks


def key_blocks(hist, limit):
    """run_oversized_bin's blocks (the block limit and the preferred block size are the same here)."""
    blocks = bisect_blocks(hist, 0, 4096, limit)
    return blocks if len(blocks) <= MAX_BLOCKS else bisect_blocks(hist, 0, 4096, limit)


def multi_cut(hist, n_ctx):
    """kmcb200_process_bin_multi: the key range [cut[g], cut[g + 1]) of every GPU."""
    n_rec = int(hist.sum())
    cut, acc, g = [0] + [4096] * n_ctx, 0, 1
    for q in range(4096):
        if g >= n_ctx:
            break
        acc += int(hist[q])
        while g < n_ctx and acc * n_ctx >= g * n_rec:
            cut[g] = q + 1
            g += 1
    return cut


def multi_blocks(hist, n_ctx, limit):
    """Every GPU's key blocks: [[(prefix, bits, n)] per GPU]."""
    cut = multi_cut(hist, n_ctx)
    for _ in range(8):
        per = [bisect_blocks(hist, cut[g], cut[g + 1], limit) for g in range(n_ctx)]
        if sum(len(x) for x in per) <= MAX_BLOCKS:
            return per
        limit *= 2
    raise AssertionError("too many blocks")


def multi_shares(pack_bytes, n_ctx):
    """kmcb200_process_bin_multi: every GPU's share of the packs, [(first pack, packs, bytes)]."""
    pack_bytes = [int(x) for x in pack_bytes]
    size = sum(pack_bytes)
    parts = [[0, 0, 0] for _ in range(n_ctx)]
    pos, g = 0, 0
    for i, pb in enumerate(pack_bytes):
        if g + 1 < n_ctx and parts[g][1] > 0 and pos >= (g + 1) * size // n_ctx and len(pack_bytes) - i >= n_ctx - g - 1:
            g += 1
            parts[g][0] = i
        parts[g][1] += 1
        parts[g][2] += pb
        pos += pb
    return [tuple(x) for x in parts]


def multi_splits(n_rec, n_packs, n_ctx, k):
    """Does kmcb200_process_bin_multi split the bin (or hand it to the first context's process_bin)?"""
    return n_rec > 0 and n_ctx > 1 and 2 * k >= 24 and n_rec >= 4096 * n_ctx and n_packs >= n_ctx


def level2_bits(n, words):
    """choose_b2 for counted leaves."""
    t, lg = (n + 1023) // 1024, 0
    while (1 << lg) < t:
        lg += 1
    return min(lg - 8 if lg > 8 else 0, (7 if n <= L2_SEVEN_BITS_MAX_MEAN << 15 else 8) if words == 1 else 10)


def block_of(blocks, top12):
    for i, (prefix, bits, n) in enumerate(blocks):
        if top12 >> (12 - bits) == prefix:
            return i
    raise AssertionError("bucket %d is in no block" % top12)


def block_leaves(recs, k, block):
    """(level-2 bits, the leaf of every record of the block, the block's record mask); None for the leaves when the block is too small for
    the leaf path."""
    prefix, bits, n = block
    b2 = level2_bits(n, recs.shape[1])
    t = top_bits(recs, k, bits + 8 + b2)
    mask = (t >> np.uint64(8 + b2)) == np.uint64(prefix)
    assert int(mask.sum()) == n
    return b2, (t[mask] & np.uint64((256 << b2) - 1) if n >= MSD_MIN_RECORDS else None), mask


def leaf_of_kmer(recs, k, block, kmer):
    """(records of the leaf that holds `kmer`, copies of `kmer` in it, most copies of any k-mer in it)."""
    prefix, bits, n = block
    b2, leaves, mask = block_leaves(recs, k, block)
    assert leaves is not None, "a block of %d records takes the plain LSD sort, not the leaf path" % n
    leaf = int(top_bits(kmer[None], k, bits + 8 + b2)[0]) & ((256 << b2) - 1)
    in_leaf = recs[mask][leaves == np.uint64(leaf)]
    _, counts = np.unique(in_leaf, axis=0, return_counts=True)
    return in_leaf.shape[0], int(np.all(in_leaf == kmer, axis=1).sum()), int(counts.max())


def assert_heavy_leaf(recs, k, block, kmer):
    """The leaf of `kmer` in `block` goes the dominant-k-mer way of leaf_warp_kernel, and is counted there (leaf_warp.cuh:248-270)."""
    m, n_eq, _ = leaf_of_kmer(recs, k, block, kmer)
    assert LW_HEAVY < m <= LW_MAX_HEAVY_LEAF and n_eq > m // 4 and m - n_eq <= LW_MAX_LEAF, (m, n_eq)


def assert_overfull_leaf(recs, k, block, kmer):
    """The leaf of `kmer` in `block` cannot be counted by any leaf kernel: the block takes the LSD fallback."""
    m, _, most = leaf_of_kmer(recs, k, block, kmer)
    assert m > LW_MAX_LEAF and (recs.shape[1] > 1 or most <= m // 4), (m, most)


# ---------------------------------------------------------------------------------------------------------------------- the GPU cases' bins
def params(k=31, both=True, p=7, cmin=2, cmax=10 ** 9, cntmax=255):
    return Params(k=k, both_strands=both, cutoff_min=cmin, cutoff_max=cmax, counter_max=cntmax, lut_prefix_len=p)


def make_bin(gen, k, both):
    """The bins of tests/test_gpu_skewed_blocks.py by name, with the k-mer each one is built around (None: poly-A/T)."""
    if gen == "dominant":
        return dominant_bin(k, COPIES, MID_BUCKET, both), dominant_kmer(k, MID_BUCKET, both, 1)
    if gen == "one_prefix":
        return one_prefix_bin(k, 400_000, both), None
    if gen == "one_prefix_bg":
        return one_prefix_bin(k, 400_000, both, n_bg=800_000), None
    if gen == "lopsided":
        return lopsided_bin(k, 0.6, both), None
    if gen == "overfull":
        return overfull_leaf_bin(k, both), np.concatenate([OVERFULL_PREFIX, np.zeros(k - 12, np.uint8)]).astype(np.uint8)
    if gen == "polyat":
        return polyat_bin(k, COPIES), None
    raise ValueError(gen)


KEY_BLOCK_GENS = [("dominant", 31, True), ("dominant", 31, False), ("polyat", 31, True), ("polyat", 31, False), ("one_prefix_bg", 31, True),
                  ("one_prefix_bg", 55, True), ("overfull", 31, True), ("overfull", 31, False), ("overfull", 55, True)]
MULTI_GENS = [("dominant", 31, True, 2), ("dominant", 31, True, 3), ("dominant", 31, True, 4), ("dominant", 31, False, 3), ("polyat", 31, False, 2),
              ("lopsided", 31, True, 3), ("lopsided", 31, True, 4), ("one_prefix", 31, True, 2), ("one_prefix", 31, True, 4), ("overfull", 31, True, 3),
              ("overfull", 55, True, 2)]


@pytest.fixture(scope="module")
def expanded(oracle):
    cache = {}

    def get(gen, k, both):
        if (gen, k, both) not in cache:
            b, kmer = make_bin(gen, k, both)
            recs = oracle.expand(b, params(k, both))
            cache[(gen, k, both)] = (b, kmer, recs)
        return cache[(gen, k, both)]
    return get


# ---------------------------------------------------------------------------------------------------------------------- checks
@pytest.mark.parametrize("gen,k,both", KEY_BLOCK_GENS, ids=["%s-k%d-%s" % (g, k, "ci" if b else "b") for g, k, b in KEY_BLOCK_GENS])
def test_key_block_layout(expanded, gen, k, both):
    """Under a block limit of BLOCK_LIMIT every bin is cut into several key blocks, and its skew lands where the GPU case needs it."""
    b, kmer, recs = expanded(gen, k, both)
    assert recs.shape[0] == b.n_rec > BLOCK_LIMIT
    hist = hist12(recs, k)
    blocks = key_blocks(hist, BLOCK_LIMIT)
    assert len(blocks) > 1
    if gen == "dominant":
        top = int(top_bits(kmer_words(kmer, both)[None], k, 12)[0])
        assert top == MID_BUCKET
        i = block_of(blocks, top)
        assert 0 < i < len(blocks) - 1 and blocks[i][0] != 0
        assert_heavy_leaf(recs, k, blocks[i], kmer_words(kmer, both))
    elif gen == "polyat":
        zero = kmer_words(np.zeros(k, np.uint8), both)
        assert block_of(blocks, 0) == 0
        assert_heavy_leaf(recs, k, blocks[0], zero)
        if not both:                        # the all-ones key: the last block, whose prefix is not 0
            ones = kmer_words(np.full(k, 3, np.uint8), both)
            assert block_of(blocks, 4095) == len(blocks) - 1 and blocks[-1][0] != 0
            assert_heavy_leaf(recs, k, blocks[-1], ones)
        else:
            m, n_eq, _ = leaf_of_kmer(recs, k, blocks[0], zero)
            assert n_eq >= 2 * COPIES
    elif gen == "one_prefix_bg":            # one bucket above the limit: a block of one 12-bit prefix that is larger than the limit
        top = int(np.dot(ONE_PREFIX, 4 ** np.arange(5, -1, -1)))
        i = block_of(blocks, top)
        assert blocks[i][1] == 12 and blocks[i][2] > BLOCK_LIMIT and i > 0
        assert blocks[i][2] == max(x[2] for x in blocks)
    elif gen == "overfull":
        i = block_of(blocks, int(np.dot(OVERFULL_PREFIX[:6], 4 ** np.arange(5, -1, -1))))
        assert i > 0 and blocks[i][0] != 0 and blocks[i][2] >= MSD_MIN_RECORDS
        assert any(x[2] for x in blocks[:i])          # earlier blocks have output: the fallback's records go behind theirs
        assert_overfull_leaf(recs, k, blocks[i], kmer_words(kmer, both))


@pytest.mark.parametrize("gen,k,both,n_ctx", MULTI_GENS, ids=["%s-k%d-%s-%dgpu" % (g, k, "ci" if b else "b", n) for g, k, b, n in MULTI_GENS])
def test_multi_layout(expanded, gen, k, both, n_ctx):
    """Over n_ctx GPUs: the dominant k-mer is in the last GPU's range (or a middle one) in a heavy leaf; a lopsided or one-bucket bin leaves
    key ranges empty; the overfull leaf is in a block of a GPU other than the first."""
    b, kmer, recs = expanded(gen, k, both)
    assert multi_splits(b.n_rec, b.pack_bytes.size, n_ctx, k)
    hist = hist12(recs, k)
    per = multi_blocks(hist, n_ctx, BLOCK_LIMIT)
    owner = lambda top: next(g for g in range(n_ctx) if any(top >> (12 - bits) == pre for pre, bits, _ in per[g]))
    if gen == "dominant":
        g = owner(MID_BUCKET)
        assert g > 0 and (g == n_ctx - 1 or not both)
        assert_heavy_leaf(recs, k, per[g][block_of(per[g], MID_BUCKET)], kmer_words(kmer, both))
    elif gen == "polyat":
        assert owner(4095) == n_ctx - 1
        assert_heavy_leaf(recs, k, per[-1][-1], kmer_words(np.full(k, 3, np.uint8), both))
    elif gen in ("lopsided", "one_prefix"):
        empty = [g for g in range(n_ctx) if not per[g]]
        assert empty
        if gen == "one_prefix":             # everything in one bucket: the first GPU owns the only block, which is above the limit
            assert empty == list(range(1, n_ctx)) and len(per[0]) == 1 and per[0][0][1] == 12 and per[0][0][2] > BLOCK_LIMIT
    elif gen == "overfull":
        top = int(np.dot(OVERFULL_PREFIX[:6], 4 ** np.arange(5, -1, -1)))
        g = owner(top)
        assert g > 0
        assert_overfull_leaf(recs, k, per[g][block_of(per[g], top)], kmer_words(kmer, both))


def zero_byte_share_packs(b, frac=0.7):
    """The bin's records in packs [one pack of the first ~frac of the bytes, 0, 0, the rest in packs of <= 64 KiB]: on 3 GPUs the second
    GPU's share is one zero-byte pack."""
    sizes = record_sizes(b)
    ends = np.cumsum(sizes)
    i = int(np.searchsorted(ends, frac * b.size)) + 1
    packs, acc = [int(ends[i - 1]), 0, 0], 0
    for s in sizes[i:]:
        if acc + s > 1 << 16:
            packs.append(acc)
            acc = 0
        acc += s
    return with_packs(b, packs + [acc])


def test_shares_of_zero_byte_packs():
    b = zero_byte_share_packs(fast_bin(11, 31, 300_000))
    shares = multi_shares(b.pack_bytes, 3)
    assert shares[1] == (1, 1, 0) and shares[0][2] > 2 * b.size // 3 and multi_splits(b.n_rec, b.pack_bytes.size, 3, 31)


def in_packs(b, n_packs):
    """The bin's records in exactly n_packs packs of about equal bytes."""
    ends = np.cumsum(record_sizes(b))
    cuts = [0] + [int(ends[np.searchsorted(ends, i * b.size / n_packs)]) for i in range(1, n_packs)] + [b.size]
    assert len(set(cuts)) == n_packs + 1
    return with_packs(b, np.diff(cuts))


def threshold_bin(n_ctx, what, split):
    """Bins on either side of the two thresholds below which kmcb200_process_bin_multi does not split: 4096 n_ctx k-mers (in n_ctx packs),
    n_ctx packs (of a bin of 300 000 k-mers)."""
    if what == "n_rec":
        return in_packs(fast_bin(20 + n_ctx, 31, 4096 * n_ctx - 1 + split), n_ctx)
    return in_packs(fast_bin(30 + n_ctx, 31, 300_000), n_ctx - 1 + split)


@pytest.mark.parametrize("n_ctx", [2, 3, 4])
def test_split_thresholds(n_ctx):
    for what in ("n_rec", "n_packs"):
        for split in (False, True):
            b = threshold_bin(n_ctx, what, split)
            assert multi_splits(b.n_rec, b.pack_bytes.size, n_ctx, 31) == split
            assert (b.n_rec - 4096 * n_ctx if what == "n_rec" else b.pack_bytes.size - n_ctx) == (0 if split else -1)


SMALL = {"dominant": lambda both: dominant_bin(31, 300, MID_BUCKET, both, n_bg=3000),
         "one_prefix": lambda both: one_prefix_bin(31, 2000, both, n_bg=1000),
         "lopsided": lambda both: lopsided_bin(31, 0.6, both, n=3000),
         "overfull": lambda both: overfull_leaf_bin(31, both, n_bg=2000, n_leaf=1500),
         "polyat": lambda both: polyat_bin(31, 600, n_bg=2000)}


@pytest.mark.parametrize("both", [True, False])
@pytest.mark.parametrize("gen", sorted(SMALL))
def test_oracle_on_small_skewed_bins(oracle, gen, both):
    """The oracle, the reference of every GPU case, against the brute-force counter on small versions of the skewed bins: cutoffs below
    and above the dominant count, clamping, a LUT prefix of 3 and 7."""
    b = SMALL[gen](both)
    for p in (params(31, both, 7, 1), params(31, both, 3, 2, cmax=500, cntmax=100)):
        cnt = brute_force_counts(b, p)
        assert max(cnt.values()) >= (256 if gen in ("dominant", "polyat") else 2)
        payload, lut, stats = expected_from_counts(cnt, p)
        e = oracle.process_bin(b, p)
        assert e.payload == payload and np.array_equal(e.lut, lut) and e.stats == stats
