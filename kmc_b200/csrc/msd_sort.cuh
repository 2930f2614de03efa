// kmc_b200 — hybrid MSD radix sort of packed k-mer records (the fast path of the sort stage).
//
// Like RADULS (kmc_core/raduls_impl.h:546-754) this is an MSD radix sort with small-sort leaves: the top digits
// split the bin into buckets, buckets that fit on chip are finished there.  An MSD partition does not have to be
// stable (a bucket is refined independently of the order inside it), which is what makes it cheap on a GPU: the
// rank of a record inside its tile is simply the value returned by ONE shared-memory atomicAdd - no match.any,
// no warp-private histograms, no serial cursor chain.
//
//   level 1   msd_partition_kernel   whole bin   -> 2^8 buckets          (per-tile digit counts written by expand_kernel)
//   count     msd_count_kernel       per tile of every level-1 bucket: counts of the next digit
//   scan      cell_*_kernel, msd_bounds_kernel   flat scan of the counts = output offsets + bucket boundaries (+ oversize check)
//   level 2   msd_partition_kernel   every level-1 bucket -> 2^b2 sub-buckets (b2 <= 8, chosen so that a leaf has ~1 K records)
//   leaves    msd_local_sort_kernel  one leaf bucket per CTA iteration: load to shared memory, LSD radix sort of the
//                                    remaining bits entirely on chip, write back
//
// Traffic: 2NW (level 1) + NW (count) + 2NW (level 2) + 2NW (leaves) = 7 N*W instead of 16 N*W for 8 LSD passes; no look-back anywhere.
// A leaf that does not fit in shared memory (heavy skew) makes the scan raise a device flag; every kernel of this file then
// returns at once and the 8-bit LSD passes of radix_sort.cuh (always enqueued behind, normally returning at once) sort the bin.
#pragma once
#include "common.cuh"
#include "expand.cuh"
#include "radix_sort.cuh"

namespace kmcb {

constexpr uint32_t kMsdFlagFallback = 1;      // flags[0] bit 0: leaves too large -> the LSD passes take over
constexpr uint32_t kMsdFlagAbort = 2;         // flags[0] and flags[1] bit 1: the bin is malformed (expand.cuh): nothing downstream may run
constexpr uint32_t kMsdFlagStop = kMsdFlagFallback | kMsdFlagAbort;

// bits [shift, shift+nbits) of a record (nbits <= 8... 32), record = little-endian multi-word integer
template <int WORDS>
__device__ __forceinline__ uint32_t rec_bits(const Rec<WORDS>& r, uint32_t shift, uint32_t mask)
{
	if (WORDS == 1) return (uint32_t)(r.w[0] >> shift) & mask;
	const uint32_t wi = shift >> 6, off = shift & 63u;
	uint64_t lo = r.w[0], hi = 0;
#pragma unroll
	for (int i = 1; i < WORDS; ++i) {
		if (wi == (uint32_t)i) lo = r.w[i];
		if (wi + 1 == (uint32_t)i) hi = r.w[i];
	}
	uint64_t v = lo >> off;
	if (off) v |= hi << (64u - off);
	return (uint32_t)v & mask;
}

template <int WORDS> struct MsdCfg;
template <> struct MsdCfg<1> { static constexpr int kThreads = 512, kKpt = 8, kMinBlocks = 2; };
template <> struct MsdCfg<2> { static constexpr int kThreads = 512, kKpt = 4, kMinBlocks = 2; };
template <> struct MsdCfg<3> { static constexpr int kThreads = 512, kKpt = 4, kMinBlocks = 1; };     // a tile must hold an expand tile (2048 records)
template <> struct MsdCfg<4> { static constexpr int kThreads = 512, kKpt = 4, kMinBlocks = 1; };
static_assert(true, "");

template <int WORDS> __host__ __device__ constexpr int msd_tile() { return MsdCfg<WORDS>::kThreads * MsdCfg<WORDS>::kKpt; }

// A partition pass is "count, scan, scatter", with the counting fused into whoever touched the records last:
//   * work items: contiguous record ranges of at most msd_tile() records that never straddle a segment.  Level 1: the output
//     tiles of expand_kernel (explicit ranges); level 2: the aligned tiles of every level-1 bucket (tables built on the device);
//   * cells: counts[segment][digit][item of the segment] (u16) - the ORDER OF THE OUTPUT.  One flat exclusive scan over the
//     cells therefore yields, for every (item, digit), the global index where that item's records of that digit go, and for
//     every (segment, digit) the boundary of the next level's bucket;
//   * the scatter kernel needs no look-back, no descriptors and no spinning: rank = return value of a shared-memory
//     atomicAdd, base = one precomputed cell.
struct MsdItems {
	// explicit ranges (level 1) ...
	const uint64_t* item_lo;     // [n_items] or nullptr
	const uint16_t* item_cnt;
	// ... or aligned tiles inside segments (level 2)
	const uint64_t* seg_start;   // [S + 1]
	const uint32_t* item_base;   // [S + 1] first item of every segment
	const uint32_t* item_seg;    // [n_items]
	const uint32_t* n_items;     // device scalar
};

struct MsdItemGeom {
	uint64_t lo, hi;      // records [lo, hi)
	uint64_t lo_al;       // first record of the 16-byte aligned load
	uint32_t n_load;
	uint64_t cell0;       // cell of (this item, digit 0); digit d is at cell0 + d * cell_stride
	uint32_t cell_stride; // items of the segment
};

template <int WORDS>
__device__ __forceinline__ MsdItemGeom msd_item_geom(const MsdItems& it, uint32_t item, uint32_t nd)
{
	constexpr uint64_t TILE = msd_tile<WORDS>();
	MsdItemGeom g;
	if (it.item_lo) {
		g.lo = it.item_lo[item];
		g.hi = g.lo + it.item_cnt[item];
		g.cell_stride = *it.n_items;
		g.cell0 = item;
	} else {
		const uint32_t seg = it.item_seg[item];
		const uint64_t sb = it.seg_start[seg], se = it.seg_start[seg + 1];
		const uint32_t first_item = it.item_base[seg];
		const uint64_t T = sb / TILE + (item - first_item);
		g.lo = T * TILE > sb ? T * TILE : sb;
		g.hi = (T + 1) * TILE < se ? (T + 1) * TILE : se;
		g.cell_stride = it.item_base[seg + 1] - first_item;
		g.cell0 = (uint64_t)nd * first_item + (item - first_item);
	}
	g.lo_al = g.lo & ~1ull;
	g.n_load = (uint32_t)(((g.hi + 1) & ~1ull) - g.lo_al);
	return g;
}


// The scatter kernel is a producer / consumer pipeline inside the CTA.  One extra PRODUCER warp runs ahead of the 16 consumer
// warps: for every work item of the CTA (static round robin: items are equally large) it resolves the item's geometry (a chain of
// dependent global loads: item -> segment -> boundaries), gathers the item's 256 output bases from the cell scan, and fetches the
// records global->shared with ONE TMA bulk copy into a ring of kStages buffers (full / empty mbarriers).  The consumers never
// wait for a global load: an item starts when its `full` barrier flips.
// Tried and dropped: thread 0 claiming tickets and issuing the copies itself; cursors precomputed from the cells by the producer
// (position = atomicAdd(&cursor[digit], 1) straight into a staging buffer, no histogram / scan, two barriers instead of five) - fewer
// instructions, but slower; the same cursors with in-place regrouping and three buffers (the single producer warp cannot gather 768
// values per item fast enough); loads / atomics / stores of a phase issued in separate batches (the pipeline is throughput-, not
// latency-bound).  The kernel is bound by the shared-memory pipeline, not by HBM.
// NDMAX = 256 or 1024 digits: the second level of a large bin uses up to 10 bits, so that a leaf still holds ~1 K records
// (the wider variant has one TMA buffer less: shared memory).
template <int WORDS, int NDMAX = 256>
struct MsdSmem {
	static constexpr int kThreads = MsdCfg<WORDS>::kThreads;          // consumer threads
	static constexpr int kKpt = MsdCfg<WORDS>::kKpt;
	static constexpr int kTile = kThreads * kKpt;
	static constexpr int kRecBytes = 8 * WORDS;
	static constexpr int kStages = NDMAX > 256 ? 2 : 3;
	static constexpr int kBufStride = ((kTile + 2) * kRecBytes + 127) & ~127;   // + 2: the aligned load may start one record early / end one late
	static constexpr int oBuf = 0;
	static constexpr int oHist = kStages * kBufStride;             // u32 [NDMAX]
	static constexpr int oExcl = oHist + 4 * NDMAX;                // u32 [NDMAX]
	static constexpr int oGoff = oExcl + 4 * NDMAX;                // u32 [NDMAX]
	static constexpr int oBase = oGoff + 4 * NDMAX;                // u32 [kStages][NDMAX] output base of (item, digit)
	static constexpr int oWarpTot = oBase + kStages * 4 * NDMAX;   // u32 [8]
	static constexpr int oGeom = oWarpTot + 64;                    // u32 [kStages][4]: head, valid
	static constexpr int oMbar = oGeom + kStages * 16;             // u64 full[kStages], empty[kStages]
	static constexpr int kBytes = oMbar + 2 * kStages * 8;
};

__device__ __forceinline__ void bar_sync_named(uint32_t id, uint32_t n_threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }

struct MsdPartArgs {
	const void* in;
	void* out;
	MsdItems items;
	const uint32_t* cell_scan;   // exclusive scan of the cells = global output index of (item, digit)
	uint32_t shift, nd;          // digit = bits [shift, shift + log2(nd)), nd <= 256
	const uint32_t* flags;
};

template <int WORDS, int NDMAX = 256>
__global__ void __launch_bounds__(MsdCfg<WORDS>::kThreads + 32, MsdCfg<WORDS>::kMinBlocks) msd_partition_kernel(const MsdPartArgs p)
{
	using S = MsdSmem<WORDS, NDMAX>;
	using R = Rec<WORDS>;
	constexpr int THREADS = S::kThreads, KPT = S::kKpt, STAGES = S::kStages;
	constexpr int DPT = NDMAX / 256;               // digits per scanning thread (threads 0..255)
	extern __shared__ __align__(128) uint8_t smem[];
	uint32_t* hist = reinterpret_cast<uint32_t*>(smem + S::oHist);
	uint32_t* tile_excl = reinterpret_cast<uint32_t*>(smem + S::oExcl);
	uint32_t* goff = reinterpret_cast<uint32_t*>(smem + S::oGoff);
	uint32_t* s_base = reinterpret_cast<uint32_t*>(smem + S::oBase);
	uint32_t* warp_tot = reinterpret_cast<uint32_t*>(smem + S::oWarpTot);
	uint32_t* s_geom = reinterpret_cast<uint32_t*>(smem + S::oGeom);
	uint64_t* full = reinterpret_cast<uint64_t*>(smem + S::oMbar);
	uint64_t* empty = full + STAGES;

	if (*p.flags & kMsdFlagStop) return;
	const uint32_t tid = threadIdx.x;
	const R* __restrict__ gin = reinterpret_cast<const R*>(p.in);
	R* __restrict__ gout = reinterpret_cast<R*>(p.out);
	const uint32_t n_items = *p.items.n_items;
	const uint32_t mask = p.nd - 1;

	if (tid == 0) {
#pragma unroll
		for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }
		fence_mbar_init();
	}
	for (uint32_t d = tid; d < (uint32_t)NDMAX; d += blockDim.x) hist[d] = 0;
	__syncthreads();

	// items of a CTA: round robin.  (One contiguous block of items per CTA - so that the bases of consecutive items of a digit share sectors
	// of the cell scan - was slower.)
	const uint32_t item_begin = blockIdx.x, item_end = n_items, item_step = gridDim.x;
	if (tid >= (uint32_t)THREADS) {
		// ---------------------------------------------------------------- producer warp
		const uint32_t lane = tid & 31u;
		uint32_t it = 0;
		for (uint32_t item = item_begin; item < item_end; item += item_step, ++it) {
			const uint32_t st = it % STAGES;
			if (it >= (uint32_t)STAGES) mbar_wait(&empty[st], ((it / STAGES) - 1u) & 1u);      // the consumers are done with this buffer
			const MsdItemGeom g = msd_item_geom<WORDS>(p.items, item, p.nd);
#pragma unroll 8
			for (int i = 0; i < NDMAX / 32; ++i) {
				const uint32_t d = i * 32 + lane;
				s_base[st * NDMAX + d] = d < p.nd ? __ldg(p.cell_scan + g.cell0 + (uint64_t)d * g.cell_stride) : 0u;
			}
			if (lane == 0) { s_geom[st * 4 + 0] = (uint32_t)(g.lo - g.lo_al); s_geom[st * 4 + 1] = (uint32_t)(g.hi - g.lo); }
			__syncwarp();
			if (lane == 0) {
				const uint32_t bytes = g.n_load * S::kRecBytes;
				fence_proxy_async();
				mbar_arrive_expect_tx(&full[st], bytes);
				bulk_g2s(smem + S::oBuf + st * S::kBufStride, gin + g.lo_al, bytes, &full[st]);
			}
		}
		return;
	}

	// -------------------------------------------------------------------- consumers (named barrier 1: the producer is not part of it)
	const uint32_t lane = tid & 31u, warp = tid >> 5;
	uint32_t it = 0;
	for (uint32_t item = item_begin; item < item_end; item += item_step, ++it) {
		const uint32_t st = it % STAGES;
		mbar_wait(&full[st], (it / STAGES) & 1u);
		const uint32_t head = s_geom[st * 4 + 0], valid = s_geom[st * 4 + 1];
		R* buf = reinterpret_cast<R*>(smem + S::oBuf + st * S::kBufStride);

		// ---- rank inside (tile, digit) = return value of one shared-memory atomicAdd (an MSD partition need not be stable)
		R key[KPT];
		uint16_t rank[KPT];
#pragma unroll
		for (int r = 0; r < KPT; ++r) {
			const uint32_t j = r * THREADS + tid;
			if (j < valid) {
				key[r] = buf[head + j];
				rank[r] = (uint16_t)atomicAdd(&hist[rec_bits<WORDS>(key[r], p.shift, mask)], 1u);
			}
		}
		bar_sync_named(1, THREADS);

		// ---- exclusive scan of the digit counts (warps 0..7, DPT consecutive digits per thread); every thread zeroes its own bins for the next item
		uint32_t cnt[DPT], tot = 0, inc = 0;
		if (tid < 256) {
#pragma unroll
			for (int i = 0; i < DPT; ++i) { cnt[i] = hist[tid * DPT + i]; hist[tid * DPT + i] = 0; tot += cnt[i]; }
			inc = tot;
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) {
				const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
				if (lane >= (uint32_t)o) inc += t;
			}
			if (lane == 31) warp_tot[warp] = inc;
		}
		bar_sync_named(1, THREADS);
		if (tid < 256) {
			uint32_t texcl = inc - tot;
#pragma unroll
			for (int w = 0; w < 8; ++w) if ((uint32_t)w < warp) texcl += warp_tot[w];
#pragma unroll
			for (int i = 0; i < DPT; ++i) {
				tile_excl[tid * DPT + i] = texcl;
				goff[tid * DPT + i] = s_base[st * NDMAX + tid * DPT + i] - texcl;          // global index of tile-sorted position q is goff[d] + q
				texcl += cnt[i];
			}
		}
		bar_sync_named(1, THREADS);

		// ---- regroup by digit in shared memory (every record is in registers, the buffer is free)
#pragma unroll
		for (int r = 0; r < KPT; ++r) {
			const uint32_t j = r * THREADS + tid;
			if (j < valid) buf[tile_excl[rec_bits<WORDS>(key[r], p.shift, mask)] + rank[r]] = key[r];
		}
		bar_sync_named(1, THREADS);

		// ---- digit-contiguous runs leave with coalesced stores
#pragma unroll
		for (int i = 0; i < KPT; ++i) {
			const uint32_t q = i * THREADS + tid;
			if (q < valid) {
				const R k = buf[q];
				gout[goff[rec_bits<WORDS>(k, p.shift, mask)] + q] = k;
			}
		}
		fence_proxy_async();                   // our generic-proxy writes to the buffer, before the next TMA copy into it
		bar_sync_named(1, THREADS);
		if (tid == 0) mbar_arrive(&empty[st]);
	}
}

// ---------------------------------------------------------------------------------------------
// counts of the next digit per item, written straight into the cell layout (u16)
struct MsdCountArgs {
	const void* in;
	MsdItems items;
	uint32_t shift, nd;
	uint16_t* cells;
	const uint32_t* flags;
};

template <int WORDS, int NDMAX = 256>
__global__ void __launch_bounds__(512) msd_count_kernel(const MsdCountArgs p)
{
	using R = Rec<WORDS>;
	__shared__ uint32_t sh[2][NDMAX];
	if (*p.flags & kMsdFlagStop) return;
	const R* __restrict__ g = reinterpret_cast<const R*>(p.in);
	const uint32_t n_items = *p.items.n_items;
	const uint32_t mask = p.nd - 1;
	const uint32_t tid = threadIdx.x;
	constexpr int U = (msd_tile<WORDS>() + 511) / 512;
	for (uint32_t d = tid; d < (uint32_t)NDMAX; d += 512) { sh[0][d] = 0; sh[1][d] = 0; }
	// software pipeline: the records of the next item are in flight while this one is counted; one barrier per item
	uint32_t item = blockIdx.x;
	MsdItemGeom gm{};
	uint32_t m = 0;
	R k[U];
	if (item < n_items) {
		gm = msd_item_geom<WORDS>(p.items, item, p.nd);
		m = (uint32_t)(gm.hi - gm.lo);
#pragma unroll
		for (int u = 0; u < U; ++u) { const uint32_t j = u * 512 + tid; if (j < m) k[u] = g[gm.lo + j]; }
	}
	__syncthreads();
	int cur = 0;
	while (item < n_items) {
#pragma unroll
		for (int u = 0; u < U; ++u) { const uint32_t j = u * 512 + tid; if (j < m) atomicAdd(&sh[cur][rec_bits<WORDS>(k[u], p.shift, mask)], 1u); }
		const MsdItemGeom done = gm;
		item += gridDim.x;
		if (item < n_items) {
			gm = msd_item_geom<WORDS>(p.items, item, p.nd);
			m = (uint32_t)(gm.hi - gm.lo);
#pragma unroll
			for (int u = 0; u < U; ++u) { const uint32_t j = u * 512 + tid; if (j < m) k[u] = g[gm.lo + j]; }
		}
		__syncthreads();
		for (uint32_t d = tid; d < (uint32_t)NDMAX; d += 512) {          // (a bin is read and zeroed by its own thread; it is used again two items later, a barrier in between)
			if (d < p.nd) p.cells[done.cell0 + (uint64_t)d * done.cell_stride] = (uint16_t)sh[cur][d];
			sh[cur][d] = 0;
		}
		cur ^= 1;
	}
}

// ---------------------------------------------------------------------------------------------
// flat exclusive scan over u16 cells -> u32 (three small kernels; the number of cells lives on the device)
constexpr int kCellChunk = 4096;     // cells per block

// 16 consecutive cells of a thread as two 16-byte loads (a vector that starts inside the array may end <= 15 cells behind it: the cell
// array is over-allocated by an eighth, and those values are masked)
__device__ __forceinline__ void cell_load16(const uint16_t* cells, uint64_t c, uint64_t n_cells, uint32_t (&v)[16])
{
	uint4 a = make_uint4(0, 0, 0, 0), b = a;
	if (c < n_cells) { a = __ldg(reinterpret_cast<const uint4*>(cells + c)); b = __ldg(reinterpret_cast<const uint4*>(cells + c) + 1); }
	const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
	for (int i = 0; i < 8; ++i) {
		v[2 * i] = c + 2 * i < n_cells ? (w[i] & 0xFFFFu) : 0u;
		v[2 * i + 1] = c + 2 * i + 1 < n_cells ? (w[i] >> 16) : 0u;
	}
}

__global__ void __launch_bounds__(256) cell_reduce_kernel(const uint16_t* cells, const uint32_t* n_items, uint32_t nd, uint32_t* block_sums, const uint32_t* flags)
{
	__shared__ uint32_t s_w[8];
	if (*flags & kMsdFlagStop) return;
	const uint64_t n_cells = (uint64_t)nd * *n_items;
	const uint64_t c0 = (uint64_t)blockIdx.x * kCellChunk;
	if (c0 >= n_cells) return;
	uint32_t v[16];
	cell_load16(cells, c0 + (uint64_t)threadIdx.x * 16, n_cells, v);
	uint32_t sum = 0;
#pragma unroll
	for (int i = 0; i < 16; ++i) sum += v[i];
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
	if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = sum;
	__syncthreads();
	if (threadIdx.x == 0) {
		uint32_t t = 0;
		for (int w = 0; w < 8; ++w) t += s_w[w];
		block_sums[blockIdx.x] = t;
	}
}

__global__ void __launch_bounds__(1024) cell_scan_sums_kernel(uint32_t* block_sums, const uint32_t* n_items, uint32_t nd, const uint32_t* flags)
{
	__shared__ uint32_t s_w[32];
	__shared__ uint32_t carry;
	if (*flags & kMsdFlagStop) return;
	const uint64_t n_cells = (uint64_t)nd * *n_items;
	const uint32_t nb = (uint32_t)((n_cells + kCellChunk - 1) / kCellChunk);
	const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid == 0) carry = 0;
	__syncthreads();
	for (uint32_t b0 = 0; b0 < nb; b0 += 1024) {
		const uint32_t b = b0 + tid;
		const uint32_t v = b < nb ? block_sums[b] : 0;
		uint32_t inc = v;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
			if (lane >= (uint32_t)o) inc += t;
		}
		if (lane == 31) s_w[warp] = inc;
		__syncthreads();
		uint32_t base = carry;
		for (uint32_t w = 0; w < warp; ++w) base += s_w[w];
		if (b < nb) block_sums[b] = base + inc - v;
		__syncthreads();
		if (tid == 1023) carry = base + inc;
		__syncthreads();
	}
}

__global__ void __launch_bounds__(256) cell_scan_kernel(const uint16_t* cells, const uint32_t* n_items, uint32_t nd, const uint32_t* block_sums, uint32_t* out, const uint32_t* flags)
{
	static_assert(kCellChunk == 256 * 16, "16 consecutive cells per thread");
	__shared__ uint32_t s_w[8];
	__shared__ uint32_t s_t[kCellChunk + kCellChunk / 16];       // the chunk's prefixes, padded (index i lives at i + i / 16): transposed for coalesced stores
	if (*flags & kMsdFlagStop) return;
	const uint64_t n_cells = (uint64_t)nd * *n_items;
	const uint64_t c0 = (uint64_t)blockIdx.x * kCellChunk;
	if (c0 >= n_cells) return;
	const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	uint32_t v[16];
	cell_load16(cells, c0 + (uint64_t)tid * 16, n_cells, v);
	uint32_t sum = 0;
#pragma unroll
	for (int i = 0; i < 16; ++i) sum += v[i];
	uint32_t inc = sum;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
		if (lane >= (uint32_t)o) inc += t;
	}
	if (lane == 31) s_w[warp] = inc;
	__syncthreads();
	uint32_t base = block_sums[blockIdx.x] + inc - sum;
	for (uint32_t w = 0; w < warp; ++w) base += s_w[w];
#pragma unroll
	for (int i = 0; i < 16; ++i) {           // thread t owns padded words 17 t .. 17 t + 15: conflict-free
		s_t[tid * 17 + i] = base;
		base += v[i];
	}
	__syncthreads();
#pragma unroll
	for (int i = 0; i < 16; ++i) {
		const uint32_t j = i * 256 + tid;
		if (c0 + j < n_cells) out[c0 + j] = s_t[j + (j >> 4)];
	}
}

// ---------------------------------------------------------------------------------------------
// single CTA: boundaries of the buckets a partition level produced (= scan value of the first item's cell of every (segment, digit)),
// optional oversize check, optional work-item table (aligned tiles) over the NEW buckets for the next level.
struct MsdBoundsArgs {
	const uint32_t* cell_scan;
	MsdItems items;              // the items of the level that was just scanned
	uint32_t S, nd;              // its segments and digits: M = S * nd new buckets
	uint64_t n;                  // records in total
	uint64_t* start;             // [M + 1]
	uint32_t cap;                // 0: no check
	uint32_t* flags;
	uint32_t tile;               // items of the next level (0: none)
	uint32_t* item_base;         // [M + 1]
	uint32_t* item_seg;
	uint32_t* n_items;
	// level 1 of the bin path (expand.cuh, kExpandPartition; msd_bounds_kernel only): the boundaries are the exclusive scan of these
	// 256 digit totals instead of scanned cells, and every bucket's cursor starts at its boundary
	const uint32_t* l1_total;    // [256] or nullptr
	uint32_t* l1_cursor;         // [256]
	uint32_t* status;            // expand status: kErrRecCount when the totals do not add up to n
};

// boundaries + oversize check only (any number of CTAs): used when no item table is needed
__global__ void __launch_bounds__(256) msd_bounds_flat_kernel(const MsdBoundsArgs a)
{
	if (*a.flags & kMsdFlagStop) return;
	const uint32_t M = a.S * a.nd;
	const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
	if (m > M) return;
	auto bound = [&](uint32_t q) -> uint64_t {
		if (q >= M) return a.n;
		const uint32_t seg = q / a.nd, d = q % a.nd;
		if (a.items.item_lo) return a.cell_scan[(uint64_t)d * *a.items.n_items];
		const uint32_t first = a.items.item_base[seg], nis = a.items.item_base[seg + 1] - first;
		return nis ? (uint64_t)a.cell_scan[(uint64_t)a.nd * first + (uint64_t)d * nis] : a.items.seg_start[seg];
	};
	const uint64_t v = bound(m);
	a.start[m] = v;
	if (a.cap && m < M && bound(m + 1) - v > a.cap) atomicOr(a.flags, kMsdFlagFallback);
}

__global__ void __launch_bounds__(1024) msd_bounds_kernel(const MsdBoundsArgs a)
{
	__shared__ uint32_t s_i[32];
	__shared__ uint32_t carry_i;
	const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (*a.flags & kMsdFlagStop) return;
	const uint32_t M = a.S * a.nd;
	// pass 1: boundaries.  Buckets of an empty segment (no items, no cells) collapse onto the segment start.
	if (a.l1_total) {          // (M = 256 digits of one segment, n < 2^32)
		const uint32_t c = tid < M ? a.l1_total[tid] : 0u;
		uint32_t inc = c;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
			if (lane >= (uint32_t)o) inc += t;
		}
		if (lane == 31) s_i[warp] = inc;
		__syncthreads();
		uint32_t ex = inc - c;
		for (uint32_t w = 0; w < warp; ++w) ex += s_i[w];
		if (tid < M) { a.start[tid] = ex; a.l1_cursor[tid] = ex; }
		if (tid == M) a.start[M] = a.n;
		if (tid == M - 1) carry_i = ex + c;
		__syncthreads();
		if (carry_i != a.n) {          // the walk counted other k-mers than the bin holds (a bug): a bin error, nothing runs behind
			if (tid == 0) { atomicOr(a.status, kErrRecCount); atomicOr(&a.flags[0], kMsdFlagAbort); atomicOr(&a.flags[1], kMsdFlagAbort); }
			return;
		}
	} else
	for (uint32_t m = tid; m <= M; m += 1024) {
		uint64_t v = a.n;
		if (m < M) {
			const uint32_t seg = m / a.nd, d = m % a.nd;
			if (a.items.item_lo) v = a.cell_scan[(uint64_t)d * *a.items.n_items];
			else {
				const uint32_t first = a.items.item_base[seg], nis = a.items.item_base[seg + 1] - first;
				v = nis ? (uint64_t)a.cell_scan[(uint64_t)a.nd * first + (uint64_t)d * nis] : a.items.seg_start[seg];
			}
		}
		a.start[m] = v;
	}
	__threadfence();
	__syncthreads();
	if (tid == 0) carry_i = 0;
	__syncthreads();
	bool over = false;
	for (uint32_t base = 0; base < M; base += 1024) {
		const uint32_t m = base + tid;
		uint64_t sb = 0, c = 0;
		if (m < M) { sb = a.start[m]; c = a.start[m + 1] - sb; }
		if (a.cap && c > a.cap) over = true;
		uint32_t ni = 0;
		if (a.tile && c) ni = (uint32_t)((sb + c - 1) / a.tile - sb / a.tile) + 1;
		uint32_t ii = ni;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xffffffffu, ii, o);
			if (lane >= (uint32_t)o) ii += t;
		}
		if (lane == 31) s_i[warp] = ii;
		__syncthreads();
		uint32_t bi = carry_i;
		for (uint32_t w = 0; w < warp; ++w) bi += s_i[w];
		const uint32_t ei = bi + ii - ni;
		if (a.tile && m < M) a.item_base[m] = ei;
		__syncthreads();
		if (tid == 1023) carry_i = ei + ni;
		__syncthreads();
	}
	if (tid == 0 && a.tile) { a.item_base[M] = carry_i; *a.n_items = carry_i; }
	if (over) atomicOr(a.flags, kMsdFlagFallback);
	// the segment of every item: one WARP per bucket (after level 1 there are 256 buckets of ~100 items each: a thread per bucket writing
	// its items one after the other took 35 us of this kernel's 36)
	if (a.tile) {
		__syncthreads();          // item_base[] of this CTA's threads is visible
		for (uint32_t m = warp; m < M; m += 32) {
			const uint32_t e0 = a.item_base[m], e1 = a.item_base[m + 1];
			for (uint32_t i = e0 + lane; i < e1; i += 32) a.item_seg[i] = m;
		}
	}
}

// ---------------------------------------------------------------------------------------------
// leaves: one bucket per CTA iteration, sorted on chip by 8-bit LSD passes over its low `low_bits` bits
struct MsdLocalArgs {
	const void* in;
	void* out;
	const uint64_t* start;       // [n_buckets + 1]
	uint32_t n_buckets;
	uint32_t low_bits;           // bits below the partition digits
	uint32_t* bucket_counter;
	const uint32_t* flags;
};

// lanes of the warp whose 8-bit digit equals this lane's: 8 ballots instead of match.any (microcoded; scripts/ubench measures both)
__device__ __forceinline__ uint32_t match_digit8(uint32_t d)
{
	uint32_t peers = 0xffffffffu;
#pragma unroll
	for (int b = 0; b < 8; ++b) {
		const uint32_t m = __ballot_sync(0xffffffffu, (d >> b) & 1u);
		peers &= ((d >> b) & 1u) ? m : ~m;
	}
	return peers;
}

template <int WORDS> struct MsdLocalCfg;
template <> struct MsdLocalCfg<1> { static constexpr int kThreads = 256, kKpt = 16; };
template <> struct MsdLocalCfg<2> { static constexpr int kThreads = 256, kKpt = 8; };
template <> struct MsdLocalCfg<3> { static constexpr int kThreads = 256, kKpt = 5; };
template <> struct MsdLocalCfg<4> { static constexpr int kThreads = 256, kKpt = 4; };
template <int WORDS> __host__ __device__ constexpr int msd_local_cap() { return MsdLocalCfg<WORDS>::kThreads * MsdLocalCfg<WORDS>::kKpt; }

template <int WORDS>
__global__ void __launch_bounds__(MsdLocalCfg<WORDS>::kThreads) msd_local_sort_kernel(const MsdLocalArgs p)
{
	using R = Rec<WORDS>;
	constexpr int THREADS = MsdLocalCfg<WORDS>::kThreads, KPT = MsdLocalCfg<WORDS>::kKpt, WARPS = THREADS / 32, CAP = THREADS * KPT;
	extern __shared__ __align__(16) uint8_t dsm[];
	R* buf = reinterpret_cast<R*>(dsm);                                                 // [CAP]
	uint32_t* whist = reinterpret_cast<uint32_t*>(dsm + (size_t)CAP * sizeof(R));       // [WARPS][256]
	__shared__ uint32_t tile_excl[256];
	__shared__ uint64_t warp_tot[8];
	__shared__ uint32_t s_bucket;

	if (*p.flags & kMsdFlagStop) return;
	const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
	const R* __restrict__ gin = reinterpret_cast<const R*>(p.in);
	R* __restrict__ gout = reinterpret_cast<R*>(p.out);
	uint32_t* wh = whist + warp * 256;

	while (true) {
		__syncthreads();
		if (tid == 0) s_bucket = atomicAdd(p.bucket_counter, 1u);
		__syncthreads();
		const uint32_t b = s_bucket;
		if (b >= p.n_buckets) break;
		const uint64_t lo = p.start[b];
		const uint32_t m = (uint32_t)(p.start[b + 1] - lo);
		if (m == 0) continue;
		// records to registers: warp w owns [w*32*kpt, ...), round r = 32 consecutive records (stable order = index order).  kpt = the rounds
		// this leaf needs (a leaf of ~1 K records fills 4 of the 16 rounds the capacity allows: the others are skipped, not padded)
		const uint32_t kpt = (m + THREADS - 1) / THREADS;
		R key[KPT];
#pragma unroll
		for (int r = 0; r < KPT; ++r) {
			if ((uint32_t)r >= kpt) break;
			const uint32_t idx = warp * (32 * kpt) + r * 32 + lane;
			if (idx < m) key[r] = gin[lo + idx];
			else {
#pragma unroll
				for (int j = 0; j < WORDS; ++j) key[r].w[j] = ~0ull;       // padding: largest possible key, stays at the end
			}
		}
		if (m > 1) {
			for (uint32_t shift = 0; shift < p.low_bits; shift += 8) {
				const uint32_t mask = (p.low_bits - shift) >= 8 ? 0xFFu : ((1u << (p.low_bits - shift)) - 1u);
				// padding must keep sorting last: its digit is forced to the largest value of this pass
#pragma unroll
				for (int i = tid; i < WARPS * 256; i += THREADS) whist[i] = 0;
				__syncthreads();
				uint32_t dg[KPT];
#pragma unroll
				for (int r = 0; r < KPT; ++r) {
					if ((uint32_t)r >= kpt) break;
					const uint32_t idx = warp * (32 * kpt) + r * 32 + lane;
					dg[r] = idx < m ? rec_bits<WORDS>(key[r], shift, mask) : mask;
					atomicAdd(&wh[dg[r]], 1u);
				}
				__syncthreads();
				uint32_t cnt = 0;
#pragma unroll
				for (int w = 0; w < WARPS; ++w) {
					const uint32_t t = whist[w * 256 + tid];
					whist[w * 256 + tid] = cnt;
					cnt += t;
				}
				const uint64_t texcl = block_excl_scan_256(cnt, warp_tot, nullptr);
				tile_excl[tid] = (uint32_t)texcl;
				__syncthreads();
				uint32_t peers[KPT];
#pragma unroll
				for (int r = 0; r < KPT; ++r) { if ((uint32_t)r >= kpt) break; peers[r] = match_digit8(dg[r]); }
#pragma unroll
				for (int r = 0; r < KPT; ++r) {
					if ((uint32_t)r >= kpt) break;
					const uint32_t d = dg[r];
					const uint32_t mm = peers[r];
					const uint32_t below = __popc(mm & lanemask_lt());
					const int leader = __ffs(mm) - 1;
					uint32_t old = 0;
					if ((int)lane == leader) {
						old = wh[d];
						wh[d] = old + __popc(mm);
					}
					old = __shfl_sync(0xffffffffu, old, leader);
					buf[tile_excl[d] + old + below] = key[r];
					__syncwarp();
				}
				__syncthreads();
#pragma unroll
				for (int r = 0; r < KPT; ++r) { if ((uint32_t)r >= kpt) break; key[r] = buf[warp * (32 * kpt) + r * 32 + lane]; }
				// (the next pass synchronises before it writes to buf again)
			}
		}
#pragma unroll
		for (int r = 0; r < KPT; ++r) {
			if ((uint32_t)r >= kpt) break;
			const uint32_t idx = warp * (32 * kpt) + r * 32 + lane;
			if (idx < m) gout[lo + idx] = key[r];
		}
	}
}

}  // namespace kmcb
