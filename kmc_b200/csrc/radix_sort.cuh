// kmc_b200 — 8-bit radix sort of packed k-mer records (replaces the reference's sort_func:
// RADULS kmc_core/raduls_impl.h:546-776 + first_dispatch.h:98-435, or radix.h:845-855 + small_sort.h).
//
// Contract kept (raduls.h:19-20, kb_sorter.h:757-780): ascending order on bytes key_bytes-1..0 of the
// record image.  Records are pure keys (no payload), so the sorted array is unique and any stable or
// unstable correct sort is bit-identical to RADULS' output.
//
// Design: one kernel launch per 8-bit digit, each pass exactly one read + one write of every
// record ("onesweep": chained scan with decoupled look-back gives every tile its global bucket
// offsets inside the same kernel).  Per pass and CTA:
//   * tiles are fetched global->shared with TMA 1-D bulk copies (cp.async.bulk + mbarrier),
//     double buffered: tile i+1 is in flight while tile i is ranked;
//   * ranks come from warp-private digit histograms in shared memory driven by match.any + popc
//     (warp-shuffle broadcast of the bucket cursor) - no atomics on the ranking path;
//   * records are regrouped by digit in shared memory and leave as digit-contiguous runs
//     (TILE/256 records = 128-256 B on average), so global stores are fully coalesced;
//   * the histogram of the NEXT digit is accumulated on the fly (the multiset of records does not
//     depend on their order), so no pass ever re-reads the data just to count:  traffic = 2*N*W / pass.
#pragma once
#include "common.cuh"
#include <cooperative_groups.h>

namespace kmcb {

struct SortPass {
	const void* in;          // N records
	void* out;               // N records
	uint64_t n;
	uint32_t n_tiles;
	uint32_t byte;           // digit = byte `byte` of the record image
	int32_t next_byte;       // digit whose histogram is accumulated for the following pass, -1: none
	const uint64_t* hist;    // [256] histogram of `byte` over all N records
	uint64_t* hist_next;     // [256] zero-initialised
	uint64_t* desc;          // [n_tiles][256] look-back descriptors (epoch-tagged, see common.cuh)
	uint32_t epoch;          // unique per launch
	uint32_t* tile_counter;  // zero-initialised
	const uint32_t* run_flag; // nullptr: always run; else run only when (*run_flag & kRunMask) == run_need (msd_sort.cuh: bit 0 = the hybrid
	uint32_t run_need;        // MSD path gave up, bit 1 = the bin is malformed and nothing may run)
};
constexpr uint32_t kRunMask = 3u;
__device__ __forceinline__ bool run_allowed(const uint32_t* flag, uint32_t need) { return !flag || (*flag & kRunMask) == need; }

template <int WORDS> struct SortCfg;
template <> struct SortCfg<1> { static constexpr int kThreads = 512, kKpt = 8, kMinBlocks = 2; };
template <> struct SortCfg<2> { static constexpr int kThreads = 512, kKpt = 4, kMinBlocks = 2; };
template <> struct SortCfg<3> { static constexpr int kThreads = 512, kKpt = 3, kMinBlocks = 2; };
template <> struct SortCfg<4> { static constexpr int kThreads = 512, kKpt = 2, kMinBlocks = 2; };

template <int WORDS>
struct SortSmem {
	static constexpr int kThreads = SortCfg<WORDS>::kThreads;
	static constexpr int kWarps = kThreads / 32;
	static constexpr int kKpt = SortCfg<WORDS>::kKpt;
	static constexpr int kTile = kThreads * kKpt;
	static constexpr int kRecBytes = 8 * WORDS;
	static constexpr int kBufBytes = kTile * kRecBytes;
	// byte offsets inside dynamic shared memory
	static constexpr int oBuf = 0;
	static constexpr int oWhist = 2 * kBufBytes;              // u32 [kWarps][256]
	static constexpr int oTileExcl = oWhist + kWarps * 1024;  // u32 [256]
	static constexpr int oGoff = oTileExcl + 1024;            // u64 [256]
	static constexpr int oNhist = oGoff + 2048;               // u32 [256]
	static constexpr int oWarpTot = oNhist + 1024;            // u32 [32]
	static constexpr int oMbar = oWarpTot + 128;              // u64 [2]
	static constexpr int oTileId = oMbar + 16;                // u32 [2]
	static constexpr int kBytes = oTileId + 16;
};

// exclusive scan of one value per thread over the first 256 threads (8 warps); all threads must call.
__device__ __forceinline__ uint64_t block_excl_scan_256(uint64_t v, uint64_t* warp_tot /* smem [8] */, uint64_t* total)
{
	const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	uint64_t inc = v;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		uint64_t t = __shfl_up_sync(0xffffffffu, inc, o);
		if (lane >= (uint32_t)o) inc += t;
	}
	if (warp < 8 && lane == 31) warp_tot[warp] = inc;
	__syncthreads();
	uint64_t base = 0, tot = 0;
#pragma unroll
	for (int w = 0; w < 8; ++w) {
		uint64_t t = warp_tot[w];
		if ((uint32_t)w < warp) base += t;
		tot += t;
	}
	if (total) *total = tot;
	__syncthreads();
	return base + inc - v;
}

// One pass over all tiles by this CTA (persistent: tiles are claimed from p.tile_counter).  The mbarriers live across passes
// (phase0 / phase1 are the caller's running parities); nhist must be zero on entry and is left zero on exit.
template <int WORDS>
__device__ __forceinline__ void radix_pass_body(const SortPass& p, uint8_t* smem, uint32_t& phase0, uint32_t& phase1)
{
	using S = SortSmem<WORDS>;
	using R = Rec<WORDS>;
	constexpr int THREADS = S::kThreads, WARPS = S::kWarps, KPT = S::kKpt, TILE = S::kTile;
	uint32_t* whist = reinterpret_cast<uint32_t*>(smem + S::oWhist);
	uint32_t* tile_excl = reinterpret_cast<uint32_t*>(smem + S::oTileExcl);
	uint64_t* goff = reinterpret_cast<uint64_t*>(smem + S::oGoff);
	uint32_t* nhist = reinterpret_cast<uint32_t*>(smem + S::oNhist);
	uint64_t* warp_tot = reinterpret_cast<uint64_t*>(smem + S::oWarpTot);
	uint64_t* mbar = reinterpret_cast<uint64_t*>(smem + S::oMbar);
	volatile uint32_t* s_tile = reinterpret_cast<volatile uint32_t*>(smem + S::oTileId);

	const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
	const R* __restrict__ gin = reinterpret_cast<const R*>(p.in);
	R* __restrict__ gout = reinterpret_cast<R*>(p.out);
	uint64_t* desc = p.desc;

	// bucket bases of this pass: exclusive scan of the digit histogram (thread d <-> digit d)
	uint64_t bucket_base = block_excl_scan_256(tid < 256 ? p.hist[tid] : 0, warp_tot, nullptr);

	auto issue_load = [&](uint32_t tile, int b) {
		// called by thread 0 only
		const uint64_t first = (uint64_t)tile * TILE;
		const uint64_t rem = p.n - first;
		const uint32_t valid = rem < (uint64_t)TILE ? (uint32_t)rem : (uint32_t)TILE;
		const uint32_t bytes = valid * S::kRecBytes;
		if ((bytes & 15u) == 0) {       // TMA path; an odd-sized last tile is fetched by all threads when it is consumed
			fence_proxy_async();
			mbar_arrive_expect_tx(&mbar[b], bytes);
			bulk_g2s(smem + S::oBuf + b * S::kBufBytes, gin + first, bytes, &mbar[b]);
		}
	};

	if (tid == 0) {
		uint32_t t = atomicAdd(p.tile_counter, 1u);
		s_tile[0] = t;
		if (t < p.n_tiles) issue_load(t, 0);
	}
	__syncthreads();

	uint32_t cnt_real = 0;
	int cur = 0;
	while (true) {
		const uint32_t tile = s_tile[cur];
		if (tile >= p.n_tiles) break;
		if (tid == 0) {   // claim and prefetch the next tile of this CTA
			uint32_t t = atomicAdd(p.tile_counter, 1u);
			s_tile[cur ^ 1] = t;
			if (t < p.n_tiles) issue_load(t, cur ^ 1);
		}
		const uint64_t first = (uint64_t)tile * TILE;
		const uint64_t rem = p.n - first;
		const uint32_t valid = rem < (uint64_t)TILE ? (uint32_t)rem : (uint32_t)TILE;
		R* buf = reinterpret_cast<R*>(smem + S::oBuf + cur * S::kBufBytes);

		// zero the warp-private histograms
#pragma unroll
		for (int i = tid; i < WARPS * 256; i += THREADS) whist[i] = 0;

		if (((valid * S::kRecBytes) & 15u) == 0) {
			if (cur == 0) { mbar_wait(&mbar[0], phase0); phase0 ^= 1; }
			else { mbar_wait(&mbar[1], phase1); phase1 ^= 1; }
		} else {
			for (uint32_t i = tid; i < valid; i += THREADS) buf[i] = gin[first + i];
		}
		__syncthreads();

		// ---- phase 1: every record into registers + warp-private digit counts (shared-memory atomics, conflicts only inside a warp).
		// Warp w owns records [w*32*KPT, (w+1)*32*KPT) of the tile, round r covers 32 consecutive ones.
		R key[KPT];
		uint32_t* wh = whist + warp * 256;
#pragma unroll
		for (int r = 0; r < KPT; ++r) {
			const uint32_t idx = warp * (32 * KPT) + r * 32 + lane;
			if (idx < valid) key[r] = buf[idx];
			else {
#pragma unroll
				for (int j = 0; j < WORDS; ++j) key[r].w[j] = ~0ull;     // padding sorts to the very end of digit 255
			}
			atomicAdd(&wh[rec_byte<WORDS>(key[r], p.byte)], 1u);
		}
		__syncthreads();

		// ---- phase 2, digit d (thread d): offsets of every warp inside the digit's run, tile count; the aggregate is
		// published BEFORE the expensive ranking so that later tiles almost never wait in their look-back
		uint32_t cnt = 0;
		if (tid < 256) {
#pragma unroll
			for (int w = 0; w < WARPS; ++w) {
				uint32_t t = whist[w * 256 + tid];
				whist[w * 256 + tid] = cnt;
				cnt += t;
			}
			uint32_t real = cnt;
			if (tid == 255) real -= (TILE - valid);       // padding records are not published
			st_relaxed(desc + (uint64_t)tile * 256 + tid, desc_pack(tile == 0 ? kDescPrefix : kDescAggregate, p.epoch, real));
			cnt_real = real;
		}
		const uint64_t texcl = block_excl_scan_256(cnt, warp_tot, nullptr);
		if (tid < 256) tile_excl[tid] = (uint32_t)texcl;
		__syncthreads();

		// ---- phase 3: stable ranks from match.any + the warp's running bucket cursor; regroup by digit in shared memory
		// (the tile buffer is dead: every record is in registers).  All match.any are issued first (independent, their
		// latency overlaps); only the short cursor update is a serial chain over the rounds.
		uint32_t peers[KPT];
#pragma unroll
		for (int r = 0; r < KPT; ++r) peers[r] = __match_any_sync(0xffffffffu, rec_byte<WORDS>(key[r], p.byte));
#pragma unroll
		for (int r = 0; r < KPT; ++r) {
			const uint32_t d = rec_byte<WORDS>(key[r], p.byte);
			const uint32_t m = peers[r];
			const uint32_t below = __popc(m & lanemask_lt());
			const int leader = __ffs(m) - 1;
			uint32_t old = 0;
			if ((int)lane == leader) {
				old = wh[d];
				wh[d] = old + __popc(m);
			}
			old = __shfl_sync(0xffffffffu, old, leader);
			buf[tile_excl[d] + old + below] = key[r];
			__syncwarp();
		}

		// ---- phase 4: chained scan over tiles (decoupled look-back), one digit per thread
		if (tid < 256) {
			const uint64_t excl = tile == 0 ? 0 : lookback_resolve(desc + tid, 256, tile, (uint64_t)cnt_real, p.epoch);
			goff[tid] = bucket_base + excl - texcl;    // global index of tile-sorted position q is goff[d] + q
		}
		__syncthreads();

		// ---- phase 5: digit-contiguous runs leave with coalesced stores; count the next digit on the way out
#pragma unroll
		for (int i = 0; i < KPT; ++i) {
			const uint32_t q = i * THREADS + tid;
			if (q < valid) {
				const R k = buf[q];
				const uint32_t d = rec_byte<WORDS>(k, p.byte);
				gout[goff[d] + q] = k;
				if (p.next_byte >= 0) atomicAdd(&nhist[rec_byte<WORDS>(k, (uint32_t)p.next_byte)], 1u);
			}
		}
		fence_proxy_async();     // generic-proxy accesses of this buffer are ordered before the TMA refill
		__syncthreads();
		cur ^= 1;
	}

	if (tid < 256) {
		const uint32_t c = nhist[tid];
		if (p.next_byte >= 0 && c) atomicAdd(reinterpret_cast<unsigned long long*>(p.hist_next) + tid, (unsigned long long)c);
		nhist[tid] = 0;
	}
	__syncthreads();
}

template <int WORDS>
__device__ __forceinline__ void radix_pass_init(uint8_t* smem)
{
	using S = SortSmem<WORDS>;
	uint32_t* nhist = reinterpret_cast<uint32_t*>(smem + S::oNhist);
	uint64_t* mbar = reinterpret_cast<uint64_t*>(smem + S::oMbar);
	if (threadIdx.x < 256) nhist[threadIdx.x] = 0;
	if (threadIdx.x == 0) {
		mbar_init(&mbar[0], 1);
		mbar_init(&mbar[1], 1);
		fence_mbar_init();
	}
	__syncthreads();
}

// a single pass (kmcb200_dev_sort with KMCB200_SORT=lsd times its passes one by one)
template <int WORDS>
__global__ void __launch_bounds__(SortCfg<WORDS>::kThreads, SortCfg<WORDS>::kMinBlocks) radix_pass_kernel(const SortPass p)
{
	extern __shared__ __align__(128) uint8_t smem[];
	if (!run_allowed(p.run_flag, p.run_need)) return;
	radix_pass_init<WORDS>(smem);
	uint32_t phase0 = 0, phase1 = 0;
	radix_pass_body<WORDS>(p, smem, phase0, phase1);
}

// histogram of the first digit over N records, in front of the LSD passes (run_flag as in SortPass)
template <int WORDS>
__global__ void __launch_bounds__(512) digit_histogram_kernel(const void* in, uint64_t n, uint32_t byte, uint64_t* hist, const uint32_t* run_flag, uint32_t run_need)
{
	__shared__ uint32_t sh[256];
	if (!run_allowed(run_flag, run_need)) return;
	const Rec<WORDS>* __restrict__ g = reinterpret_cast<const Rec<WORDS>*>(in);
	if (threadIdx.x < 256) sh[threadIdx.x] = 0;
	__syncthreads();
	const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	// one CTA never sees 2^32 records of one digit (n / gridDim.x < 2^32)
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
		atomicAdd(&sh[rec_byte<WORDS>(g[i], byte)], 1u);
	__syncthreads();
	if (threadIdx.x < 256) { uint32_t c = sh[threadIdx.x]; if (c) atomicAdd((unsigned long long*)hist + threadIdx.x, (unsigned long long)c); }
}

// ---------------------------------------------------------------------------------------------------------------------
// All key_bytes LSD passes in ONE cooperative launch (grid-wide barrier between the passes).  This is the whole sort of small
// bins / KMCB200_SORT=lsd, and the device-flagged fallback of the hybrid MSD path: enqueued behind it, it returns at once unless
// the flag says that the hybrid path gave up - one no-op launch instead of one per pass.
struct LsdSortArgs {
	void* a;                 // pass 0 reads a and writes b, pass 1 the other way round, ...
	void* b;
	uint64_t n;
	uint32_t n_tiles;
	uint32_t key_bytes;
	uint64_t* hist;          // [key_bytes + 1][256], zero-initialised
	uint64_t* desc;          // [n_tiles][256]
	uint32_t epoch0;         // pass i uses epoch0 + i
	uint32_t* tile_counters; // [key_bytes], zero-initialised
	const uint32_t* run_flag;
	uint32_t run_need;
	// fallback of the leaf-count path: forget what the leaves have already added to the LUT / the statistics
	uint64_t* reset_lut;     // nullptr: nothing to reset
	uint64_t reset_lut_entries;
	uint64_t* reset_result;  // [6]
};

template <int WORDS>
__global__ void __launch_bounds__(SortCfg<WORDS>::kThreads, SortCfg<WORDS>::kMinBlocks) lsd_sort_kernel(const LsdSortArgs a)
{
	extern __shared__ __align__(128) uint8_t smem[];
	if (!run_allowed(a.run_flag, a.run_need)) return;          // (every CTA takes the same decision: nobody waits at a grid barrier)
	cooperative_groups::grid_group grid = cooperative_groups::this_grid();
	using S = SortSmem<WORDS>;
	const uint32_t tid = threadIdx.x;
	radix_pass_init<WORDS>(smem);
	{	// histogram of digit 0 (+ the resets)
		uint32_t* sh = reinterpret_cast<uint32_t*>(smem + S::oWhist);
		if (tid < 256) sh[tid] = 0;
		__syncthreads();
		const Rec<WORDS>* __restrict__ g = reinterpret_cast<const Rec<WORDS>*>(a.a);
		const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
		for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + tid; i < a.n; i += stride) atomicAdd(&sh[rec_byte<WORDS>(g[i], 0)], 1u);
		__syncthreads();
		if (tid < 256) { const uint32_t c = sh[tid]; if (c) atomicAdd(reinterpret_cast<unsigned long long*>(a.hist) + tid, (unsigned long long)c); }
		if (a.reset_lut) {
			for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + tid; i < a.reset_lut_entries; i += stride) a.reset_lut[i] = 0;
			if (blockIdx.x == 0 && tid < 6) a.reset_result[tid] = 0;
		}
		__syncthreads();
	}
	grid.sync();
	uint32_t phase0 = 0, phase1 = 0;
	for (uint32_t pass = 0; pass < a.key_bytes; ++pass) {
		SortPass p;
		p.in = (pass & 1u) ? a.b : a.a;
		p.out = (pass & 1u) ? a.a : a.b;
		p.n = a.n; p.n_tiles = a.n_tiles; p.byte = pass;
		p.next_byte = pass + 1 < a.key_bytes ? (int32_t)(pass + 1) : -1;
		p.hist = a.hist + 256 * pass;
		p.hist_next = a.hist + 256 * (pass + 1);
		p.desc = a.desc; p.epoch = a.epoch0 + pass;
		p.tile_counter = a.tile_counters + pass;
		p.run_flag = nullptr; p.run_need = 0;
		radix_pass_body<WORDS>(p, smem, phase0, phase1);
		if (pass + 1 < a.key_bytes) grid.sync();
	}
}

}  // namespace kmcb
