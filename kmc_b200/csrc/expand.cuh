// kmc_b200 — super-k-mer expansion (replaces CKmerBinSorter::ExpandKmersBoth / ExpandKmersAll,
// kmc_core/kb_sorter.h:251-362; for k % 32 != 0 also ExpandKxmersBoth/All :371-724 — we always expand to
// plain k-mers, the emitted database depends only on the multiset of canonical k-mers).
//
// Input : the bin byte stream written by stage 1 (kb_collector.cpp:34-90): records
//         [u8 a][ceil((k+a)/4) bytes], 2 bits per symbol, first symbol in bits 7-6 of the first byte.
// Output: n_rec records Rec<WORDS>, byte image identical to CKmer<SIZE> (kmer.h:22-67).
//
// The stream is self-delimiting, so record starts need a walk.  Packs (one per <=64 KiB collector flush,
// CExpanderPackDesc, queues.h:376-396) start on record boundaries and give the parallelism:
//   1. walk_packs_kernel  : one warp per pack walks its records and writes, per super-k-mer, its byte offset
//                           and the number of k-mers before it in the pack (both in a gap-free-per-pack region
//                           addressed by pack_start / min_rec_bytes, so no allocation scan is needed);
//   2. scan_packs_kernel  : exclusive scans over packs (k-mer base, output-tile base) + tile->pack map;
//   3. expand_kernel      : one CTA per 2048 consecutive OUTPUT k-mers (perfect load balance whatever the
//                           super-k-mer lengths): head flags + max-scan map every output slot to its
//                           super-k-mer, then each thread extracts its k-mer straight from the packed bytes
//                           with funnel shifts, reverse-complements it with brev, takes the canonical one and
//                           stores it coalesced.  The histogram of the first radix digit is counted on the
//                           way out, so the sort never re-reads the records just to count.
#pragma once
#include "common.cuh"

#ifndef KMCB200_EXPAND_UNROLL
#define KMCB200_EXPAND_UNROLL 8
#endif

namespace kmcb {

constexpr int kExpandUnroll = KMCB200_EXPAND_UNROLL;

// output tile of expand_kernel = work item of the level-1 MSD partition: 4096 one-word records, 2048 wider ones
#ifndef KMCB200_EXPAND_IPT
#define KMCB200_EXPAND_IPT 8
#endif
template <int WORDS> struct ExpandCfg { static constexpr int kTile = WORDS == 1 ? 4096 : 2048, kThreads = WORDS == 1 ? 4096 / KMCB200_EXPAND_IPT : 256; };
constexpr int kExpandMinTile = 2048;

struct ExpandArgs {
	const uint8_t* bin;          // bin byte stream (device)
	uint64_t size;
	const uint64_t* pack_start;  // [n_packs + 1] byte offsets (device)
	uint32_t n_packs;
	uint32_t k;
	uint32_t min_rec_bytes;      // 1 + ceil(k/4)
	uint32_t tile;               // ExpandCfg<WORDS>::kTile
	uint32_t both_strands;
	uint64_t n_rec;              // expected number of k-mers (CBinDesc::n_rec)
	// index produced by walk/scan
	uint32_t* sk_off;            // [size / min_rec_bytes + 1]
	uint32_t* sk_kpre;           // same
	uint32_t* tile_first;        // [4 * size / kExpandTile + n_packs + 1] first super-k-mer of every output tile of a pack
	uint32_t* pack_nsk;          // [n_packs]
	uint32_t* pack_nk;           // [n_packs]
	uint64_t* pack_kbase;        // [n_packs + 1]
	uint32_t* pack_tbase;        // [n_packs + 1]
	uint32_t* tile_pack;         // [tile_pack_cap]
	uint4* tile_desc;            // [2 * tile_pack_cap] everything expand_kernel needs to know about an output tile, gathered by tile_desc_kernel:
	                             //   {slot0, nsk, j_lo, off_lo} {tile_start | (cnt - 1), pack_end, obase lo, obase hi}
	uint64_t tile_pack_cap;      // n_rec / kExpandMinTile + n_packs + 2 (sized from the CALLER's n_rec: writes are clamped to it)
	uint32_t* status;            // [0] error bits, [1] total tiles (0 when the bin is malformed: nothing is expanded)
	uint32_t* flags;             // msd_sort.cuh: [0] / [1] get kMsdFlagAbort when the bin is malformed, so that no kernel behind touches the records
	// output
	void* recs;
	// level-1 work items of the MSD partition = the output tiles of this kernel (msd_sort.cuh)
	uint16_t* cells1;            // [256][total_tiles] counts of bits [top_shift, top_shift + 8) per tile
	uint64_t* item_lo1;          // [total_tiles] first output record of the tile
	uint16_t* item_cnt1;         // [total_tiles]
	uint32_t top_shift;
	// kExpandPartition (the bin path of one-word records): the level-1 buckets come from digit totals the index kernels count
	uint32_t* l1_total;          // [256] when set, the walk adds the level-1 digit of every k-mer here
	uint32_t* l1_cursor;         // [256] next free record of every level-1 bucket (msd_bounds_kernel starts it at l1_start[d])
	const uint64_t* l1_start;    // [257] level-1 bucket boundaries
	// oversized bins (kmc_b200.cu, run_oversized_bin): the bin is expanded chunk by chunk, once to count and once per key block
	uint32_t mode;               // 0: everything (above); 1: only count the top 12 bits into hist12; 2: only k-mers of one key block, appended to recs
	uint32_t fshift, fprefix, fmask;    // mode 2: keep the k-mers with ((kmer >> fshift) & fmask) == fprefix
	uint64_t* hist12;            // mode 1: [4096]
	unsigned long long* out_counter;     // mode 2: records appended so far; mode 3: [n_blocks] records appended to every key block's region
	// mode 3 (oversized bins whose records fit in HBM once): ONE expansion scatters every k-mer into the region of its key block
	const uint16_t* blk_of_prefix;       // [4096] key block of a 12-bit prefix
	const uint64_t* region_start;        // [n_blocks] first record of every block's region inside recs
	uint32_t n_blocks;                   // <= kExpandMaxBlocks
};
// kExpandPartition: the bin path expands a bin of one-word records straight into its level-1 buckets instead of writing the records in
// tile order and partitioning them by their top digit afterwards.  The pack walk counts the level-1 digit of every k-mer into 256 totals,
// msd_bounds_kernel turns them into the bucket boundaries, and every tile of the expansion reserves its run inside each bucket with one
// global atomicAdd (an MSD partition need not be stable, so the order of the runs does not matter).  The tile-ordered copy of the
// records (8N bytes written, 8N read back) never exists, and the bin is expanded once.
enum : uint32_t { kExpandAll = 0, kExpandCount12 = 1, kExpandFilter = 2, kExpandScatter = 3, kExpandPartition = 4 };
// kExpandPartition regroups a tile in shared memory over the staged bytes (8 bytes * 4096 records); wider records would need a larger
// buffer than static shared memory allows and more registers for the keys it holds
template <int WORDS> __host__ __device__ constexpr bool expand_partition_supported() { return WORDS == 1; }
constexpr uint32_t kExpandMaxBlocks = 512;
constexpr uint64_t kExpandUnknownRecs = ~0ull;      // n_rec of a chunk: not checked

enum : uint32_t { kErrPackWalk = 1, kErrRecCount = 2 };
constexpr uint32_t kExpandAbortFlag = 2;      // = kMsdFlagAbort (msd_sort.cuh)

__device__ __forceinline__ uint64_t tile_first_base(uint64_t pack_start, uint32_t p, uint32_t tile) { return pack_start * 4 / tile + p; }

// Level-1 digits of the x + 1 k-mers of one super-k-mer whose packed symbols start at `sym` (2 bits per symbol, the first in bits 7-6),
// added to the 256-entry histogram `hist`.  The digit is the top 8 bits of min(k-mer, reverse complement) of a k-mer of 2k >= 24 bits:
// min(its first 4 symbols, the complement of its last 4 reversed), or the first 4 alone in -b mode.  Four k-mers at a time: symbols
// s .. s+7 (bytes s/4 and s/4 + 1) hold the forward digits of k-mers s .. s+3, symbols s+k-4 .. s+k+3 (reversed and complemented once)
// their reverse ones, so four k-mers cost five byte loads and no chain runs from one group to the next.  The last group may read up to
// two bytes past the super-k-mer (the next record, or the slack behind the pack); those digits are not counted.
__device__ __forceinline__ void count_l1_digits(const uint8_t* sym, uint32_t x, uint32_t k, bool both_strands, uint32_t* hist)
{
	for (uint32_t s = 0; s <= x; s += 4) {
		const uint32_t fw = ((uint32_t)sym[s >> 2] << 8) | sym[(s >> 2) + 1];            // symbols s .. s+7, s at bits 15-14
		uint32_t rw = 0;
		if (both_strands) {
			const uint32_t b = s + k - 4, q = b >> 2;
			const uint32_t v = (((uint32_t)sym[q] << 16) | ((uint32_t)sym[q + 1] << 8) | sym[q + 2]) >> (8u - 2u * (b & 3u));     // symbols b .. b+7 in bits 15..0
			const uint32_t y = __brev(v) >> 16;                                            // bit order reversed ...
			rw = ~(((y >> 1) & 0x5555u) | ((y & 0x5555u) << 1));                          // ... symbol order reversed, complemented: b+i at bits 2i+1..2i
		}
		const uint32_t n = min(x + 1 - s, 4u);
#pragma unroll
		for (uint32_t j = 0; j < 4; ++j) {
			if (j < n) {
				const uint32_t f = (fw >> (8u - 2u * j)) & 0xFFu;
				atomicAdd(&hist[both_strands ? min(f, (rw >> (2u * j)) & 0xFFu) : f], 1u);
			}
		}
	}
}

// ---------------------------------------------------------------------------------------------------------------------
// Walking a pack is a serial chain (the length byte of a record says where the next record starts).  For the usual pack
// (one collector flush, <= 64 KiB) the chain is cut into 256 segments of 256 bytes that are walked IN PARALLEL, one thread each,
// from shared memory: thread t does not know where the first record of its segment begins, so it starts 1 KB earlier at an
// arbitrary byte and follows the chain from there.  Any chain that ever lands on a true record start stays on the true chain,
// and a landing hits a true start with probability ~1/12, so after 1 KB the two have merged for ~9 segments out of 10.
// The rest is repaired, not assumed: the entry of segment t must be exactly the exit of segment t-1 (segment 0 starts on the
// true start); a segment whose entry is off re-walks from the true one, round after round until nothing changes (chains merge,
// so exits rarely move: one or two rounds).  A final check of the whole chain guards the result; a pack that fails it is left
// to the exact warp-per-pack walker below.  A step costs one shared-memory load; ~150 steps per thread.
constexpr int kWalkSegBytes = 256;
constexpr int kWalkSegs = 256;                                   // threads per CTA = segments per pack
constexpr int kWalkChunk = kWalkSegBytes * kWalkSegs;            // 64 KiB
#ifndef KMCB200_WALK_SPEC
#define KMCB200_WALK_SPEC 1024
#endif
constexpr int kWalkSpec = KMCB200_WALK_SPEC;

__global__ void __launch_bounds__(kWalkSegs, 3) walk_packs_parallel_kernel(const ExpandArgs a, uint32_t* pack_done)
{
	extern __shared__ __align__(16) uint8_t wsm[];               // the pack (+ 16 bytes of slack)
	__shared__ uint32_t s_entry[kWalkSegs], s_exit[kWalkSegs], s_w[16];
	__shared__ uint32_t s_bad;
	__shared__ uint32_t s_hist[256];                             // a.l1_total: the pack's level-1 digits
	static_assert(kWalkSegs == 256, "one histogram entry per thread");
	const uint32_t p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const uint64_t pstart = a.pack_start[p];
	const uint32_t len = (uint32_t)min(a.pack_start[p + 1] - pstart, (uint64_t)kWalkChunk + 1);
	if (len > (uint32_t)kWalkChunk || len == 0) { if (tid == 0) pack_done[p] = len == 0 ? 1u : 0u; if (len == 0 && tid == 0) { a.pack_nsk[p] = 0; a.pack_nk[p] = 0; } return; }
	s_hist[tid] = 0;
	// ---- the pack into shared memory (16-byte loads on the absolute 16-byte grid)
	{
		const uintptr_t g0 = reinterpret_cast<uintptr_t>(a.bin + pstart);
		const uintptr_t g0a = g0 & ~(uintptr_t)15;
		const uint32_t shift = (uint32_t)(g0 - g0a);
		const uint32_t nvec = (len + shift + 15) >> 4;
		// (8 independent loads in flight per thread: a loop of load -> store pairs would pay the DRAM latency 16 times in a row)
		for (uint32_t v0 = tid; v0 < nvec; v0 += 8 * kWalkSegs) {
			uint4 r[8];
#pragma unroll
			for (int i = 0; i < 8; ++i) { const uint32_t v = v0 + i * kWalkSegs; r[i] = v < nvec ? __ldg(reinterpret_cast<const uint4*>(g0a) + v) : make_uint4(0, 0, 0, 0); }
#pragma unroll
			for (int i = 0; i < 8; ++i) { const uint32_t v = v0 + i * kWalkSegs; if (v < nvec) reinterpret_cast<uint4*>(wsm)[v] = r[i]; }
		}
		if (tid == 0) s_bad = 0;
		__syncthreads();
		// byte i of the pack is wsm[shift + i]
		const uint8_t* pk = wsm + shift;
		const uint32_t k3 = a.k + 3;
		const uint32_t seg_lo = tid * kWalkSegBytes, seg_hi = min(seg_lo + (uint32_t)kWalkSegBytes, len);
		uint32_t pos = seg_lo > (uint32_t)kWalkSpec ? seg_lo - kWalkSpec : 0;       // speculative start (exact for the first segments)
		if (seg_lo < len) {
			while (pos < seg_lo) pos += 1 + ((pk[pos] + k3) >> 2);
		} else pos = len;
		uint32_t entry = min(pos, len);
		uint32_t nrec = 0, nk = 0;
		pos = entry;
		while (pos < seg_hi) { const uint32_t x = pk[pos]; nk += x + 1; ++nrec; pos += 1 + ((x + k3) >> 2); }
		s_entry[tid] = entry; s_exit[tid] = seg_lo < len ? pos : len;
		// ---- make the chain of segments consistent: the entry of segment t must be the exit of segment t-1 (segment 0 starts on the true
		// start).  A segment whose speculative entry was off re-walks from the true one; since chains merge, its exit rarely changes,
		// so one or two rounds settle a pack (at most one round per segment: every round fixes at least the first wrong segment).
		for (int it = 0; it < kWalkSegs; ++it) {
			__syncthreads();
			const uint32_t want = tid > 0 ? min(s_exit[tid - 1], len) : 0u;
			const bool fix = tid > 0 && seg_lo < len && entry != want;
			if (!__syncthreads_or(fix)) break;
			if (fix) {
				entry = want; nrec = 0; nk = 0; pos = entry;
				while (pos < seg_hi) { const uint32_t x = pk[pos]; nk += x + 1; ++nrec; pos += 1 + ((x + k3) >> 2); }
				s_entry[tid] = entry; s_exit[tid] = pos;
			}
		}
		__syncthreads();
		// ---- verify (cheap, and the only thing correctness rests on)
		bool bad = false;
		if (tid > 0 && seg_lo < len && s_entry[tid] != min(s_exit[tid - 1], len)) bad = true;
		if (tid == kWalkSegs - 1 || seg_hi == len) { if (seg_lo < len && s_exit[tid] != len) bad = true; }     // the last record must end with the pack
		if (bad) atomicOr(&s_bad, 1u);
		// ---- exclusive scans of records and k-mers over the segments
		uint32_t ir = nrec, ik = nk;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t tr = __shfl_up_sync(0xffffffffu, ir, o), tk = __shfl_up_sync(0xffffffffu, ik, o);
			if (lane >= (uint32_t)o) { ir += tr; ik += tk; }
		}
		if (lane == 31) { s_w[warp] = ir; s_w[8 + warp] = ik; }
		__syncthreads();
		if (s_bad) {          // the repaired chain IS the exact chain: its last record does not end with the pack -> the bin is malformed
			if (tid == 0) { atomicOr(a.status, kErrPackWalk); a.pack_nsk[p] = 0; a.pack_nk[p] = 0; pack_done[p] = 1; }
			return;
		}
		uint32_t br = ir - nrec, bk = ik - nk, tr = 0, tk = 0;
#pragma unroll
		for (int w = 0; w < 8; ++w) { if ((uint32_t)w < warp) { br += s_w[w]; bk += s_w[8 + w]; } tr += s_w[w]; tk += s_w[8 + w]; }
		// ---- second walk of the own segment: the index (and the level-1 digits of the pack's k-mers)
		const uint64_t slot = pstart / a.min_rec_bytes;
		const uint64_t tfb = tile_first_base(pstart, p, a.tile);
		uint32_t j = br, kk = bk;
		pos = entry;
		while (pos < seg_hi) {
			const uint32_t x = pk[pos];
			a.sk_off[slot + j] = (uint32_t)(pstart + pos);
			a.sk_kpre[slot + j] = kk;
			const uint32_t tb = (kk + a.tile - 1) / a.tile;                     // first tile boundary at or after this super-k-mer's first k-mer
			if (tb * a.tile < kk + x + 1) a.tile_first[tfb + tb] = j;
			if (a.l1_total) count_l1_digits(pk + pos + 1, x, a.k, a.both_strands != 0, s_hist);
			kk += x + 1;
			pos += 1 + ((x + k3) >> 2);
			++j;
		}
		if (tid == 0) { a.pack_nsk[p] = tr; a.pack_nk[p] = tk; pack_done[p] = 1; }
		if (a.l1_total) {
			__syncthreads();
			if (s_hist[tid]) atomicAdd(&a.l1_total[tid], s_hist[tid]);
		}
	}
}

// One WARP per pack.  The walk itself is a serial chain (the length byte of a record tells where the next one
// starts), so the only thing that matters is the latency of one step.  The warp keeps a 512-byte window of the stream
// in registers (one uint4 per lane, the next window already in flight), a step is one shuffle + a few integer ops
// and never waits for DRAM; the per-super-k-mer index leaves with coalesced 128-byte stores.
constexpr int kWalkWarpsPerBlock = 4;

__device__ __forceinline__ uint4 walk_load_window(const uint8_t* bin_aligned, uint64_t wbase, uint64_t limit, uint32_t lane)
{
	const uint64_t o = wbase + 16ull * lane;
	return o < limit ? __ldg(reinterpret_cast<const uint4*>(bin_aligned + o)) : make_uint4(0, 0, 0, 0);
}

__global__ void __launch_bounds__(32 * kWalkWarpsPerBlock) walk_packs_kernel(const ExpandArgs a, const uint32_t* pack_done)
{
	const uint32_t lane = threadIdx.x & 31u;
	const uint32_t p = blockIdx.x * kWalkWarpsPerBlock + (threadIdx.x >> 5);
	if (p >= a.n_packs) return;
	if (pack_done && pack_done[p]) return;              // the parallel walker has done this pack
	uint64_t pos = a.pack_start[p];
	const uint64_t end = a.pack_start[p + 1];
	const uint64_t slot = pos / a.min_rec_bytes;
	const uint64_t tfb = tile_first_base(pos, p, a.tile);
	// 16-byte aligned view of the stream (the bin pointer is at least 8-byte aligned; the window grid is aligned on absolute addresses)
	const uintptr_t base_addr = reinterpret_cast<uintptr_t>(a.bin);
	const uint8_t* bin_aligned = reinterpret_cast<const uint8_t*>(base_addr & ~(uintptr_t)15);
	const uint64_t shift = base_addr & 15u;                 // stream offset x lives at aligned offset x + shift
	const uint64_t limit = ((a.size + shift + 15) & ~15ull);  // readable bytes of the aligned view
	uint64_t wbase = (pos + shift) & ~511ull;
	uint4 cur = walk_load_window(bin_aligned, wbase, limit, lane);
	uint4 nxt = walk_load_window(bin_aligned, wbase + 512, limit, lane);
	uint32_t j = 0, nk = 0, next_tile = 0;
	uint32_t my_off = 0, my_kpre = 0, my_x = 0;
	// a.l1_total: every lane counts the level-1 digits of the super-k-mers it stores, from global memory (packs this large are rare)
	auto count = [&]() { if (a.l1_total) count_l1_digits(a.bin + my_off + 1, my_x, a.k, a.both_strands != 0, a.l1_total); };
	while (pos < end) {
		uint64_t rel = pos + shift - wbase;
		if (rel >= 512) {            // a record is at most 1 + (k + 255 + 3) / 4 <= 97 bytes: one window shift is enough
			cur = nxt;
			wbase += 512;
			nxt = walk_load_window(bin_aligned, wbase + 512, limit, lane);
			rel -= 512;
		}
		const uint32_t r = (uint32_t)rel;
		const uint32_t comp = (r >> 2) & 3u;
		uint32_t w = comp == 0 ? cur.x : comp == 1 ? cur.y : comp == 2 ? cur.z : cur.w;
		w = __shfl_sync(0xffffffffu, w, r >> 4);
		const uint32_t x = (w >> ((r & 3u) * 8u)) & 0xFFu;
		if (lane == (j & 31u)) { my_off = (uint32_t)pos; my_kpre = nk; my_x = x; }
		if ((j & 31u) == 31u) {      // 32 super-k-mers collected: one coalesced store each
			a.sk_off[slot + j - 31 + lane] = my_off;
			a.sk_kpre[slot + j - 31 + lane] = my_kpre;
			count();
		}
		if (nk + x + 1 > next_tile * a.tile) {   // this super-k-mer holds k-mer number next_tile * tile of the pack
			if (lane == 0) a.tile_first[tfb + next_tile] = j;
			++next_tile;
		}
		nk += x + 1;
		pos += 1 + ((x + a.k + 3) >> 2);
		++j;
	}
	if (lane < (j & 31u)) {          // the unfinished group
		a.sk_off[slot + (j & ~31u) + lane] = my_off;
		a.sk_kpre[slot + (j & ~31u) + lane] = my_kpre;
		count();
	}
	if (lane == 0) {
		if (pos != end) atomicOr(a.status, kErrPackWalk);
		a.pack_nsk[p] = j;
		a.pack_nk[p] = nk;
	}
}

// SURVEY section 8f N4 - a device-friendly stage-1 output.  The walk above exists only because the stream is self-delimiting.  If stage 1
// also hands over the length bytes as a SEPARATE array (`extras[i]` = the byte `a` of record i, 1 byte per super-k-mer; the collector has
// it in a register when it writes the record, kb_collector.cpp:60-66) plus the number of records of every pack, the index is two block-wide
// prefix sums per pack instead of a serial chain: one CTA per pack, one thread per record.  The result is checked against the stream (the
// byte at every computed offset must be that record's `a`, the last record must end with the pack), so a wrong array is a reported bin
// format error, never a wrong result.
__global__ void __launch_bounds__(1024) index_from_extras_kernel(const ExpandArgs a, const uint8_t* __restrict__ extras, const uint64_t* __restrict__ pack_rec_start)
{
	__shared__ uint32_t s_b[32], s_k[32];
	__shared__ uint32_t carry_b, carry_k;
	__shared__ uint32_t s_bad;
	__shared__ uint32_t s_hist[256];          // a.l1_total: the pack's level-1 digits
	const uint32_t p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const uint64_t pstart = a.pack_start[p];
	const uint32_t len = (uint32_t)min(a.pack_start[p + 1] - pstart, (uint64_t)0xffffffffu);
	const uint64_t r0 = pack_rec_start[p];
	const uint32_t nrec = (uint32_t)min(pack_rec_start[p + 1] - r0, (uint64_t)0xffffffffu);
	const uint64_t slot = pstart / a.min_rec_bytes;
	const uint64_t tfb = tile_first_base(pstart, p, a.tile);
	if (tid < 256) s_hist[tid] = 0;
	if (tid == 0) { carry_b = 0; carry_k = 0; s_bad = 0; }
	__syncthreads();
	// (more records than the pack's bytes can hold: the array is wrong; also keeps the index writes inside the pack's own slots)
	const bool too_many = (uint64_t)nrec * a.min_rec_bytes > (uint64_t)len;
	for (uint32_t j0 = 0; j0 < nrec && !too_many; j0 += 1024) {
		const uint32_t j = j0 + tid;
		const uint32_t x = j < nrec ? extras[r0 + j] : 0u;
		const uint32_t nb = j < nrec ? 1u + ((x + a.k + 3u) >> 2) : 0u, nk = j < nrec ? x + 1u : 0u;
		uint32_t ib = nb, ik = nk;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t tb = __shfl_up_sync(0xffffffffu, ib, o), tk = __shfl_up_sync(0xffffffffu, ik, o);
			if (lane >= (uint32_t)o) { ib += tb; ik += tk; }
		}
		if (lane == 31) { s_b[warp] = ib; s_k[warp] = ik; }
		__syncthreads();
		uint32_t bb = carry_b, bk = carry_k;
		for (uint32_t w = 0; w < warp; ++w) { bb += s_b[w]; bk += s_k[w]; }
		const uint32_t off = bb + ib - nb, kk = bk + ik - nk;          // byte offset inside the pack / k-mers before this record
		if (j < nrec) {
			if (off + nb > len || a.bin[pstart + off] != (uint8_t)x) atomicOr(&s_bad, 1u);          // the stream disagrees with the array
			else {
				a.sk_off[slot + j] = (uint32_t)(pstart + off);
				a.sk_kpre[slot + j] = kk;
				const uint32_t tb = (kk + a.tile - 1) / a.tile;
				if (tb * a.tile < kk + x + 1) a.tile_first[tfb + tb] = j;
				if (a.l1_total) count_l1_digits(a.bin + pstart + off + 1, x, a.k, a.both_strands != 0, s_hist);
			}
		}
		__syncthreads();
		if (tid == 1023) { carry_b = bb + ib; carry_k = bk + ik; }
		__syncthreads();
	}
	const bool bad = too_many || s_bad || carry_b != len;          // (uniform: the last barrier is behind every write of these)
	if (tid == 0) {
		if (bad) atomicOr(a.status, kErrPackWalk);
		a.pack_nsk[p] = bad ? 0u : nrec;
		a.pack_nk[p] = bad ? 0u : carry_k;
	}
	if (a.l1_total && !bad && tid < 256 && s_hist[tid]) atomicAdd(&a.l1_total[tid], s_hist[tid]);          // (a malformed pack counts nothing)
}

// single CTA: exclusive scans over packs
__global__ void __launch_bounds__(1024) scan_packs_kernel(const ExpandArgs a)
{
	__shared__ uint64_t s_k[32];
	__shared__ uint32_t s_t[32];
	__shared__ uint64_t carry_k;
	__shared__ uint32_t carry_t;
	const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid == 0) { carry_k = 0; carry_t = 0; }
	__syncthreads();
	// A malformed bin (a pack that does not end on a record boundary, more / fewer k-mers than n_rec) must not reach the kernels
	// behind: their buffers are sized from the caller's n_rec.  It is stopped here: no tiles, and the abort flag for the sort / count.
	const bool walk_failed = (a.status[0] & kErrPackWalk) != 0;
	for (uint32_t base = 0; base < a.n_packs && !walk_failed; base += 1024) {
		const uint32_t p = base + tid;
		const uint32_t nk = p < a.n_packs ? a.pack_nk[p] : 0;
		const uint32_t nt = (nk + a.tile - 1) / a.tile;
		uint64_t ik = nk;
		uint32_t it = nt;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			uint64_t tk = __shfl_up_sync(0xffffffffu, ik, o);
			uint32_t tt = __shfl_up_sync(0xffffffffu, it, o);
			if (lane >= (uint32_t)o) { ik += tk; it += tt; }
		}
		if (lane == 31) { s_k[warp] = ik; s_t[warp] = it; }
		__syncthreads();
		uint64_t bk = carry_k;
		uint32_t bt = carry_t;
		for (uint32_t w = 0; w < warp; ++w) { bk += s_k[w]; bt += s_t[w]; }
		const uint64_t ek = bk + ik - nk;
		const uint32_t et = bt + it - nt;
		if (p < a.n_packs) {
			a.pack_kbase[p] = ek;
			a.pack_tbase[p] = et;
			for (uint32_t t = 0; t < nt && (uint64_t)et + t < a.tile_pack_cap; ++t) a.tile_pack[et + t] = p;
		}
		__syncthreads();
		if (tid == 1023) { carry_k = ek + nk; carry_t = et + nt; }
		__syncthreads();
	}
	if (tid == 0) {
		a.pack_kbase[a.n_packs] = carry_k;
		a.pack_tbase[a.n_packs] = carry_t;
		bool bad = walk_failed;
		if (a.n_rec != kExpandUnknownRecs && carry_k != a.n_rec) { atomicOr(a.status, kErrRecCount); bad = true; }
		if ((uint64_t)carry_t > a.tile_pack_cap) bad = true;
		a.status[1] = bad ? 0u : carry_t;
		if (bad && a.flags) { atomicOr(&a.flags[0], kExpandAbortFlag); atomicOr(&a.flags[1], kExpandAbortFlag); }
	}
}

// one thread per output tile: the tile's geometry, gathered from the per-pack tables and the index into ONE 32-byte descriptor, so that
// expand_kernel starts a tile with one load instead of a chain of four dependent ones (tile -> pack -> pack tables -> first super-k-mer ->
// its offset: a third of the stall samples of expand_kernel were waits for global loads, round 2) and without a 64-bit division
__global__ void __launch_bounds__(256) tile_desc_kernel(const ExpandArgs a)
{
	const uint32_t g = blockIdx.x * 256 + threadIdx.x;
	if (g >= a.status[1]) return;
	const uint32_t p = a.tile_pack[g];
	const uint32_t t = g - a.pack_tbase[p];
	const uint64_t pstart = a.pack_start[p];
	const uint64_t slot0 = pstart / a.min_rec_bytes;
	const uint32_t nk = a.pack_nk[p];
	const uint32_t tile_start = t * a.tile;
	const uint32_t cnt = min(a.tile, nk - tile_start);
	const uint32_t j_lo = a.tile_first[tile_first_base(pstart, p, a.tile) + t];
	const uint64_t obase = a.pack_kbase[p] + tile_start;
	a.tile_desc[2 * (size_t)g] = make_uint4((uint32_t)slot0, a.pack_nsk[p], j_lo, a.sk_off[slot0 + j_lo]);
	a.tile_desc[2 * (size_t)g + 1] = make_uint4(tile_start | (cnt - 1u), (uint32_t)a.pack_start[p + 1], (uint32_t)obase, (uint32_t)(obase >> 32));
}

__device__ __forceinline__ uint64_t bswap64(uint64_t x)
{
	const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
	return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | (uint64_t)__byte_perm(hi, 0, 0x0123);
}
// reverse the order of the 32 two-bit symbols of a word
__device__ __forceinline__ uint64_t rev_symbols64(uint64_t x)
{
	const uint64_t y = __brevll(x);
	return ((y >> 1) & 0x5555555555555555ull) | ((y & 0x5555555555555555ull) << 1);
}

// k-mer number `s` of the super-k-mer whose packed symbols start at global byte address `payload`.
// `load8(addr)` returns the 8 bytes at the 8-byte aligned absolute address addr (from global memory, or from a staged copy).
template <int WORDS, typename Load8>
__device__ __forceinline__ Rec<WORDS> extract_kmer(const uint8_t* payload, uint32_t s, uint32_t k, bool canonical, Load8 load8)
{
	const uint8_t* A = payload + (s >> 2);
	const uint32_t sh = (s & 3u) * 2u;
	const uintptr_t a0 = reinterpret_cast<uintptr_t>(A) & ~(uintptr_t)7;
	const uint32_t bo = (uint32_t)(reinterpret_cast<uintptr_t>(A) - a0) * 8u + sh;    // 0..62: bit offset inside b[0]
	const uintptr_t need_end = reinterpret_cast<uintptr_t>(A) + ((sh + 2u * k + 7u) >> 3);
	uint64_t b[WORDS + 1];
#pragma unroll
	for (int i = 0; i <= WORDS; ++i) {
		const uintptr_t wa = a0 + 8u * i;
		b[i] = wa < need_end ? bswap64(load8(wa)) : 0ull;
	}
	// t = the WORDS-word big number (t[0] most significant) holding bits [bo, bo + 64*WORDS)
	uint64_t t[WORDS];
#pragma unroll
	for (int i = 0; i < WORDS; ++i) t[i] = bo ? ((b[i] << bo) | (b[i + 1] >> (64u - bo))) : b[i];
	// right-align the top 2k bits
	const uint32_t rs = 64u * WORDS - 2u * k;     // 0..63
	Rec<WORDS> f;
#pragma unroll
	for (int i = 0; i < WORDS; ++i) {
		// word i counted from the most significant end after the shift
		uint64_t v = t[i] >> rs;
		if (i > 0 && rs) v |= t[i - 1] << (64u - rs);
		f.w[WORDS - 1 - i] = v;
	}
	if (!canonical) return f;
	// reverse complement: reverse all symbols of the 64*WORDS-bit number (puts the k-mer top-aligned), complement, right-align
	uint64_t u[WORDS];      // u[0] most significant
#pragma unroll
	for (int i = 0; i < WORDS; ++i) u[i] = ~rev_symbols64(f.w[i]);      // f.w[i] (i-th least significant) becomes i-th most significant
	Rec<WORDS> r;
#pragma unroll
	for (int i = 0; i < WORDS; ++i) {
		uint64_t v = u[i] >> rs;
		if (i > 0 && rs) v |= u[i - 1] << (64u - rs);
		r.w[WORDS - 1 - i] = v;
	}
	return rec_less<WORDS>(f, r) ? f : r;       // kmer < rev ? kmer : rev  (kb_sorter.h:340,356)
}

// The staged fast path: the tile's bytes lie in shared memory as BIG-ENDIAN 32-bit words (one byte_perm per word when they are
// staged, not per k-mer), so the k-mer that starts at bit B of the staged stream is a funnel shift over 2*WORDS+1 consecutive words.
// Bits past the k-mer (the next super-k-mer, or stale bytes behind the tile) only reach positions that the right-alignment shifts out.
template <int WORDS>
__device__ __forceinline__ Rec<WORDS> extract_kmer_be32(const uint32_t* sw, uint32_t B, uint32_t k, bool canonical)
{
	const uint32_t wi = B >> 5, bo = B & 31u;
	uint32_t w[2 * WORDS + 1];
#pragma unroll
	for (int i = 0; i <= 2 * WORDS; ++i) w[i] = sw[wi + i];
	uint64_t t[WORDS];          // t[0] most significant: bits [B, B + 64*WORDS)
#pragma unroll
	for (int i = 0; i < WORDS; ++i)
		t[i] = ((uint64_t)__funnelshift_l(w[2 * i + 1], w[2 * i], bo) << 32) | (uint64_t)__funnelshift_l(w[2 * i + 2], w[2 * i + 1], bo);
	const uint32_t rs = 64u * WORDS - 2u * k;     // 0..63
	Rec<WORDS> f;
#pragma unroll
	for (int i = 0; i < WORDS; ++i) {
		uint64_t v = t[i] >> rs;
		if (i > 0 && rs) v |= t[i - 1] << (64u - rs);
		f.w[WORDS - 1 - i] = v;
	}
	if (!canonical) return f;
	uint64_t u[WORDS];
#pragma unroll
	for (int i = 0; i < WORDS; ++i) u[i] = ~rev_symbols64(f.w[i]);
	Rec<WORDS> r;
#pragma unroll
	for (int i = 0; i < WORDS; ++i) {
		uint64_t v = u[i] >> rs;
		if (i > 0 && rs) v |= u[i - 1] << (64u - rs);
		r.w[WORDS - 1 - i] = v;
	}
	return rec_less<WORDS>(f, r) ? f : r;       // kmer < rev ? kmer : rev  (kb_sorter.h:340,356)
}

// 8 bits starting at bit `shift` of the record
template <int WORDS>
__device__ __forceinline__ uint32_t rec_top_digit(const Rec<WORDS>& r, uint32_t shift)
{
	const uint32_t wi = shift >> 6, off = shift & 63u;
	uint64_t lo = r.w[0], hi = 0;
#pragma unroll
	for (int i = 1; i < WORDS; ++i) {
		if (wi == (uint32_t)i) lo = r.w[i];
		if (wi + 1 == (uint32_t)i) hi = r.w[i];
	}
	uint64_t v = lo >> off;
	if (WORDS > 1 && off) v |= hi << (64u - off);
	return (uint32_t)v & 0xFFu;
}

// bits [shift, shift + ...) of a record under `mask` (mask <= 32 bits)
template <int WORDS>
__device__ __forceinline__ uint32_t msd_free_bits(const Rec<WORDS>& r, uint32_t shift, uint32_t mask)
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

// (<= 32 registers for one- and two-word records, <= 42 beyond: the occupancy the kernel was tuned at.  kExpandPartition holds the tile's
// 8 k-mers and their ranks per thread across its barriers: <= 40 registers, 3 CTAs of 512 threads per SM, which measured faster than 2)
template <int WORDS, uint32_t MODE>
__host__ __device__ constexpr int expand_min_blocks() { return MODE == kExpandPartition ? 3 : WORDS <= 2 ? 2048 / ExpandCfg<WORDS>::kThreads : 6; }

// MODE is a template parameter: the bin path (kExpandAll) must not pay registers / shared memory for the oversized-bin modes
// (with the scatter code in the same instance the kernel needs more than 32 registers and the expansion is slower)
template <int WORDS, uint32_t MODE = kExpandAll>
__global__ void __launch_bounds__(ExpandCfg<WORDS>::kThreads, expand_min_blocks<WORDS, MODE>()) expand_kernel(const ExpandArgs a)
{
	constexpr int kExpandTile = ExpandCfg<WORDS>::kTile, kExpandThreads = ExpandCfg<WORDS>::kThreads;
	constexpr int IPT = kExpandTile / kExpandThreads;    // 8 k-mers per thread
	constexpr int MAXSK = 1024, STAGE = 12288;          // per-tile staging of the super-k-mer index and bytes (typical tile: ~350 super-k-mers, ~4.5 KB)
	constexpr int HW = kExpandTile / 32;                 // words of the head bitmap
	// kExpandPartition regroups the tile's records in the staging buffer once they are all extracted
	constexpr int SBYTES = MODE == kExpandPartition && kExpandTile * 8 * WORDS > STAGE + 32 ? kExpandTile * 8 * WORDS : STAGE + 32;
	static_assert(MODE != kExpandPartition || expand_partition_supported<WORDS>(), "kExpandPartition: one-word records only");
	__shared__ uint32_t hbits[HW];                       // bit s: a super-k-mer (other than the tile's first) starts at output slot s
	__shared__ uint32_t hpre[HW];                        // set bits before the word
	__shared__ uint32_t s_bit[MAXSK];                    // staged tiles: bit position of (k-mer of output slot 0) of every super-k-mer, minus 2 * slot
	__shared__ __align__(16) uint8_t s_bytes[SBYTES];    // the tile's bytes as big-endian 32-bit words (+ slack: a funnel shift looks 2*WORDS words ahead)
	__shared__ uint32_t s_jmax;
	__shared__ unsigned long long s_fbase;
	__shared__ uint32_t warp_max[kExpandThreads / 32];   // (scratch of the filter mode)
	__shared__ uint32_t htop[256];
	static_assert(HW <= 128 && HW % 32 == 0, "the head bitmap is scanned by one warp, HW / 32 words per lane");
	const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const uint32_t le_mask = 0xffffffffu >> (31u - lane);
	static_assert(kExpandThreads % 32 == 0, "output slot i * threads + tid belongs to lane tid % 32");
	if constexpr (MODE == kExpandPartition)
		if (a.flags[1] & kExpandAbortFlag) return;       // (a malformed bin also has no tiles)
	if (tid < 256) htop[tid] = 0;
	const uint32_t total_tiles = a.status[1];
	// (kExpandPartition runs at its register limit: it re-reads the tile count, written by scan_packs_kernel, instead of holding it)
	auto tiles = [&]() { return MODE == kExpandPartition ? __ldg(a.status + 1) : total_tiles; };
	Rec<WORDS>* __restrict__ out = reinterpret_cast<Rec<WORDS>*>(a.recs);

	for (uint32_t g = blockIdx.x; g < tiles(); g += gridDim.x) {
		const uint4 da = __ldg(a.tile_desc + 2 * (size_t)g), db = __ldg(a.tile_desc + 2 * (size_t)g + 1);
		if (g + gridDim.x < tiles()) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.tile_desc + 2 * (size_t)(g + gridDim.x)));
		const uint64_t slot0 = da.x;
		const uint32_t nsk = da.y;
		const uint32_t j_lo = da.z;
		const uint32_t off_lo = da.w;
		const uint32_t tile_start = db.x & ~(uint32_t)(kExpandTile - 1);
		const uint32_t cnt = (db.x & (uint32_t)(kExpandTile - 1)) + 1u;
		const uint32_t* __restrict__ kpre = a.sk_kpre + slot0;
		const uint32_t* __restrict__ off = a.sk_off + slot0;
		const uintptr_t g0a = reinterpret_cast<uintptr_t>(a.bin + off_lo) & ~(uintptr_t)15;          // staging starts on the absolute 16-byte grid
		const uint32_t base_off = (uint32_t)(reinterpret_cast<uintptr_t>(a.bin + off_lo) - g0a);

		__syncthreads();      // previous tile is done with the bitmap
		if (tid < (uint32_t)HW) hbits[tid] = 0;
		if (tid == 0) s_jmax = j_lo;
		__syncthreads();
		// head flags: super-k-mer j_lo + r starts at output slot kpre - tile_start; its index entry is staged in shared memory
		{
			uint32_t jm = j_lo;
			for (uint32_t j = j_lo + tid; j < nsk; j += kExpandThreads) {
				const uint32_t kp = kpre[j];
				if (j > j_lo && kp >= tile_start + cnt) break;
				const uint32_t rel = j - j_lo;
				if (rel < (uint32_t)MAXSK) s_bit[rel] = 8u * (base_off + (off[j] - off_lo) + 1u) + 2u * tile_start - 2u * kp;      // (mod 2^32; + 2 * slot is the k-mer's bit)
				if (j > j_lo) atomicOr(&hbits[(kp - tile_start) >> 5], 1u << ((kp - tile_start) & 31u));
				jm = j;
			}
			if (jm > j_lo) atomicMax(&s_jmax, jm);
		}
		__syncthreads();
		// stage the tile's bytes of the bin (contiguous: from its first super-k-mer to the end of its last one) when they fit
		const uint32_t j_hi = s_jmax;
		const uint64_t b_hi = j_hi + 1 < nsk ? (uint64_t)off[j_hi + 1] : (uint64_t)db.y;
		const uint64_t span = reinterpret_cast<uintptr_t>(a.bin + b_hi) - g0a;
		const bool staged = (j_hi - j_lo) < (uint32_t)MAXSK && span + 16 <= (uint64_t)STAGE;
		if (staged)
			for (uint32_t v = tid; v * 16 < span + 8; v += kExpandThreads) {
				uint4 x = __ldg(reinterpret_cast<const uint4*>(g0a) + v);
				x.x = __byte_perm(x.x, 0, 0x0123); x.y = __byte_perm(x.y, 0, 0x0123); x.z = __byte_perm(x.z, 0, 0x0123); x.w = __byte_perm(x.w, 0, 0x0123);
				reinterpret_cast<uint4*>(s_bytes)[v] = x;
			}
		// the super-k-mer of output slot s = number of head bits at or before s: prefix popcounts of the bitmap words (one warp)
		if (warp == 0) {
			constexpr int WPL = HW / 32;
			uint32_t c[WPL], tot = 0;
#pragma unroll
			for (int i = 0; i < WPL; ++i) { c[i] = __popc(hbits[lane * WPL + i]); tot += c[i]; }
			uint32_t inc = tot;
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) {
				const uint32_t x = __shfl_up_sync(0xffffffffu, inc, o);
				if (lane >= (uint32_t)o) inc += x;
			}
			uint32_t ex = inc - tot;
#pragma unroll
			for (int i = 0; i < WPL; ++i) { hpre[lane * WPL + i] = ex; ex += c[i]; }
		}
		__syncthreads();

		// striped extraction: consecutive lanes <-> consecutive output k-mers
		const uint64_t obase = ((uint64_t)db.w << 32) | db.z;
		auto kmer_of = [&](uint32_t slot) -> Rec<WORDS> {
			const uint32_t rel = hpre[slot >> 5] + __popc(hbits[slot >> 5] & le_mask);          // (slot = i * threads + tid: bit (slot & 31) is this lane's)
			if (staged) return extract_kmer_be32<WORDS>(reinterpret_cast<const uint32_t*>(s_bytes), s_bit[rel] + 2u * slot, a.k, a.both_strands != 0);
			const uint32_t j = j_lo + rel;
			const uint32_t s = tile_start + slot - kpre[j];
			return extract_kmer<WORDS>(a.bin + off[j] + 1, s, a.k, a.both_strands != 0,
				[](uintptr_t wa) { return __ldg(reinterpret_cast<const unsigned long long*>(wa)); });
		};
		if constexpr (MODE == kExpandAll) {
#pragma unroll kExpandUnroll
			for (int i = 0; i < IPT; ++i) {
				const uint32_t slot = i * kExpandThreads + tid;
				if (slot < cnt) {
					const Rec<WORDS> r = kmer_of(slot);
					out[obase + slot] = r;
					atomicAdd(&htop[rec_top_digit<WORDS>(r, a.top_shift)], 1u);
				}
			}
			__syncthreads();
			// this tile is one work item of the level-1 partition: its digit counts go straight into the cell layout
			if (tid < 256) {
				a.cells1[(uint64_t)tid * total_tiles + g] = (uint16_t)htop[tid];
				htop[tid] = 0;
			}
			if (tid == 0) { a.item_lo1[g] = obase; a.item_cnt1[g] = (uint16_t)cnt; }
		} else if constexpr (MODE == kExpandPartition) {
			// level-1 partition of the tile straight from the bin (msd_partition_kernel's consumer, with the extraction in place of the load):
			// rank inside (tile, digit) = return value of one shared-memory atomicAdd, the tile's run inside every bucket = return value of
			// one global atomicAdd, scan of the digit counts, regroup by digit in shared memory, digit-contiguous runs leave with coalesced stores
			__shared__ uint32_t s_excl[256], s_goff[256];
			Rec<WORDS> key[IPT];
			uint32_t rank[IPT / 2] = {};          // two 16-bit ranks per register (a tile holds at most 4096 records)
#pragma unroll
			for (int i = 0; i < IPT; ++i) {
				const uint32_t slot = i * kExpandThreads + tid;
				if (slot < cnt) {
					key[i] = kmer_of(slot);
					rank[i / 2] |= atomicAdd(&htop[rec_top_digit<WORDS>(key[i], a.top_shift)], 1u) << (16 * (i & 1));
				}
			}
			__syncthreads();
			uint32_t c = 0, inc = 0, base = 0;
			if (tid < 256) {          // (warps 0..7; every thread zeroes its own digit for the next tile)
				c = htop[tid];
				htop[tid] = 0;
				if (c) base = atomicAdd(&a.l1_cursor[tid], c);          // (issued first: its latency hides behind the scan)
				inc = c;
#pragma unroll
				for (int o = 1; o < 32; o <<= 1) {
					const uint32_t x = __shfl_up_sync(0xffffffffu, inc, o);
					if (lane >= (uint32_t)o) inc += x;
				}
				if (lane == 31) warp_max[warp] = inc;
			}
			__syncthreads();
			bool overrun = false;
			if (tid < 256) {
				uint32_t ex = inc - c;
#pragma unroll
				for (int w = 0; w < 8; ++w) if ((uint32_t)w < warp) ex += warp_max[w];
				s_excl[tid] = ex;
				s_goff[tid] = base - ex;          // global index of tile-sorted position q is s_goff[d] + q
				// a run beyond its bucket: the walk's totals and this expansion disagree (a bug, never valid input).  The bin then ends as
				// a reported error, and the tile writes nothing.  (The boundaries of a bin of < 2^32 records fit in 32 bits.)
				overrun = c && (uint64_t)base + c > (uint32_t)__ldg(a.l1_start + tid + 1);
				if (overrun) { atomicOr(a.status, kErrRecCount); atomicOr(&a.flags[0], kExpandAbortFlag); atomicOr(&a.flags[1], kExpandAbortFlag); }
			}
			if (__syncthreads_or(overrun)) continue;
			// every k-mer of the tile is in registers: the staged bytes are free for the regrouping (the next tile stages after a barrier)
			Rec<WORDS>* buf = reinterpret_cast<Rec<WORDS>*>(s_bytes);
#pragma unroll
			for (int i = 0; i < IPT; ++i) {
				const uint32_t slot = i * kExpandThreads + tid;
				if (slot < cnt) buf[s_excl[rec_top_digit<WORDS>(key[i], a.top_shift)] + ((rank[i / 2] >> (16 * (i & 1))) & 0xFFFFu)] = key[i];
			}
			__syncthreads();
#pragma unroll
			for (int i = 0; i < IPT; ++i) {
				const uint32_t q = i * kExpandThreads + tid;
				if (q < cnt) {
					const Rec<WORDS> r = buf[q];
					out[s_goff[rec_top_digit<WORDS>(r, a.top_shift)] + q] = r;
				}
			}
		} else if constexpr (MODE == kExpandCount12) {
			// oversized bin, first pass: where do the k-mers fall?  (top 12 bits; nothing is written)
			for (int i = 0; i < IPT; ++i) {
				const uint32_t slot = i * kExpandThreads + tid;
				if (slot < cnt) {
					const Rec<WORDS> r = kmer_of(slot);
					atomicAdd(reinterpret_cast<unsigned long long*>(a.hist12) + msd_free_bits<WORDS>(r, a.fshift, 0xFFFu), 1ull);
				}
			}
		} else if constexpr (MODE == kExpandScatter) {
			// oversized bin, all key blocks at once: rank inside (tile, block) from a shared-memory counter, one global atomicAdd per
			// (tile, block) reserves the run inside the block's region, the k-mers are extracted a second time and written there
			// (holding 8 wide records per thread across the barriers would cost the registers)
			__shared__ uint32_t s_bcnt[kExpandMaxBlocks];
			__shared__ unsigned long long s_bbase[kExpandMaxBlocks];
			for (uint32_t b = tid; b < a.n_blocks; b += kExpandThreads) s_bcnt[b] = 0;
			__syncthreads();
			uint16_t blk[IPT], rnk[IPT];
#pragma unroll
			for (int i = 0; i < IPT; ++i) {
				const uint32_t slot = i * kExpandThreads + tid;
				if (slot < cnt) {
					const Rec<WORDS> r = kmer_of(slot);
					blk[i] = a.blk_of_prefix[msd_free_bits<WORDS>(r, a.fshift, 0xFFFu)];          // 0xFFFF: not a k-mer of these blocks (another GPU's key range)
					if (blk[i] != 0xFFFFu) rnk[i] = (uint16_t)atomicAdd(&s_bcnt[blk[i]], 1u);
				}
			}
			__syncthreads();
			for (uint32_t b = tid; b < a.n_blocks; b += kExpandThreads) {
				const uint32_t c = s_bcnt[b];
				if (c) s_bbase[b] = a.region_start[b] + atomicAdd(a.out_counter + b, (unsigned long long)c);
			}
			__syncthreads();
#pragma unroll
			for (int i = 0; i < IPT; ++i) {
				const uint32_t slot = i * kExpandThreads + tid;
				if (slot < cnt && blk[i] != 0xFFFFu) out[s_bbase[blk[i]] + rnk[i]] = kmer_of(slot);
			}
		} else {
			// oversized bin, one key block: the k-mers of the block are appended densely (their order does not matter, they get sorted)
			for (int i = 0; i < IPT; ++i) {
				const uint32_t slot = i * kExpandThreads + tid;
				Rec<WORDS> r;
				bool keep = false;
				if (slot < cnt) { r = kmer_of(slot); keep = msd_free_bits<WORDS>(r, a.fshift, a.fmask) == a.fprefix; }
				const uint32_t bal = __ballot_sync(0xffffffffu, keep);
				__syncthreads();          // (warp_max / s_jmax are free again)
				if (lane == 0) warp_max[warp] = __popc(bal);
				__syncthreads();
				if (tid == 0) {
					uint32_t tot = 0;
					for (int w = 0; w < kExpandThreads / 32; ++w) { const uint32_t c = warp_max[w]; warp_max[w] = tot; tot += c; }
					s_fbase = tot ? atomicAdd(a.out_counter, (unsigned long long)tot) : 0ull;
				}
				__syncthreads();
				if (keep) out[s_fbase + warp_max[warp] + __popc(bal & lanemask_lt())] = r;
			}
		}
	}
}

}  // namespace kmcb
