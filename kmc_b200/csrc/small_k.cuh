// kmc_b200 — small k (k <= 13) on the GPU: a direct array of 4^k counters instead of bins, the reference's small-k mode
// (CSplitter::ProcessReadsSmallK, kmc_core/splitter.cpp:681-805, and CSmallKCompleter::CompleteKMCFormat, kb_completer.h:148-308).
// Included by kmc_b200.cu.
//
// The batch format is kmcb200_split's: every byte other than ACGTacgt separates, so a k-mer is counted exactly when its k bases are all
// ACGT.  Its value is its 2k-bit code (first symbol most significant), or min(code, reverse complement) with both strands.
// Kernels:
//   smallk_count_kernel<true>   k <= 7: privatised u32 counters in shared memory, a persistent grid, non-zero entries flushed with u64
//                               atomics at the end
//   smallk_count_kernel<false>  k >= 8: one u64 atomic per run of equal values straight on the 4^k counters (L2-resident up to k = 11)
//   smallk_finish_kernel        per tile of 4096 counters: kept k-mers, and the four totals (unique, below cutoff_min, above cutoff_max,
//                               sum of the counts)
//   smallk_emit_kernel          per tile: the records of the kept k-mers in k-mer order, staged in shared memory and stored coalesced, and
//                               the LUT entries whose prefix starts in the tile
// The tile words are scanned between finish and emit by split_scan_launch.
#pragma once
#include "split.cuh"

namespace kmcb {

constexpr uint32_t kSmallKMax = 13;
constexpr uint32_t kSmallKSharedMax = 7;                                // 4^7 u32 = 64 KiB of shared counters
constexpr uint32_t kSmallKThreads = 256;
constexpr uint32_t kSmallKPer = 16;                                     // consecutive positions (or counters) per thread
constexpr uint32_t kSmallKTile = kSmallKThreads * kSmallKPer;
constexpr uint32_t kSmallKHalo = kSmallKMax - 1;
constexpr uint32_t kSmallKMaxRec = 3 + 8;                               // (13 - 1) / 4 suffix bytes + an 8-byte counter
enum { kSkUnique = 0, kSkCutMin = 1, kSkCutMax = 2, kSkTotal = 3, kSkKept = 4, kSkWords = 8 };

// reverse complement of a k-mer code (k <= 16) from its bits, as split_norm computes it
__device__ __forceinline__ uint32_t smallk_revcomp(uint32_t x, uint32_t k)
{
	uint32_t r = __brev(~x);
	r = ((r >> 1) & 0x55555555u) | ((r & 0x55555555u) << 1);
	return r >> (32 - 2 * k);
}

// cnt[value] += every k-mer of the batch.  A tile is kSmallKTile k-mer end positions; thread j walks positions 16 j .. 16 j + 15 of it
// with a rolling code over the bases from k - 1 before them, and adds a run of equal values once.
template <bool SHARED>
__global__ void __launch_bounds__(kSmallKThreads) smallk_count_kernel(const uint8_t* __restrict__ seq, uint64_t len, uint32_t k,
	uint32_t both_strands, unsigned long long* __restrict__ cnt)
{
	extern __shared__ uint32_t s_cnt[];                                 // [4^k] when SHARED
	__shared__ uint8_t s_code[kSmallKTile + kSmallKHalo + 4];
	const uint32_t tid = threadIdx.x;
	const uint32_t n_cnt = 1u << (2 * k);
	const uint32_t mask = n_cnt - 1u;
	const uint64_t n_tiles = (len + kSmallKTile - 1) / kSmallKTile;
	if (SHARED) {
		for (uint32_t i = tid; i < n_cnt; i += kSmallKThreads) s_cnt[i] = 0;
	}
	auto add = [&](uint32_t v, uint32_t n) {
		if (SHARED) atomicAdd(&s_cnt[v], n);
		else atomicAdd(&cnt[v], (unsigned long long)n);
	};
	for (uint64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
		const uint64_t t0 = tile * kSmallKTile;
		__syncthreads();
		// s_code[i] = code of base t0 - kSmallKHalo + i (4 outside the batch)
		for (uint32_t i = tid; i < kSmallKTile + kSmallKHalo; i += kSmallKThreads) {
			const int64_t b = (int64_t)t0 - (int64_t)kSmallKHalo + (int64_t)i;
			s_code[i] = (b >= 0 && (uint64_t)b < len) ? (uint8_t)split_code(seq[b]) : (uint8_t)4;
		}
		__syncthreads();
		const uint8_t* c = s_code + kSmallKHalo + tid * kSmallKPer - (k - 1);
		uint32_t x = 0, ok = 0;                                         // rolling code, ACGT bases since the last separator
		for (uint32_t j = 0; j + 1 < k; ++j) {
			const uint32_t b = c[j];
			x = (x << 2) | (b & 3u);
			ok = b < 4 ? ok + 1 : 0;
		}
		uint32_t pv = 0, pn = 0;                                        // the pending run of equal values
#pragma unroll
		for (uint32_t e = 0; e < kSmallKPer; ++e) {
			const uint32_t b = c[k - 1 + e];
			x = ((x << 2) | (b & 3u)) & mask;
			ok = b < 4 ? ok + 1 : 0;
			if (ok >= k) {
				uint32_t v = x;
				if (both_strands) { const uint32_t r = smallk_revcomp(x, k); v = r < x ? r : x; }
				if (pn && v == pv) {
					++pn;
				} else {
					if (pn) add(pv, pn);
					pv = v;
					pn = 1;
				}
			}
		}
		if (pn) add(pv, pn);
	}
	if (SHARED) {
		__syncthreads();
		for (uint32_t i = tid; i < n_cnt; i += kSmallKThreads)
			if (s_cnt[i]) atomicAdd(&cnt[i], (unsigned long long)s_cnt[i]);
	}
}

// a counter's class: 0 absent, 1 below cutoff_min, 2 above cutoff_max, 3 kept
__device__ __forceinline__ uint32_t smallk_class(uint64_t c, uint64_t cutoff_min, uint64_t cutoff_max)
{
	return c == 0 ? 0u : c < cutoff_min ? 1u : c > cutoff_max ? 2u : 3u;
}

// one CTA per tile of kSmallKTile counters: tile_kept[tile] = kept k-mers of the tile; stats[kSkUnique .. kSkTotal] += the tile's totals
__global__ void __launch_bounds__(kSmallKThreads) smallk_finish_kernel(const uint64_t* __restrict__ cnt, uint64_t n_cnt, uint64_t cutoff_min,
	uint64_t cutoff_max, uint64_t* __restrict__ tile_kept, unsigned long long* __restrict__ stats)
{
	__shared__ uint64_t s_warp[kSplitThreads / 32];
	const uint64_t i0 = (uint64_t)blockIdx.x * kSmallKTile + (uint64_t)threadIdx.x * kSmallKPer;
	uint64_t n[4] = {0, 0, 0, 0};                                       // unique, below, above, kept
	uint64_t total = 0;
#pragma unroll
	for (uint32_t e = 0; e < kSmallKPer; ++e) {
		const uint64_t c = i0 + e < n_cnt ? cnt[i0 + e] : 0;
		const uint32_t cl = smallk_class(c, cutoff_min, cutoff_max);
		n[0] += cl != 0;
		n[1] += cl == 1;
		n[2] += cl == 2;
		n[3] += cl == 3;
		total += c;
	}
	uint64_t t[5];
	split_block_excl<0>(n[0], s_warp, &t[0]);
	split_block_excl<0>(n[1], s_warp, &t[1]);
	split_block_excl<0>(n[2], s_warp, &t[2]);
	split_block_excl<0>(n[3], s_warp, &t[3]);
	split_block_excl<0>(total, s_warp, &t[4]);
	if (threadIdx.x == 0) {
		tile_kept[blockIdx.x] = t[3];
		if (t[0]) {
			atomicAdd(&stats[kSkUnique], (unsigned long long)t[0]);
			atomicAdd(&stats[kSkCutMin], (unsigned long long)t[1]);
			atomicAdd(&stats[kSkCutMax], (unsigned long long)t[2]);
			atomicAdd(&stats[kSkTotal], (unsigned long long)t[4]);
		}
	}
}

// One CTA per tile of counters, after tile_kept has been scanned (exclusive): the tile's records go to out at record tile_kept[tile], each
// suffix_bytes of the value (most significant first) and then min(count, counter_max) in counter_size bytes (least significant first).
// lut[p] = kept k-mers below p * 4^(k - lp), written by the thread that holds counter p * 4^(k - lp).
__global__ void __launch_bounds__(kSmallKThreads) smallk_emit_kernel(const uint64_t* __restrict__ cnt, uint64_t n_cnt, uint64_t cutoff_min,
	uint64_t cutoff_max, uint64_t counter_max, uint32_t suffix_bytes, uint32_t counter_size, uint32_t suffix_bits,
	const uint64_t* __restrict__ tile_kept, uint8_t* __restrict__ out, uint64_t* __restrict__ lut)
{
	__shared__ uint64_t s_warp[kSplitThreads / 32];
	__shared__ __align__(16) uint8_t s_out[kSmallKTile * kSmallKMaxRec];
	const uint64_t i0 = (uint64_t)blockIdx.x * kSmallKTile + (uint64_t)threadIdx.x * kSmallKPer;
	const uint32_t rec = suffix_bytes + counter_size;
	uint64_t c[kSmallKPer];
	uint32_t kept = 0;
#pragma unroll
	for (uint32_t e = 0; e < kSmallKPer; ++e) {
		c[e] = i0 + e < n_cnt ? cnt[i0 + e] : 0;
		kept += smallk_class(c[e], cutoff_min, cutoff_max) == 3;
	}
	uint64_t block_kept;
	uint32_t r = (uint32_t)split_block_excl<0>(kept, s_warp, &block_kept);
	const uint64_t base = tile_kept[blockIdx.x];
	const uint64_t span_mask = (1ull << suffix_bits) - 1;
#pragma unroll
	for (uint32_t e = 0; e < kSmallKPer; ++e) {
		const uint64_t i = i0 + e;
		if (i < n_cnt && (i & span_mask) == 0) lut[i >> suffix_bits] = base + r;
		if (smallk_class(c[e], cutoff_min, cutoff_max) != 3) continue;
		uint8_t* o = s_out + (uint64_t)r * rec;
		for (uint32_t j = 0; j < suffix_bytes; ++j) o[j] = (uint8_t)(i >> (8 * (suffix_bytes - 1 - j)));
		const uint64_t v = c[e] < counter_max ? c[e] : counter_max;
		for (uint32_t j = 0; j < counter_size; ++j) o[suffix_bytes + j] = (uint8_t)(v >> (8 * j));
		++r;
	}
	__syncthreads();
	const uint64_t bytes = block_kept * rec;
	uint8_t* dst = out + base * rec;
	for (uint64_t j = threadIdx.x; j < bytes; j += kSmallKThreads) dst[j] = s_out[j];
}

}  // namespace kmcb
