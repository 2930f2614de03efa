// kmc_b200 — homopolymer compression of a batch on the GPU (`kmc -hc`, CSplitter::HomopolymerCompressSeq, kmc_core/splitter.cpp:424-435):
// every run of one base collapsed to a single base before stage 0, stage 1 or the small-k counter sees the batch.  Included by kmc_b200.cu
// after fastx.cuh (it reuses the parser's 64-byte thread loads, its CTA reduction, the CTA scan and the three-phase device scan).
//
// The rule, on a batch (reads joined by separators): byte i is dropped iff i > 0, b[i] is one of ACGTacgt and b[i-1] is the same base
// ignoring case.  Other bytes are never dropped.  The reference drops every repeated symbol code of one read (runs of N too), but each
// non-ACGT byte already ends an N-free segment in every count this library makes, a separator ends every read, and a batch starts on a
// read, so both rules give the same k-mers, super-k-mers, statistics and counts (DESIGN.md section 3.13).
//
// The output is stable and out of place, and it is padded back to the input length with '\n': separators produce no k-mer, record,
// statistic or count, so the kernels downstream run unchanged over `bytes` bytes and no size has to come back to the host.
//
// Kernels (3 launches per call, whatever the size; grids over tiles of kHcTile bytes, no per-byte global atomics):
//   hc_count_kernel            per tile: the kept bytes (each thread also reads the byte before its 64)
//   split_scan_top_kernel<0>   exclusive sum of the tile counts in place: every tile's output offset; the total after the last tile
//   hc_compact_kernel          per tile: the kept bytes at their CTA-scan offsets in shared memory, written out; the tile's share of the
//                              padding (its own input range past the total)
#pragma once
#include "fastx.cuh"

namespace kmcb {

constexpr uint32_t kHcThreads = kFastxThreads;                          // = kSplitThreads, what split_block_excl assumes
constexpr uint32_t kHcPer = kFastxPer;
constexpr uint32_t kHcTile = kFastxTile;                                // 16 KiB

__host__ __device__ constexpr uint64_t hc_tiles(uint64_t bytes) { return (bytes + kHcTile - 1) / kHcTile; }

// bit i: the thread's byte p0 + i (of its n) is kept
__device__ __forceinline__ uint64_t hc_keep(const uint8_t* __restrict__ seq, uint64_t p0, const FxBytes& b, uint32_t n)
{
	uint32_t prev = (p0 && n) ? split_code(seq[p0 - 1]) : 4u;             // 4: no base, never equal to one
	uint64_t keep = 0;
#pragma unroll
	for (uint32_t i = 0; i < kHcPer; ++i) {
		const uint32_t c = split_code(b[i]);
		if (i < n && (c == 4u || c != prev)) keep |= 1ull << i;
		prev = c;
	}
	return keep;
}

__global__ void __launch_bounds__(kHcThreads) hc_count_kernel(const uint8_t* __restrict__ seq, uint64_t bytes, uint64_t* __restrict__ tile_kept)
{
	__shared__ uint64_t s_red[kHcThreads / 32];
	const uint64_t p0 = (uint64_t)blockIdx.x * kHcTile + (uint64_t)threadIdx.x * kHcPer;
	FxBytes b;
	const uint32_t n = fastx_load(seq, bytes, p0, b);
	uint64_t kept[1] = {(uint64_t)__popcll(hc_keep(seq, p0, b, n))};
	fastx_block_reduce<0, 1>(kept, s_red);
	if (threadIdx.x == 0) tile_kept[blockIdx.x] = kept[0];
}

// tile_off[0, n_tiles): exclusive offsets, tile_off[n_tiles]: the kept bytes of the batch
__global__ void __launch_bounds__(kHcThreads) hc_compact_kernel(const uint8_t* __restrict__ seq, uint64_t bytes, const uint64_t* __restrict__ tile_off,
	uint64_t n_tiles, uint8_t* __restrict__ out)
{
	__shared__ uint64_t s_warp[kSplitThreads / 32];
	__shared__ uint8_t s_out[kHcTile];
	const uint64_t t0 = (uint64_t)blockIdx.x * kHcTile;
	const uint64_t p0 = t0 + (uint64_t)threadIdx.x * kHcPer;
	FxBytes b;
	const uint32_t n = fastx_load(seq, bytes, p0, b);
	const uint64_t keep = hc_keep(seq, p0, b, n);
	uint64_t total;
	uint32_t o = (uint32_t)split_block_excl<0>((uint64_t)__popcll(keep), s_warp, &total);
#pragma unroll
	for (uint32_t i = 0; i < kHcPer; ++i)
		if ((keep >> i) & 1ull) s_out[o++] = b[i];
	__syncthreads();
	const uint64_t base = tile_off[blockIdx.x];
	for (uint32_t i = threadIdx.x; i < (uint32_t)total; i += kHcThreads) out[base + i] = s_out[i];
	// every output byte past the batch's kept bytes lies in exactly one tile's input range
	const uint64_t kept_all = tile_off[n_tiles];
	const uint64_t t1 = t0 + kHcTile < bytes ? t0 + kHcTile : bytes;
	for (uint64_t i = (t0 > kept_all ? t0 : kept_all) + threadIdx.x; i < t1; i += kHcThreads) out[i] = '\n';
}

// The 3 launches on `st`: seq[0, bytes) -> out[0, bytes), compressed and padded.  tile holds hc_tiles(bytes) + 1 words.  bytes > 0.
inline cudaError_t hc_launch(const uint8_t* seq, uint64_t bytes, uint64_t* tile, uint8_t* out, cudaStream_t st)
{
	const uint64_t n_tiles = hc_tiles(bytes);
	hc_count_kernel<<<(unsigned)n_tiles, kHcThreads, 0, st>>>(seq, bytes, tile);
	split_scan_top_kernel<0><<<1, kSplitThreads, 0, st>>>(tile, n_tiles, tile + n_tiles);
	hc_compact_kernel<<<(unsigned)n_tiles, kHcThreads, 0, st>>>(seq, bytes, tile, n_tiles, out);
	return cudaGetLastError();
}

}  // namespace kmcb
