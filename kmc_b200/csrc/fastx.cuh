// kmc_b200 — reads text -> batch on the GPU (include/kmc_b200.h, "reads text -> batch"): one chunk of a FASTQ or FASTA file becomes the
// batch kmcb200_split and kmcb200_sigstats_add take, byte for byte what kmc_b200.reads.sequences_to_batch makes of it.  Included by
// kmc_b200.cu after split.cuh (it reuses the three-phase device scans and the CTA scan).
//
// The parse is a byte classification plus a stable compaction.  What a byte becomes depends only on the state of the line it lies in:
//   FASTQ  the line's index modulo 4 (lines counted from the chunk's start): line 1 of every 4 is kept with its '\n';
//   FASTA  whether the line starts with '>': a header becomes its '\n', any other line is kept without its '\n' (blank lines vanish).
// So a tile's kept-byte count is a function of the state the tile is entered in, and a tile records it for every possible entry state.
//
// Kernels (9 launches per call, whatever the size; grids over tiles of kFastxTile bytes, no per-byte global atomics):
//   fastx_tile_kernel     per tile: '\n' count (FASTQ) or 1 + its last '\n' (FASTA); kept bytes, last record end and first record end at or
//                         past `limit`, each for every entry state
//   split_scan_*_kernel   exclusive sum (FASTQ) / max (FASTA) of the first word over the tiles: every tile's entry state
//   fastx_select_kernel   the entry state's kept count per tile; the last record end and the limit cut over all tiles (one atomic per CTA)
//   split_scan_*_kernel   exclusive sum of the selected kept counts: every tile's output offset
//   fastx_compact_kernel  per tile: consumed / error from the record ends, each byte's class again, a CTA scan, the kept bytes below
//                         consumed staged in shared memory and written out; the result words
#pragma once
#include "split.cuh"

namespace kmcb {

constexpr uint32_t kFastxThreads = 256;
constexpr uint32_t kFastxPer = 64;                                       // bytes per thread: four 16-byte loads
constexpr uint32_t kFastxTile = kFastxThreads * kFastxPer;               // 16 KiB
constexpr uint64_t kFastxNone = ~0ull;

// per-tile summary words, each an array of n_tiles (state s = FASTQ line phase 0..3, FASTA 0 / 1 = not / a header line)
enum { kFxScan = 0, kFxKept = 1, kFxLast = 5, kFxLim = 9, kFxSel = 13, kFxState = 14, kFxWords = 15 };
// work words: scan total ('\n' count / start of the last line), last record end, first record end >= limit
enum { kFwTotal = 0, kFwLast = 1, kFwLim = 2, kFwWords = 4 };
// result words
enum { kFrConsumed = 0, kFrSeqBytes = 1, kFrRecords = 2, kFrError = 3, kFrWords = 4 };

// a thread's 64 bytes, four to a register (byte i in bits 8 (i % 4) of word i / 4); indices are compile-time after unrolling
struct FxBytes {
	uint32_t w[kFastxPer / 4];
	__device__ __forceinline__ uint8_t operator[](uint32_t i) const { return (uint8_t)(w[i >> 2] >> (8 * (i & 3u))); }
};

// the thread's bytes [p0, p0 + n), n = min(64, bytes - p0); 16-byte loads where the chunk is aligned and the run is whole
__device__ __forceinline__ uint32_t fastx_load(const uint8_t* __restrict__ raw, uint64_t bytes, uint64_t p0, FxBytes& b)
{
	const uint32_t n = p0 >= bytes ? 0u : (uint32_t)(bytes - p0 < kFastxPer ? bytes - p0 : kFastxPer);
	if (n == kFastxPer && ((reinterpret_cast<uintptr_t>(raw) & 15u) == 0)) {
		const uint4* v = reinterpret_cast<const uint4*>(raw + p0);
#pragma unroll
		for (uint32_t q = 0; q < kFastxPer / 16; ++q) {
			const uint4 x = __ldg(v + q);
			b.w[4 * q] = x.x; b.w[4 * q + 1] = x.y; b.w[4 * q + 2] = x.z; b.w[4 * q + 3] = x.w;
		}
	} else {
#pragma unroll
		for (uint32_t q = 0; q < kFastxPer / 4; ++q) {
			uint32_t x = 0;
#pragma unroll
			for (uint32_t j = 0; j < 4; ++j) x |= (4 * q + j < n ? (uint32_t)raw[p0 + 4 * q + j] : 0u) << (8 * j);
			b.w[q] = x;
		}
	}
	return n;
}

// CTA reduction of N values (OP 0 sum, 1 max, 2 min); the result is valid in every thread.  Ends with a barrier.
template <int OP, int N>
__device__ __forceinline__ void fastx_block_reduce(uint64_t (&v)[N], uint64_t* s_red /* [N * kFastxThreads / 32] */)
{
	auto op = [](uint64_t a, uint64_t b) { return OP == 0 ? a + b : OP == 1 ? (a > b ? a : b) : (a < b ? a : b); };
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
#pragma unroll
	for (int i = 0; i < N; ++i) {
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) v[i] = op(v[i], __shfl_xor_sync(0xffffffffu, v[i], o));
		if (lane == 0) s_red[i * (kFastxThreads / 32) + warp] = v[i];
	}
	__syncthreads();
#pragma unroll
	for (int i = 0; i < N; ++i) {
		uint64_t r = s_red[i * (kFastxThreads / 32)];
		for (uint32_t w = 1; w < kFastxThreads / 32; ++w) r = op(r, s_red[i * (kFastxThreads / 32) + w]);
		v[i] = r;
	}
	__syncthreads();
}

// field r % 4 of four 16-bit fields packed in a word
__device__ __forceinline__ uint64_t fastx_field(uint64_t x, uint32_t r) { return (x >> (16 * (r & 3u))) & 0xffffu; }

// ------------------------------------------------------------------------------------------------ FASTQ thread summary
// Segment j of the thread = its bytes after its j-th '\n' up to and including the next one.  seg = the segment lengths summed by j % 4
// (16-bit fields).  With pre = the '\n's of the tile before the thread, the thread's m-th '\n' ends a record when the tile is entered in
// phase s = (3 - pre - m) % 4; last[s] / first[s] = the record end (1 + position) of the last such '\n' / the first one at or past limit
// (0 / kFastxNone: none).
struct FastqThread {
	uint64_t seg;
	uint64_t last[4], first[4];
};

__device__ __forceinline__ uint32_t fastq_newlines(const FxBytes& b, uint32_t n)
{
	uint32_t nl = 0;
#pragma unroll
	for (uint32_t i = 0; i < kFastxPer; ++i) nl += (i < n && b[i] == '\n');
	return nl;
}

__device__ __forceinline__ FastqThread fastq_thread(const FxBytes& b, uint32_t n, uint64_t p0, uint64_t limit, uint32_t pre)
{
	FastqThread t;
	t.seg = 0;
#pragma unroll
	for (int r = 0; r < 4; ++r) { t.last[r] = 0; t.first[r] = kFastxNone; }
	uint32_t m = 0;
#pragma unroll
	for (uint32_t i = 0; i < kFastxPer; ++i) {
		if (i < n) {
			t.seg += 1ull << (16 * (m & 3u));
			if (b[i] == '\n') {
				const uint64_t p = p0 + i + 1;
				const uint32_t st = (3u - pre - m) & 3u;
#pragma unroll
				for (uint32_t r = 0; r < 4; ++r) {
					if (st == r) {
						t.last[r] = p;
						if (p >= limit && t.first[r] == kFastxNone) t.first[r] = p;
					}
				}
				++m;
			}
		}
	}
	return t;
}

// ------------------------------------------------------------------------------------------------ FASTA thread summary
// keep[h]: bytes kept when the line running into the thread is (h = 1) or is not a header; has_nl / exit_hdr: whether the thread holds a '\n'
// and whether the line after its last '\n' is a header; line: 1 + the position of its last '\n' (0: none); last / first: record ends (header
// starts after a '\n') as for FASTQ.
struct FastaThread {
	uint32_t keep[2];
	bool has_nl, exit_hdr;
	uint64_t line, last, first;
};

__device__ __forceinline__ FastaThread fasta_thread(const FxBytes& b, uint32_t n, uint8_t next, uint64_t p0, uint64_t bytes, uint64_t limit)
{
	FastaThread t;
	uint32_t k0 = 0, rest = 0;
	bool hdr = false;
	t.has_nl = false;
	t.line = 0;
	t.last = 0;
	t.first = kFastxNone;
#pragma unroll
	for (uint32_t i = 0; i < kFastxPer; ++i) {
		if (i < n) {
			const uint8_t nx = i + 1 < n ? b[i + 1 < kFastxPer ? i + 1 : i] : next;
			if (b[i] == '\n') {
				if (t.has_nl) rest += hdr;
				t.has_nl = true;
				hdr = nx == '>';
				const uint64_t p = p0 + i + 1;
				t.line = p;
				if (hdr && p < bytes) {                                  // a header start after a '\n' ends the record before it
					t.last = p;
					if (p >= limit && t.first == kFastxNone) t.first = p;
				}
			} else if (t.has_nl) {
				rest += !hdr;
			} else {
				++k0;
			}
		}
	}
	t.exit_hdr = hdr;
	t.keep[0] = k0 + rest;
	t.keep[1] = (t.has_nl ? 1u : 0u) + rest;
	return t;
}

// the byte after the thread's bytes (FASTA looks one byte ahead: a record end is a '\n' followed by '>')
__device__ __forceinline__ uint8_t fastx_next(const uint8_t* __restrict__ raw, uint64_t bytes, uint64_t p0, uint32_t n)
{
	return (n == kFastxPer && p0 + n < bytes) ? raw[p0 + n] : (uint8_t)0;
}

// The entry state of every thread of a FASTA tile: the exit state of the latest thread before it that holds a '\n', else the tile's.
__device__ __forceinline__ uint32_t fasta_entry(const FastaThread& t, uint32_t tile_state, uint64_t* s_warp)
{
	const uint64_t v = t.has_nl ? (((uint64_t)threadIdx.x + 1) << 1) | (t.exit_hdr ? 1u : 0u) : 0u;
	const uint64_t prev = split_block_excl<1>(v, s_warp, nullptr);
	return prev ? (uint32_t)(prev & 1u) : tile_state;
}

// ------------------------------------------------------------------------------------------------ tile pass
template <bool FQ>
__global__ void __launch_bounds__(kFastxThreads) fastx_tile_kernel(const uint8_t* __restrict__ raw, uint64_t bytes, uint64_t limit, uint64_t n_tiles,
	uint64_t* __restrict__ sum, uint64_t* __restrict__ work, uint64_t* __restrict__ result)
{
	__shared__ uint64_t s_warp[kSplitThreads / 32];
	__shared__ uint64_t s_red[12 * kFastxThreads / 32];
	const uint64_t tile = blockIdx.x;
	const uint64_t p0 = tile * kFastxTile + (uint64_t)threadIdx.x * kFastxPer;
	if (tile == 0 && threadIdx.x == 0) {
		work[kFwLast] = 0;
		work[kFwLim] = kFastxNone;
		result[kFrRecords] = 0;
	}
	FxBytes b;
	const uint32_t n = fastx_load(raw, bytes, p0, b);
	if (FQ) {
		uint64_t tot;
		const uint32_t pre = (uint32_t)split_block_excl<0>(fastq_newlines(b, n), s_warp, &tot);
		const FastqThread t = fastq_thread(b, n, p0, limit, pre);
		// tile entry phase s: the thread's segment j has phase (s + pre + j) % 4, kept when 1
		uint64_t kept[4], last[4], first[4];
#pragma unroll
		for (uint32_t s = 0; s < 4; ++s) {
			kept[s] = fastx_field(t.seg, 1u - s - pre);
			last[s] = t.last[s];
			first[s] = t.first[s];
		}
		fastx_block_reduce<0, 4>(kept, s_red);
		fastx_block_reduce<1, 4>(last, s_red);
		fastx_block_reduce<2, 4>(first, s_red);
		if (threadIdx.x == 0) {
			sum[kFxScan * n_tiles + tile] = tot;
#pragma unroll
			for (uint32_t s = 0; s < 4; ++s) {
				sum[(kFxKept + s) * n_tiles + tile] = kept[s];
				sum[(kFxLast + s) * n_tiles + tile] = last[s];
				sum[(kFxLim + s) * n_tiles + tile] = first[s];
			}
		}
	} else {
		const FastaThread t = fasta_thread(b, n, fastx_next(raw, bytes, p0, n), p0, bytes, limit);
		const uint64_t v = t.has_nl ? (((uint64_t)threadIdx.x + 1) << 1) | (t.exit_hdr ? 1u : 0u) : 0u;
		const uint64_t prev = split_block_excl<1>(v, s_warp, nullptr);
		uint64_t kept[2];
#pragma unroll
		for (uint32_t h = 0; h < 2; ++h) kept[h] = (prev ? (prev & 1u) : h) ? t.keep[1] : t.keep[0];
		uint64_t mx[2] = {t.last, t.line}, mn[1] = {t.first};            // mx[1]: where the line running into the next tile starts
		fastx_block_reduce<0, 2>(kept, s_red);
		fastx_block_reduce<1, 2>(mx, s_red);
		fastx_block_reduce<2, 1>(mn, s_red);
		if (threadIdx.x == 0) {
			sum[kFxScan * n_tiles + tile] = mx[1];
#pragma unroll
			for (uint32_t h = 0; h < 2; ++h) {
				sum[(kFxKept + h) * n_tiles + tile] = kept[h];
				sum[(kFxLast + h) * n_tiles + tile] = mx[0];
				sum[(kFxLim + h) * n_tiles + tile] = mn[0];
			}
		}
	}
}

// ------------------------------------------------------------------------------------------------ entry states, record ends
// One thread per tile: the entry state from the scanned first word (FASTQ: '\n's before the tile mod 4; FASTA: the line running into
// the tile starts at the scanned position, a header when that byte is '>'), its kept count and record ends.
template <bool FQ>
__global__ void __launch_bounds__(kFastxThreads) fastx_select_kernel(const uint8_t* __restrict__ raw, uint64_t bytes, uint64_t n_tiles,
	uint64_t* __restrict__ sum, uint64_t* __restrict__ work)
{
	__shared__ uint64_t s_red[2 * kFastxThreads / 32];
	const uint64_t t = (uint64_t)blockIdx.x * kFastxThreads + threadIdx.x;
	uint64_t mx[1] = {0}, mn[1] = {kFastxNone};
	if (t < n_tiles) {
		const uint64_t x = sum[kFxScan * n_tiles + t];
		const uint32_t s = FQ ? (uint32_t)(x & 3u) : ((x < bytes && raw[x] == '>') ? 1u : 0u);
		sum[kFxSel * n_tiles + t] = sum[(kFxKept + s) * n_tiles + t];
		sum[kFxState * n_tiles + t] = s;
		mx[0] = sum[(kFxLast + s) * n_tiles + t];
		mn[0] = sum[(kFxLim + s) * n_tiles + t];
	}
	fastx_block_reduce<1, 1>(mx, s_red);
	fastx_block_reduce<2, 1>(mn, s_red);
	if (threadIdx.x == 0) {
		if (mx[0]) atomicMax(reinterpret_cast<unsigned long long*>(work + kFwLast), (unsigned long long)mx[0]);
		if (mn[0] != kFastxNone) atomicMin(reinterpret_cast<unsigned long long*>(work + kFwLim), (unsigned long long)mn[0]);
	}
}

// ------------------------------------------------------------------------------------------------ the cut
// consumed: a final chunk is parsed to its end, a non-final one to its last record end; with limit < bytes, to the first record end at or
// past limit when there is one (kmc_b200.reads._record_end(data, limit - 1)).  Its FASTA rule never ends a record at an unterminated last
// line of the data, so neither does this.  Returns false for a non-final chunk without a record end.
__device__ __forceinline__ bool fastx_cut(const uint8_t* __restrict__ raw, uint64_t bytes, uint32_t is_final, uint64_t limit, bool fq,
	const uint64_t* __restrict__ work, uint64_t* consumed)
{
	const uint64_t lim = work[kFwLim], last = work[kFwLast];
	const bool use_lim = limit < bytes && lim != kFastxNone;
	if (is_final) {
		*consumed = bytes;
		if (use_lim) *consumed = (!fq && lim == work[kFwTotal] && raw[bytes - 1] != '\n') ? bytes : lim;
		return true;
	}
	*consumed = use_lim ? lim : last;
	return *consumed != 0;
}

// ------------------------------------------------------------------------------------------------ compaction
template <bool FQ>
__global__ void __launch_bounds__(kFastxThreads) fastx_compact_kernel(const uint8_t* __restrict__ raw, uint64_t bytes, uint32_t is_final, uint64_t limit,
	uint64_t n_tiles, const uint64_t* __restrict__ sum, const uint64_t* __restrict__ work, uint8_t* __restrict__ seq, uint64_t* __restrict__ result)
{
	__shared__ uint64_t s_warp[kSplitThreads / 32];
	__shared__ uint64_t s_red[kFastxThreads / 32];
	__shared__ uint8_t s_out[kFastxTile + 16];
	const uint64_t tile = blockIdx.x;
	const uint64_t p0 = tile * kFastxTile + (uint64_t)threadIdx.x * kFastxPer;
	uint64_t consumed;
	const bool ok = fastx_cut(raw, bytes, is_final, limit, FQ, work, &consumed);
	// the appended '\n' of a final chunk without one, when its last line is kept with its '\n'
	bool extra = false;
	if (is_final && bytes && consumed == bytes && raw[bytes - 1] != '\n') {
		const uint64_t tot = work[kFwTotal];
		extra = FQ ? (tot & 3u) == 1u : raw[tot] == '>';
	}
	if (tile == 0 && threadIdx.x == 0) {
		result[kFrConsumed] = ok ? consumed : 0;
		result[kFrError] = ok ? 0 : 1;
		if (!ok || consumed == 0) result[kFrSeqBytes] = 0;
		if (ok && consumed) atomicAdd(reinterpret_cast<unsigned long long*>(result + kFrRecords), 1ull);
	}
	if (!ok || tile * kFastxTile >= consumed) return;                   // uniform over the CTA
	FxBytes b;
	const uint32_t n = fastx_load(raw, bytes, p0, b);
	const uint32_t state = (uint32_t)sum[kFxState * n_tiles + tile];
	uint64_t keep = 0, ends = 0;                                        // kept-byte mask, record ends below consumed
	if (FQ) {
		uint32_t ph = (state + (uint32_t)split_block_excl<0>(fastq_newlines(b, n), s_warp, nullptr)) & 3u;
#pragma unroll
		for (uint32_t i = 0; i < kFastxPer; ++i) {
			if (i < n && p0 + i < consumed) {
				if (ph == 1u) keep |= 1ull << i;
				if (b[i] == '\n') {
					ends += (ph == 3u && p0 + i + 1 < consumed);
					ph = (ph + 1) & 3u;
				}
			}
		}
	} else {
		const uint8_t next = fastx_next(raw, bytes, p0, n);
		const FastaThread t = fasta_thread(b, n, next, p0, bytes, limit);
		bool hdr = fasta_entry(t, state, s_warp) != 0;
#pragma unroll
		for (uint32_t i = 0; i < kFastxPer; ++i) {
			if (i < n && p0 + i < consumed) {
				if (b[i] == '\n') {
					if (hdr) keep |= 1ull << i;
					const uint8_t nx = i + 1 < n ? b[i + 1 < kFastxPer ? i + 1 : i] : next;
					hdr = nx == '>';
					ends += (hdr && p0 + i + 1 < consumed);
				} else if (!hdr) {
					keep |= 1ull << i;
				}
			}
		}
	}
	uint64_t total;
	uint64_t o = split_block_excl<0>((uint64_t)__popcll(keep), s_warp, &total);
#pragma unroll
	for (uint32_t i = 0; i < kFastxPer; ++i)
		if ((keep >> i) & 1ull) s_out[o++] = b[i];
	uint64_t cnt[1] = {ends};
	fastx_block_reduce<0, 1>(cnt, s_red);                              // ends with a barrier: s_out is complete
	const uint64_t base = sum[kFxSel * n_tiles + tile];
	for (uint64_t i = threadIdx.x; i < total; i += kFastxThreads) seq[base + i] = s_out[i];
	if (threadIdx.x == 0) {
		if (cnt[0]) atomicAdd(reinterpret_cast<unsigned long long*>(result + kFrRecords), (unsigned long long)cnt[0]);
		if ((consumed - 1) / kFastxTile == tile) {                      // the tile holding the last parsed byte
			if (extra) seq[base + total] = '\n';
			result[kFrSeqBytes] = base + total + (extra ? 1 : 0);
		}
	}
}

}  // namespace kmcb
