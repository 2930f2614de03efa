// kmc_b200 — BAM records -> batch on the GPU (include/kmc_b200.h, "reads text -> batch", formats KMCB200_BAM / KMCB200_BAM_ORIGINAL_STRAND):
// one chunk of decompressed BAM record bytes becomes the batch kmcb200_split takes, byte for byte what kmc_b200.reads.bam_to_batch makes
// of it, which is what KMC's CSplitter::GetSeq reads from a BAM file (kmc_core/splitter.cpp:326-418).  Included by kmc_b200.cu after
// fastx.cuh (it reuses its tile size, result words and the three-phase device scans).
//
// The record starts form a chain, next(p) = p + 4 + block_size(p), that no finite-state tile summary captures.  The walk is made exact
// for any block layout and parallel in the common case by guessing every tile's first record start and checking the guesses in order:
//   bam_tile_kernel     per 16 KiB tile: every position tested (in rounds of 256, first one wins) for a well-formed whole record with a
//                       NUL-terminated name followed by two more — the tile's guess; one thread walks the chain from the guess until it
//                       leaves the tile and records the exit, how the walk stopped, and the kept records and their output bytes
//   bam_resolve_kernel  one warp, 32 tiles per step: the true entry of tile 0 is 0, of tile t the true exit of tile t-1.  A tile entered
//                       at or past its end holds no record start; one entered at its guess keeps its walk; any other is walked again from
//                       the true entry (the only serial cost, paid where a guess was wrong).  Decides consumed and the error.
//   split_scan_*        exclusive sum of (kept records << 32 | output bytes) over the tiles: every tile's first kept record and output
//                       offset (3 launches)
//   bam_table_kernel    one thread per tile: the tile's kept records' starts and output offsets, walked from the resolved entry
//   bam_decode_kernel   one CTA per 16 KiB of output: each thread's 64 output bytes, its first record found by binary search; SEQ
//                       nibbles through a 16-entry table, reverse complemented for FLAG 0x10 with KMCB200_BAM_ORIGINAL_STRAND, a '\n'
//                       after each record; staged in shared memory and stored 16 bytes at a time
// 7 launches per call, whatever the size; consumed, the cut and the error never leave the device.
#pragma once
#include "fastx.cuh"

namespace kmcb {

constexpr uint32_t kBamThreads = kFastxThreads;
constexpr uint32_t kBamTile = kFastxTile;                                // 16 KiB of chunk per tile, 16 KiB of output per decode CTA
constexpr uint32_t kBamPer = kBamTile / kBamThreads;                     // output bytes per decode thread
constexpr uint32_t kBamMinRecord = 36;                                   // block_size word + 32 fixed bytes
constexpr uint32_t kBamOutShift = 32;                                    // scan word: kept records << 32 | output bytes
static_assert(KMCB200_SPLIT_MAX_BATCH <= (1ull << kBamOutShift) && KMCB200_SPLIT_MAX_BATCH / kBamMinRecord < (1ull << (64 - kBamOutShift)),
	"a chunk's output bytes and its kept records each fit their half of the scan word");

// per-tile words in the parser's summary buffer (each an array of n_tiles)
enum { kBsGuess = 0, kBsExit = 1, kBsStatus = 2, kBsScan = 3, kBsEntry = 4, kBsWords = 5 };
// work words
enum { kBwConsumed = 0, kBwError = 1, kBwTotal = 2, kBwWords = 3 };
// how a walk stopped: left the tile; stopped for good (end of the chunk or the limit cut), consumed = exit; the record at exit is not
// whole in the chunk; the record at exit is malformed
enum { kBamOn = 0, kBamStop = 1, kBamPartial = 2, kBamBad = 3 };
// result word kFrError: 0, or one of these
enum { kBamErrTooLong = 1, kBamErrTruncated = 2, kBamErrMalformed = 3 };

__device__ __forceinline__ uint32_t bam_u32(const uint8_t* __restrict__ raw, uint64_t p)
{
	return (uint32_t)raw[p] | ((uint32_t)raw[p + 1] << 8) | ((uint32_t)raw[p + 2] << 16) | ((uint32_t)raw[p + 3] << 24);
}

struct BamRec {
	uint64_t next;                                                       // the record's end
	uint32_t l_seq, flag;
	uint64_t seq;                                                        // the SEQ nibbles' first byte
};

// The record at p: kBamOn when it is whole in the chunk and well formed (r filled in), kBamPartial when it is not whole, kBamBad when its
// block_size is below 32, its l_seq negative, or its fixed fields do not fit its block_size.
__device__ __forceinline__ uint32_t bam_record(const uint8_t* __restrict__ raw, uint64_t bytes, uint64_t p, BamRec& r)
{
	if (bytes - p < 4) return kBamPartial;
	const int32_t bs = (int32_t)bam_u32(raw, p);
	if (bs < 32) return kBamBad;
	if (bytes - p - 4 < (uint64_t)bs) return kBamPartial;
	const uint32_t l_name = raw[p + 12];
	const uint32_t n_cigar = (uint32_t)raw[p + 16] | ((uint32_t)raw[p + 17] << 8);
	const int32_t l_seq = (int32_t)bam_u32(raw, p + 20);
	if (l_seq < 0) return kBamBad;
	if (32ull + l_name + 4ull * n_cigar + ((uint64_t)l_seq + 1) / 2 + (uint64_t)l_seq > (uint64_t)bs) return kBamBad;
	r.next = p + 4 + (uint64_t)bs;
	r.l_seq = (uint32_t)l_seq;
	r.flag = (uint32_t)raw[p + 18] | ((uint32_t)raw[p + 19] << 8);
	r.seq = p + 36 + l_name + 4ull * n_cigar;
	return kBamOn;
}

__device__ __forceinline__ bool bam_kept(uint32_t flag) { return (flag & 0x900u) == 0; }

struct BamWalk {
	uint64_t exit, scan;
	uint32_t status;
};

// The chain from `p` through the tile ending at t1 (and no further than the limit cut).  scan: kept records << 32 | their l_seq + 1 summed.
__device__ __forceinline__ BamWalk bam_walk(const uint8_t* __restrict__ raw, uint64_t bytes, uint64_t limit, uint64_t p, uint64_t t1)
{
	BamWalk w{p, 0, kBamOn};
	while (true) {
		if (w.exit >= bytes) { w.status = kBamStop; break; }
		if (w.exit >= t1) break;
		BamRec r;
		const uint32_t st = bam_record(raw, bytes, w.exit, r);
		if (st != kBamOn) { w.status = st; break; }
		if (bam_kept(r.flag)) w.scan += (1ull << kBamOutShift) + r.l_seq + 1;
		w.exit = r.next;
		if (limit < bytes && w.exit >= limit) { w.status = kBamStop; break; }
	}
	return w;
}

// ------------------------------------------------------------------------------------------------ tile pass
// A guess: a whole well-formed record with a NUL-terminated name, followed by two more (or by the chunk's end).  Bytes inside a record
// (qualities, tags, the fixed fields of a neighbour) pass the first test now and then; the chain test rejects nearly all of them.  A
// true record whose chain runs into the unfinished record at the chunk's end is rejected too: that tile is walked again by the resolve.
__device__ __forceinline__ bool bam_guess_ok(const uint8_t* __restrict__ raw, uint64_t bytes, uint64_t p)
{
	for (uint32_t step = 0; step < 3 && p < bytes; ++step) {
		BamRec r;
		if (bytes - p < kBamMinRecord || bam_record(raw, bytes, p, r) != kBamOn) return false;
		const uint32_t l_name = raw[p + 12];
		if (l_name == 0 || raw[p + 36 + l_name - 1] != 0) return false;
		p = r.next;
	}
	return true;
}

__global__ void __launch_bounds__(kBamThreads) bam_tile_kernel(const uint8_t* __restrict__ raw, uint64_t bytes, uint64_t limit, uint64_t n_tiles,
	uint64_t* __restrict__ sum)
{
	__shared__ uint32_t s_first;
	const uint64_t tile = blockIdx.x;
	const uint64_t t0 = tile * kBamTile, t1 = t0 + kBamTile;
	if (threadIdx.x == 0) s_first = ~0u;
	__syncthreads();
	for (uint32_t r = 0; r < kBamTile / kBamThreads; ++r) {
		const uint32_t off = r * kBamThreads + threadIdx.x;
		const uint64_t p = t0 + off;
		const bool cand = p < bytes && bam_guess_ok(raw, bytes, p);
		if (cand) atomicMin(&s_first, off);
		if (__syncthreads_or(cand)) break;
	}
	if (threadIdx.x != 0) return;
	const uint64_t guess = s_first == ~0u ? kFastxNone : t0 + s_first;
	sum[kBsGuess * n_tiles + tile] = guess;
	if (guess == kFastxNone) return;
	const BamWalk w = bam_walk(raw, bytes, limit, guess, t1);
	sum[kBsExit * n_tiles + tile] = w.exit;
	sum[kBsStatus * n_tiles + tile] = w.status;
	sum[kBsScan * n_tiles + tile] = w.scan;
}

// ------------------------------------------------------------------------------------------------ resolve
// One warp.  Lane i holds tile c0 + i's guess and walk; the entries are settled tile by tile in registers, the wrong guesses walked
// again by the whole warp (uniform control flow: every lane reads the same bytes).  Writes every tile's entry (kFastxNone past the end of
// the chain) and scan word, and the work words consumed / error.
__global__ void __launch_bounds__(32) bam_resolve_kernel(const uint8_t* __restrict__ raw, uint64_t bytes, uint32_t is_final, uint64_t limit,
	uint64_t n_tiles, uint64_t* __restrict__ sum, uint64_t* __restrict__ work)
{
	const uint32_t lane = threadIdx.x;
	uint64_t e = 0, consumed = 0;
	uint32_t err = 0;
	bool ended = false;
	for (uint64_t c0 = 0; c0 < n_tiles; c0 += 32) {
		const uint64_t t = c0 + lane;
		uint64_t g = kFastxNone, x = 0, s = 0, my_scan = 0, my_entry = kFastxNone;
		if (t < n_tiles) {
			g = sum[kBsGuess * n_tiles + t];
			if (g != kFastxNone) { x = sum[kBsExit * n_tiles + t]; s = sum[kBsStatus * n_tiles + t]; my_scan = sum[kBsScan * n_tiles + t]; }
		}
		const uint32_t n = (uint32_t)(n_tiles - c0 < 32 ? n_tiles - c0 : 32);
		for (uint32_t i = 0; i < n; ++i) {
			const uint64_t gi = __shfl_sync(0xffffffffu, g, i), xi = __shfl_sync(0xffffffffu, x, i);
			const uint32_t si = (uint32_t)__shfl_sync(0xffffffffu, s, i);
			if (ended) { if (lane == i) my_scan = 0; continue; }
			const uint64_t t1 = (c0 + i + 1) * kBamTile;
			if (lane == i) my_entry = e;
			if (e >= t1) { if (lane == i) my_scan = 0; continue; }   // no record starts in this tile
			BamWalk w{xi, 0, si};
			if (e != gi) {
				w = bam_walk(raw, bytes, limit, e, t1);
				if (lane == i) my_scan = w.scan;
			}
			e = w.exit;
			if (w.status == kBamOn) continue;
			ended = true;
			if (w.status == kBamStop) consumed = e;
			else if (w.status == kBamBad) err = kBamErrMalformed;
			else if (is_final) err = kBamErrTruncated;
			else consumed = e;
		}
		if (t < n_tiles) {
			sum[kBsEntry * n_tiles + t] = my_entry;
			sum[kBsScan * n_tiles + t] = my_scan;
		}
	}
	if (!ended) consumed = e;
	if (!err && !is_final && consumed == 0) err = kBamErrTooLong;
	if (lane == 0) {
		work[kBwConsumed] = err ? 0 : consumed;
		work[kBwError] = err;
	}
}

// ------------------------------------------------------------------------------------------------ record table
// One thread per tile: the kept records that start in it, below consumed.  Thread 0 also writes the result words.
__global__ void __launch_bounds__(kBamThreads) bam_table_kernel(const uint8_t* __restrict__ raw, uint64_t bytes, uint64_t n_tiles,
	const uint64_t* __restrict__ sum, const uint64_t* __restrict__ work, uint64_t* __restrict__ rec_start, uint64_t* __restrict__ rec_out,
	uint64_t* __restrict__ result)
{
	const uint64_t t = (uint64_t)blockIdx.x * kBamThreads + threadIdx.x;
	const uint64_t err = work[kBwError], consumed = work[kBwConsumed], total = work[kBwTotal];
	if (t == 0) {
		result[kFrConsumed] = err ? 0 : consumed;
		result[kFrSeqBytes] = err ? 0 : total & ((1ull << kBamOutShift) - 1);
		result[kFrRecords] = err ? 0 : total >> kBamOutShift;
		result[kFrError] = err;
	}
	if (err || t >= n_tiles) return;
	const uint64_t t1 = (t + 1) * kBamTile;
	uint64_t p = sum[kBsEntry * n_tiles + t];
	const uint64_t base = sum[kBsScan * n_tiles + t];
	uint64_t j = base >> kBamOutShift, o = base & ((1ull << kBamOutShift) - 1);
	while (p < t1 && p < consumed) {
		BamRec r;
		bam_record(raw, bytes, p, r);                                      // well formed: the resolve walked it
		if (bam_kept(r.flag)) {
			rec_start[j] = p;
			rec_out[j] = o;
			++j;
			o += r.l_seq + 1;
		}
		p = r.next;
	}
}

// ------------------------------------------------------------------------------------------------ decode
// SEQ code -> base: =ACMGRSVTWYHKDBN, only A C G T (1 2 4 8) are bases, every other code an N; rc: the complement
__device__ __forceinline__ uint8_t bam_base(uint32_t code, bool rc)
{
	switch (code) {
	case 1: return rc ? 'T' : 'A';
	case 2: return rc ? 'G' : 'C';
	case 4: return rc ? 'C' : 'G';
	case 8: return rc ? 'A' : 'T';
	default: return 'N';
	}
}

// Thread t's q-th 16 bytes of output are kept in shared slot t * 4 + (q ^ ((t >> 1) & 3)): the eight threads of one phase of a 16-byte
// store then hit eight different groups of four banks.
__device__ __forceinline__ uint32_t bam_slot(uint32_t c /* 16-byte piece of the CTA's output */)
{
	const uint32_t t = c >> 2, q = c & 3u;
	return t * 4 + (q ^ ((t >> 1) & 3u));
}

__global__ void __launch_bounds__(kBamThreads) bam_decode_kernel(const uint8_t* __restrict__ raw, uint32_t original_strand,
	const uint64_t* __restrict__ work, const uint64_t* __restrict__ rec_start, const uint64_t* __restrict__ rec_out, uint8_t* __restrict__ seq)
{
	__shared__ uint4 s_out[kBamTile / 16];
	if (work[kBwError]) return;
	const uint64_t total = work[kBwTotal] & ((1ull << kBamOutShift) - 1), n_rec = work[kBwTotal] >> kBamOutShift;
	const uint64_t c0 = (uint64_t)blockIdx.x * kBamTile;
	if (c0 >= total) return;                                             // uniform over the CTA
	const uint64_t o0 = c0 + (uint64_t)threadIdx.x * kBamPer;
	if (o0 < total) {
		uint64_t lo = 0, hi = n_rec;                                       // the last record whose output starts at or before o0
		while (hi - lo > 1) {
			const uint64_t mid = (lo + hi) / 2;
			if (rec_out[mid] <= o0) lo = mid; else hi = mid;
		}
		uint64_t r = lo, R = rec_out[r];
		BamRec rec;
		bam_record(raw, ~0ull, rec_start[r], rec);
		bool rc = original_strand && (rec.flag & 0x10u);
		for (uint32_t q = 0; q < kBamPer / 16; ++q) {
			uint32_t word[4] = {0, 0, 0, 0};
#pragma unroll
			for (uint32_t b = 0; b < 16; ++b) {
				const uint64_t o = o0 + 16 * q + b;
				if (o < total) {
					while (o > R + rec.l_seq) {                             // past this record's '\n'
						R = rec_out[++r];
						bam_record(raw, ~0ull, rec_start[r], rec);
						rc = original_strand && (rec.flag & 0x10u);
					}
					const uint64_t i = o - R;
					uint8_t c = '\n';
					if (i < rec.l_seq) {
						const uint64_t j = rc ? rec.l_seq - 1 - i : i;
						c = bam_base((raw[rec.seq + j / 2] >> ((j & 1) ? 0 : 4)) & 15u, rc);
					}
					word[b / 4] |= (uint32_t)c << (8 * (b & 3u));
				}
			}
			s_out[bam_slot(threadIdx.x * 4 + q)] = make_uint4(word[0], word[1], word[2], word[3]);
		}
	}
	__syncthreads();
	const uint64_t n = total - c0 < kBamTile ? total - c0 : kBamTile;
	const uint8_t* s_bytes = reinterpret_cast<const uint8_t*>(s_out);
	uint64_t head = 0;                                                   // bytes stored 16 at a time
	if ((reinterpret_cast<uintptr_t>(seq) & 15u) == 0) {
		head = n / 16 * 16;
		for (uint32_t c = threadIdx.x; c < n / 16; c += kBamThreads) reinterpret_cast<uint4*>(seq + c0)[c] = s_out[bam_slot(c)];
	}
	for (uint64_t i = head + threadIdx.x; i < n; i += kBamThreads)
		seq[c0 + i] = s_bytes[16 * bam_slot((uint32_t)(i / 16)) + (i & 15u)];
}

}  // namespace kmcb
