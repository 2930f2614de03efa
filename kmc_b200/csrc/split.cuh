// kmc_b200 — stage 1 on the GPU: a batch of reads -> KMC bins of minimizer super-k-mers (the work of CSplitter::ProcessReads,
// kmc_core/splitter.cpp:557-677, and CKmerBinCollector::PutExtendedKmer, kb_collector.cpp:34-90).  Included by kmc_b200.cu.
//
// The reference walks every read serially.  Its loop is equivalent to a rule per k-mer, and that rule is what these kernels compute
// over flat positions of the batch (DESIGN.md section 3.8):
//   * symbol codes: ACGTacgt -> 0..3, every other byte ends the N-free segment it lies in (a read separator is just such a byte);
//   * the signature of a k-mer is the minimum over its k-m+1 m-mers of norm(m-mer) = min(m-mer if allowed, its reverse complement if
//     allowed), where a disallowed orientation counts as the special value 4^m (kmc_api/mmer.h:40-91);
//   * a super-k-mer is a maximal run of consecutive k-mers of one segment with one signature value, cut every 256 k-mers counted from
//     the start of the run (the len == kmer_len + 255 branch);
//   * records are `n - k`, then the n symbols 4 per byte, first symbol in bits 7-6 (kb_collector.cpp:57-71); a bin's stream holds its
//     records in input order.
//
// Kernels (one launch each, all grids over positions or records, none walks a read):
//   split_signature_kernel   per k-mer: m-mer values, windowed minimum (log-step sparse table in shared memory), run starts per tile
//   split_scan_*_kernel      three-phase device scans (sum / max) of per-tile values
//   split_records_kernel     record starts and ends from the run starts (count pass, then compaction pass)
//   split_bin_hist_kernel    per record tile: bytes / k-mers / records per bin
//   split_rank_kernel        stable rank of every record inside its bin -> output offset; expander pack starts
//   split_frag_kernel        per-bin fragments, pack numbering, sizes and the capacity check
//   split_pack_bytes_kernel  pack lengths
//   split_emit_kernel        the packed records, written at their offsets
//   split_kxmer_kernel       opt-in (kmcb200_splitter_count_kxmers): per record tile, the collector's (k+x)-mer count per bin
// Stage 0 shares the windowed minimum (split_window_table) and adds one kernel of its own:
//   sigstats_kernel          k-mers per signature over a batch (CSplitter::CalcStats), runs aggregated per warp before the global atomics
#pragma once
#include "common.cuh"

namespace kmcb {

constexpr uint32_t kSplitThreads = 256;
constexpr uint32_t kSplitPerThread = 16;
constexpr uint32_t kSplitTile = kSplitThreads * kSplitPerThread;      // k-mer positions per CTA
constexpr uint32_t kSplitRecTile = 8192;                                 // records per tile of the bin histogram / rank
constexpr uint64_t kSplitPackWindow = 65536 - 128;                       // a record starting at s in a bin fragment belongs to pack s / 65408
constexpr uint32_t kSplitInvalid = 0x80000000u;                          // signature word of a k-mer that contains a non-ACGT byte
constexpr uint32_t kSplitMaxSpan = KMCB200_MAX_KMER_LEN;                 // halo of a position tile
constexpr uint32_t kSplitScanItems = 16;
constexpr uint32_t kSplitScanBlock = kSplitThreads * kSplitScanItems;    // elements per CTA of the device scans

// words of the splitter's device state (the device twin's d_result takes the first five)
enum { kStBytes = 0, kStPacks = 1, kStCapErr = 2, kStSuperKmers = 3, kStKmers = 4, kStRecords = 5, kStWords = 8 };

__device__ __forceinline__ uint32_t split_code(uint8_t c)
{
	switch (c) {
	case 'A': case 'a': return 0;
	case 'C': case 'c': return 1;
	case 'G': case 'g': return 2;
	case 'T': case 't': return 3;
	default: return 4;
	}
}

// An orientation of an m-mer is allowed unless it has AA at symbols (i, i+1) with i >= 1, starts with ACA, or ends with TT? or TGT.
__device__ __forceinline__ bool split_allowed(uint32_t x, uint32_t m)
{
	const uint32_t a = ~x & ~(x >> 1) & 0x55555555u;                     // bit 2j: symbol group j is A (group 0 = last symbol)
	if ((a & (a >> 2)) & ((1u << (2 * (m - 2))) - 1u)) return false;       // groups j, j+1 both A for j <= m-3, i.e. i = m-2-j >= 1
	if ((x >> (2 * (m - 3))) == 4u) return false;                         // first three symbols ACA
	if ((x & 0x3cu) == 0x3cu) return false;                               // last three symbols TT?
	if ((x & 0x3fu) == 0x3bu) return false;                               // last three symbols TGT
	return true;
}

__device__ __forceinline__ uint32_t split_norm(uint32_t x, uint32_t m)
{
	uint32_t r = __brev(~x);                                              // complement, reversed bit by bit ...
	r = ((r >> 1) & 0x55555555u) | ((r & 0x55555555u) << 1);              // ... and back to 2-bit symbols
	r >>= 32 - 2 * m;
	const uint32_t special = 1u << (2 * m);
	const uint32_t f = split_allowed(x, m) ? x : special;
	const uint32_t b = split_allowed(r, m) ? r : special;
	return f < b ? f : b;
}

// minimum of the values, OR of the invalid bit: associative, so windows can be assembled from power-of-two spans
__device__ __forceinline__ uint32_t split_combine(uint32_t a, uint32_t b)
{
	const uint32_t va = a & ~kSplitInvalid, vb = b & ~kSplitInvalid;
	return (va < vb ? va : vb) | ((a | b) & kSplitInvalid);
}

// exclusive scan over the CTA (one value per thread, kSplitThreads threads); OP 0 = sum, 1 = max
template <int OP>
__device__ __forceinline__ uint64_t split_block_excl(uint64_t v, uint64_t* s_warp /* [kSplitThreads/32] */, uint64_t* total)
{
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	uint64_t inc = v;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		const uint64_t t = __shfl_up_sync(0xffffffffu, inc, o);
		if (lane >= (uint32_t)o) inc = OP == 0 ? inc + t : (t > inc ? t : inc);
	}
	if (lane == 31) s_warp[warp] = inc;
	__syncthreads();
	uint64_t base = 0, tot = 0;
	for (uint32_t w = 0; w < kSplitThreads / 32; ++w) {
		const uint64_t t = s_warp[w];
		if (w < warp) base = OP == 0 ? base + t : (t > base ? t : base);
		tot = OP == 0 ? tot + t : (t > tot ? t : tot);
	}
	__syncthreads();
	if (total) *total = tot;
	// exclusive: the inclusive value of the previous lane, combined with the warps before
	uint64_t prev = __shfl_up_sync(0xffffffffu, inc, 1);
	if (lane == 0) prev = 0;
	return OP == 0 ? base + prev : (prev > base ? prev : base);
}

// ------------------------------------------------------------------------------------------------ per k-mer signatures
// The windowed minimum of one tile (kSplitTile k-mer positions t0 .. t0+T-1, plus t0-1): loads the bases [t0-1, t0+T+k-1) into s_code,
// their normalised m-mer values into s_val, and folds s_val into a log-step sparse table.  Returns `span`: the signature of position
// t0-1+i is then split_window_sig(s_val, i, w, span).  Called by every thread of the CTA; ends with a barrier.
__device__ __forceinline__ uint32_t split_window_table(const uint8_t* __restrict__ seq, uint64_t len, uint64_t t0, uint32_t k, uint32_t m,
	uint8_t* s_code /* [kSplitTile + kSplitMaxSpan + 8] */, uint32_t* s_val /* [kSplitTile + kSplitMaxSpan + 8] */)
{
	constexpr uint32_t kPer = (kSplitTile + kSplitMaxSpan + kSplitThreads) / kSplitThreads;
	const uint32_t tid = threadIdx.x;
	const uint32_t w = k - m + 1;
	const uint32_t n_base = kSplitTile + k, n_val = kSplitTile + w;
	for (uint32_t i = tid; i < n_base; i += kSplitThreads) {
		const int64_t b = (int64_t)t0 - 1 + (int64_t)i;
		s_code[i] = (b >= 0 && (uint64_t)b < len) ? (uint8_t)split_code(seq[b]) : (uint8_t)4;
	}
	__syncthreads();
	const uint32_t mask = (m == 16) ? 0xffffffffu : ((1u << (2 * m)) - 1u);
	for (uint32_t j = tid; j < n_val; j += kSplitThreads) {
		uint32_t x = 0, bad = 0;
		for (uint32_t q = 0; q < m; ++q) {
			const uint32_t c = s_code[j + q];
			bad |= c >> 2;
			x = (x << 2) | (c & 3u);
		}
		s_val[j] = bad ? kSplitInvalid : split_norm(x & mask, m);
	}
	__syncthreads();
	// sparse table: after the step with span s, s_val[j] covers the m-mers j .. j+2s-1
	uint32_t span = 1;
	while (2 * span <= w) {
		uint32_t nv[kPer];
#pragma unroll
		for (uint32_t e = 0; e < kPer; ++e) {
			const uint32_t j = tid + e * kSplitThreads;
			nv[e] = (j + span < n_val) ? split_combine(s_val[j], s_val[j + span]) : 0u;
		}
		__syncthreads();
#pragma unroll
		for (uint32_t e = 0; e < kPer; ++e) {
			const uint32_t j = tid + e * kSplitThreads;
			if (j + span < n_val) s_val[j] = nv[e];
		}
		__syncthreads();
		span *= 2;
	}
	return span;
}

// signature word of position t0-1+i of a tile after split_window_table (w = k - m + 1 m-mers per k-mer)
__device__ __forceinline__ uint32_t split_window_sig(const uint32_t* s_val, uint32_t i, uint32_t w, uint32_t span)
{
	return split_combine(s_val[i], s_val[i + w - span]);
}

// sig[t] = min of the m-mer values of the k-mer at t, with kSplitInvalid set when the k-mer holds a non-ACGT byte or runs past the batch.
// tile_last[tile] = 1 + the last position of the tile where a run of equal signatures starts (0: none).
__global__ void __launch_bounds__(kSplitThreads) split_signature_kernel(const uint8_t* __restrict__ seq, uint64_t len, uint32_t k, uint32_t m,
	uint32_t* __restrict__ sig, uint64_t* __restrict__ tile_last)
{
	__shared__ uint8_t s_code[kSplitTile + kSplitMaxSpan + 8];
	__shared__ uint32_t s_val[kSplitTile + kSplitMaxSpan + 8];
	__shared__ uint32_t s_last;
	const uint32_t tid = threadIdx.x;
	const uint64_t t0 = (uint64_t)blockIdx.x * kSplitTile;
	const uint32_t w = k - m + 1;
	if (tid == 0) s_last = 0;
	const uint32_t span = split_window_table(seq, len, t0, k, m, s_code, s_val);
	// positions t0-1+i for i = tid*16 .. tid*16+16
	const uint32_t i0 = tid * kSplitPerThread;
	uint32_t prev = split_window_sig(s_val, i0, w, span);
	uint32_t last = 0;
	for (uint32_t e = 1; e <= kSplitPerThread; ++e) {
		const uint32_t i = i0 + e;
		const uint32_t cur = split_window_sig(s_val, i, w, span);
		const uint64_t t = t0 - 1 + i;
		if (t < len) {
			sig[t] = cur;
			if (!(cur & kSplitInvalid) && cur != prev) last = (uint32_t)(t + 1);
		}
		prev = cur;
	}
	if (last) atomicMax(&s_last, last);
	__syncthreads();
	if (tid == 0) tile_last[blockIdx.x] = s_last;
}

// ------------------------------------------------------------------------------------------------ stage 0: k-mers per signature
// counts[sig] += the valid k-mers of the tile whose signature is sig (CSplitter::CalcStats, kmc_core/splitter.cpp:439-533, adds up the same
// numbers read by read).  Same tiles and windowed minimum as split_signature_kernel, but nothing per position leaves the chip: a run of equal
// signatures is counted where it ends.  Thread j of a warp holds 16 consecutive positions; the length of a run that enters it from lane
// j-1 (carry) comes from a segmented scan over the lanes, so a run costs one global atomic per warp it touches, however long it is.
__global__ void __launch_bounds__(kSplitThreads) sigstats_kernel(const uint8_t* __restrict__ seq, uint64_t len, uint32_t k, uint32_t m,
	uint32_t* __restrict__ counts)
{
	__shared__ uint8_t s_code[kSplitTile + kSplitMaxSpan + 8];
	__shared__ uint32_t s_val[kSplitTile + kSplitMaxSpan + 8];
	const uint32_t tid = threadIdx.x, lane = tid & 31u;
	const uint64_t t0 = (uint64_t)blockIdx.x * kSplitTile;
	const uint32_t w = k - m + 1;
	const uint32_t span = split_window_table(seq, len, t0, k, m, s_code, s_val);
	// this thread's positions t0 + 16 tid + e, e = 0..15, and the one before them
	const uint32_t i0 = tid * kSplitPerThread;
	const uint32_t before = split_window_sig(s_val, i0, w, span);
	uint32_t s[kSplitPerThread];
#pragma unroll
	for (uint32_t e = 0; e < kSplitPerThread; ++e) s[e] = split_window_sig(s_val, i0 + 1 + e, w, span);
	// in: position 0 continues the run of the position before it (lane 0 starts the warp's runs afresh)
	const bool in = lane != 0 && !(s[0] & kSplitInvalid) && s[0] == before;
	// tail: length of the run that ends at position 15 (0 when position 15 is invalid); whole: one run covers all 16 positions
	uint32_t tail = (s[kSplitPerThread - 1] & kSplitInvalid) ? 0u : 1u;
	bool open = tail != 0;
#pragma unroll
	for (int e = (int)kSplitPerThread - 2; e >= 0; --e) {
		open = open && s[e] == s[e + 1];
		tail += open;
	}
	const bool whole = tail == kSplitPerThread;
	// carry_j = in_j ? tail_{j-1} + (whole_{j-1} ? carry_{j-1} : 0) : 0, as an inclusive scan of the affine maps c -> a + b c
	const uint32_t prev_tail = __shfl_up_sync(0xffffffffu, tail, 1);
	const bool prev_whole = __shfl_up_sync(0xffffffffu, (uint32_t)whole, 1) != 0;
	uint32_t a = in ? prev_tail : 0u, b = (in && prev_whole) ? 1u : 0u;
#pragma unroll
	for (uint32_t o = 1; o < 32; o <<= 1) {
		const uint32_t pa = __shfl_up_sync(0xffffffffu, a, o), pb = __shfl_up_sync(0xffffffffu, b, o);
		if (lane >= o) { a += b * pa; b *= pb; }
	}
	const uint32_t carry = a;
	// out: the run that ends at position 15 goes on into lane j+1, which counts it
	const bool out = __shfl_down_sync(0xffffffffu, (uint32_t)in, 1) != 0 && lane != 31;
	uint32_t run = 0;
	bool first = true;                                                  // the current run started at position 0
#pragma unroll
	for (uint32_t e = 0; e < kSplitPerThread; ++e) {
		const uint32_t v = s[e];
		if (v & kSplitInvalid) { first = false; continue; }
		++run;
		const bool ends = e + 1 == kSplitPerThread ? !out : s[e + 1] != v;
		if (ends) {
			atomicAdd(&counts[v], run + (first && in ? carry : 0u));
			run = 0;
			first = false;
		}
	}
}

// ------------------------------------------------------------------------------------------------ device scans (in place, exclusive)
// The element count is `n`, or, when d_cnt is given, ceil(*d_cnt / div) * mul (sizes that are only known on the device).
__device__ __forceinline__ uint64_t split_scan_count(const uint64_t* d_cnt, uint64_t div, uint64_t mul, uint64_t n)
{
	return d_cnt ? (*d_cnt + div - 1) / div * mul : n;
}

template <int OP>
__global__ void __launch_bounds__(kSplitThreads) split_scan_reduce_kernel(const uint64_t* __restrict__ a, const uint64_t* d_cnt, uint64_t div,
	uint64_t mul, uint64_t n_host, uint64_t* __restrict__ partial)
{
	__shared__ uint64_t s_warp[kSplitThreads / 32];
	const uint64_t n = split_scan_count(d_cnt, div, mul, n_host);
	const uint64_t base = (uint64_t)blockIdx.x * kSplitScanBlock;
	uint64_t v = 0;
	if (base < n) {
		for (uint32_t e = 0; e < kSplitScanItems; ++e) {
			const uint64_t i = base + threadIdx.x + (uint64_t)e * kSplitThreads;
			if (i < n) { const uint64_t x = a[i]; v = OP == 0 ? v + x : (x > v ? x : v); }
		}
	}
	uint64_t tot;
	split_block_excl<OP>(v, s_warp, &tot);
	if (threadIdx.x == 0) partial[blockIdx.x] = tot;
}

// one CTA: exclusive scan of the n_part partial values; *d_total (optional) receives the total
template <int OP>
__global__ void __launch_bounds__(kSplitThreads) split_scan_top_kernel(uint64_t* __restrict__ partial, uint64_t n_part, uint64_t* d_total)
{
	__shared__ uint64_t s_warp[kSplitThreads / 32];
	uint64_t carry = 0;
	for (uint64_t c = 0; c < n_part; c += kSplitThreads) {
		const uint64_t i = c + threadIdx.x;
		const uint64_t v = i < n_part ? partial[i] : 0;
		uint64_t tot;
		const uint64_t ex = split_block_excl<OP>(v, s_warp, &tot);
		if (i < n_part) partial[i] = OP == 0 ? carry + ex : (carry > ex ? carry : ex);
		carry = OP == 0 ? carry + tot : (carry > tot ? carry : tot);
	}
	if (threadIdx.x == 0 && d_total) *d_total = carry;
}

template <int OP>
__global__ void __launch_bounds__(kSplitThreads) split_scan_down_kernel(uint64_t* __restrict__ a, const uint64_t* d_cnt, uint64_t div, uint64_t mul,
	uint64_t n_host, const uint64_t* __restrict__ partial)
{
	__shared__ uint64_t s_warp[kSplitThreads / 32];
	const uint64_t n = split_scan_count(d_cnt, div, mul, n_host);
	const uint64_t base = (uint64_t)blockIdx.x * kSplitScanBlock;
	if (base >= n) return;                                              // uniform over the CTA
	const uint64_t i0 = base + (uint64_t)threadIdx.x * kSplitScanItems;
	uint64_t x[kSplitScanItems];
	uint64_t v = 0;
#pragma unroll
	for (uint32_t e = 0; e < kSplitScanItems; ++e) {
		x[e] = (i0 + e < n) ? a[i0 + e] : 0;
		v = OP == 0 ? v + x[e] : (x[e] > v ? x[e] : v);
	}
	const uint64_t c = partial[blockIdx.x];
	uint64_t run = split_block_excl<OP>(v, s_warp, nullptr);
	run = OP == 0 ? run + c : (run > c ? run : c);
#pragma unroll
	for (uint32_t e = 0; e < kSplitScanItems; ++e) {
		if (i0 + e < n) a[i0 + e] = run;
		run = OP == 0 ? run + x[e] : (x[e] > run ? x[e] : run);
	}
}

// The three launches of an in-place exclusive scan of a device array (OP 0 = sum, 1 = max) on `st`, with d_partial holding at least
// ceil(n_max / kSplitScanBlock) words; see split_scan_count for d_cnt / div / mul.  Used by the splitter and the reads-text parser.
template <int OP>
inline cudaError_t split_scan_launch(uint64_t* a, uint64_t n_max, const uint64_t* d_cnt, uint64_t div, uint64_t mul, uint64_t* d_total,
	uint64_t* d_partial, cudaStream_t st)
{
	const uint64_t n_blocks = (n_max + kSplitScanBlock - 1) / kSplitScanBlock > 1 ? (n_max + kSplitScanBlock - 1) / kSplitScanBlock : 1;
	split_scan_reduce_kernel<OP><<<(unsigned)n_blocks, kSplitThreads, 0, st>>>(a, d_cnt, div, mul, n_max, d_partial);
	split_scan_top_kernel<OP><<<1, kSplitThreads, 0, st>>>(d_partial, n_blocks, d_total);
	split_scan_down_kernel<OP><<<(unsigned)n_blocks, kSplitThreads, 0, st>>>(a, d_cnt, div, mul, n_max, d_partial);
	return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ records
// Same tiles as split_signature_kernel.  carry[tile] = 1 + the last run start before the tile (exclusive max-scan of tile_last).
// A valid k-mer t starts a record when (t - start of its run) % 256 == 0; it ends one when t+1 is invalid or starts a record.
// Count pass (WRITE = false): cnt_start[tile], cnt_end[tile].  Write pass: rec_start / rec_end at the scanned offsets.
template <bool WRITE>
__global__ void __launch_bounds__(kSplitThreads) split_records_kernel(const uint32_t* __restrict__ sig, uint64_t len,
	const uint64_t* __restrict__ carry, uint64_t* __restrict__ cnt_start, uint64_t* __restrict__ cnt_end,
	uint32_t* __restrict__ rec_start, uint32_t* __restrict__ rec_end)
{
	__shared__ uint64_t s_warp[kSplitThreads / 32];
	const uint64_t t0 = (uint64_t)blockIdx.x * kSplitTile + (uint64_t)threadIdx.x * kSplitPerThread;
	auto sig_at = [&](int64_t t) -> uint32_t { return (t >= 0 && (uint64_t)t < len) ? sig[t] : kSplitInvalid; };
	uint32_t e[kSplitPerThread + 2];                                    // positions t0-1 .. t0+16
#pragma unroll
	for (uint32_t q = 0; q < kSplitPerThread + 2; ++q) e[q] = sig_at((int64_t)t0 - 1 + q);
	auto run_start = [&](uint32_t q) { return !(e[q] & kSplitInvalid) && e[q] != e[q - 1]; };   // for position t0-1+q
	uint64_t local = 0;
#pragma unroll
	for (uint32_t q = 1; q <= kSplitPerThread; ++q) if (run_start(q)) local = t0 + q;        // 1 + (t0 - 1 + q)
	uint64_t rs = split_block_excl<1>(local, s_warp, nullptr);
	const uint64_t c = carry[blockIdx.x];
	rs = rs > c ? rs : c;
	bool starts[kSplitPerThread + 1];
#pragma unroll
	for (uint32_t q = 1; q <= kSplitPerThread + 1; ++q) {
		if (run_start(q)) rs = t0 + q;
		const uint64_t t = t0 - 1 + q;
		starts[q - 1] = !(e[q] & kSplitInvalid) && ((t - (rs - 1)) & 255u) == 0;
	}
	uint32_t ns = 0, ne = 0;
#pragma unroll
	for (uint32_t q = 0; q < kSplitPerThread; ++q) {
		const bool valid = !(e[q + 1] & kSplitInvalid);
		ns += starts[q];
		ne += valid && ((e[q + 2] & kSplitInvalid) || starts[q + 1]);
	}
	uint64_t tot_s, tot_e;
	const uint64_t xs = split_block_excl<0>(ns, s_warp, &tot_s);
	const uint64_t xe = split_block_excl<0>(ne, s_warp, &tot_e);
	if (!WRITE) {
		if (threadIdx.x == 0) { cnt_start[blockIdx.x] = tot_s; cnt_end[blockIdx.x] = tot_e; }
		return;
	}
	uint64_t os = cnt_start[blockIdx.x] + xs, oe = cnt_end[blockIdx.x] + xe;
#pragma unroll
	for (uint32_t q = 0; q < kSplitPerThread; ++q) {
		const bool valid = !(e[q + 1] & kSplitInvalid);
		const uint32_t t = (uint32_t)(t0 + q);
		if (starts[q]) rec_start[os++] = t;
		if (valid && ((e[q + 2] & kSplitInvalid) || starts[q + 1])) rec_end[oe++] = t;
	}
}

__device__ __forceinline__ uint32_t split_rec_bytes(uint32_t first, uint32_t last, uint32_t k) { return 1u + (last - first + k + 3u) / 4u; }

// ------------------------------------------------------------------------------------------------ per-bin sizes
// One CTA per tile of kSplitRecTile records (the grid covers the worst case; tiles past the record count return).
// hist[b * n_rt + tile] = bytes of bin b's records in the tile; bin_kmers / bin_recs accumulate per bin.
__global__ void __launch_bounds__(kSplitThreads) split_bin_hist_kernel(const uint32_t* __restrict__ rec_start, const uint32_t* __restrict__ rec_end,
	const uint32_t* __restrict__ sig, const uint32_t* __restrict__ map, uint32_t k, uint32_t n_bins, const uint64_t* __restrict__ state,
	uint32_t* __restrict__ rec_bin, uint64_t* __restrict__ hist, unsigned long long* __restrict__ bin_kmers, unsigned long long* __restrict__ bin_recs)
{
	extern __shared__ uint32_t s_hist[];                               // [3][n_bins]: bytes, k-mers, records
	const uint64_t n_rec = state[kStRecords];
	const uint64_t n_rt = (n_rec + kSplitRecTile - 1) / kSplitRecTile;
	if (blockIdx.x >= n_rt) return;
	for (uint32_t b = threadIdx.x; b < 3 * n_bins; b += blockDim.x) s_hist[b] = 0;
	__syncthreads();
	const uint64_t r0 = (uint64_t)blockIdx.x * kSplitRecTile;
	const uint64_t r1 = r0 + kSplitRecTile < n_rec ? r0 + kSplitRecTile : n_rec;
	for (uint64_t r = r0 + threadIdx.x; r < r1; r += blockDim.x) {
		const uint32_t s = rec_start[r], e = rec_end[r];
		const uint32_t b = map[sig[s] & ~kSplitInvalid];
		rec_bin[r] = b;
		atomicAdd(&s_hist[b], split_rec_bytes(s, e, k));
		atomicAdd(&s_hist[n_bins + b], e - s + 1);
		atomicAdd(&s_hist[2 * n_bins + b], 1u);
	}
	__syncthreads();
	for (uint32_t b = threadIdx.x; b < n_bins; b += blockDim.x) {
		hist[(uint64_t)b * n_rt + blockIdx.x] = s_hist[b];
		if (s_hist[2 * n_bins + b]) {
			atomicAdd(&bin_kmers[b], (unsigned long long)s_hist[n_bins + b]);
			atomicAdd(&bin_recs[b], (unsigned long long)s_hist[2 * n_bins + b]);
		}
	}
}

// ------------------------------------------------------------------------------------------------ (k+x)-mers per bin (opt-in)
// The collector's n_plus_x_recs of one canonical record of n symbols (CKmerBinCollector::update_n_plus_x_recs, kb_collector.h:66-116):
// along the record, the order of the last 4 symbols of the k-mer and of its reverse complement's first 4 gives a state; a stretch of one
// strict state of x + 1 k-mers counts 1 + x / div, every k-mer of the equal state counts 1.
__device__ __forceinline__ uint32_t split_kxmer_canonical(const uint8_t* __restrict__ p, uint32_t n, uint32_t k, uint32_t div)
{
	auto sym = [&](uint32_t i) { return split_code(p[i]) & 3u; };
	auto order = [](uint32_t f, uint32_t r) { return f < r ? 0u : (r < f ? 1u : 2u); };
	uint32_t fw = (sym(0) << 6) | (sym(1) << 4) | (sym(2) << 2) | sym(3);
	uint32_t rc = ((3u - sym(k - 1)) << 6) | ((3u - sym(k - 2)) << 4) | ((3u - sym(k - 3)) << 2) | (3u - sym(k - 4));
	uint32_t cur = order(fw, rc), x = 0, total = 0;
	for (uint32_t i = 0; i + k < n; ++i) {
		rc = (rc >> 2) | ((3u - sym(k + i)) << 6);
		fw = ((fw << 2) | sym(4 + i)) & 0xffu;
		const uint32_t st = order(fw, rc);
		if (st == cur) {
			if (cur == 2) ++total;
			else ++x;
		} else {
			cur = st;
			total += 1 + x / div;
			x = 0;
		}
	}
	return total + 1 + x / div;
}

// Same record tiles as split_bin_hist_kernel (after it: rec_bin is set).  kx[b] += the (k+x)-mers of bin b's records, max_x > 0:
// 1 + (n - k) / (max_x + 1) per record of n symbols for plain k-mers (kb_collector.cpp:76-78), split_kxmer_canonical for canonical ones.
// Nothing is added for a batch whose outputs do not fit (the split writes nothing then either).
__global__ void __launch_bounds__(kSplitThreads) split_kxmer_kernel(const uint8_t* __restrict__ seq, const uint32_t* __restrict__ rec_start,
	const uint32_t* __restrict__ rec_end, const uint32_t* __restrict__ rec_bin, uint32_t k, uint32_t max_x, uint32_t both_strands, uint32_t n_bins,
	const uint64_t* __restrict__ state, unsigned long long* __restrict__ kx)
{
	extern __shared__ uint32_t s_kx[];                                 // [n_bins]
	if (state[kStCapErr]) return;
	const uint64_t n_rec = state[kStRecords];
	const uint64_t n_rt = (n_rec + kSplitRecTile - 1) / kSplitRecTile;
	if (blockIdx.x >= n_rt) return;
	for (uint32_t b = threadIdx.x; b < n_bins; b += blockDim.x) s_kx[b] = 0;
	__syncthreads();
	const uint64_t r0 = (uint64_t)blockIdx.x * kSplitRecTile;
	const uint64_t r1 = r0 + kSplitRecTile < n_rec ? r0 + kSplitRecTile : n_rec;
	for (uint64_t r = r0 + threadIdx.x; r < r1; r += blockDim.x) {
		const uint32_t s = rec_start[r];
		const uint32_t n = rec_end[r] - s + k;
		const uint32_t v = both_strands ? split_kxmer_canonical(seq + s, n, k, max_x + 1) : 1u + (n - k) / (max_x + 1);
		atomicAdd(&s_kx[rec_bin[r]], v);
	}
	__syncthreads();
	for (uint32_t b = threadIdx.x; b < n_bins; b += blockDim.x)
		if (s_kx[b]) atomicAdd(&kx[b], (unsigned long long)s_kx[b]);
}

__device__ __forceinline__ uint64_t split_bin_base(const uint64_t* hist, uint64_t n_rt, uint32_t b, uint32_t n_bins, const uint64_t* state)
{
	return b < n_bins ? hist[(uint64_t)b * n_rt] : state[kStBytes];
}

// ------------------------------------------------------------------------------------------------ stable rank inside the bins
// One warp per record tile, records in input order 32 at a time: equal bins in a round are found with match.any, their byte prefix with
// 32 shuffles, and a per-bin cursor in shared memory carries the offset from round to round.  hist holds the exclusive scan (output
// offset of every (bin, tile) block).  Also records where expander packs start: in bin b, the record that starts at offset s is in pack
// s / W; pack_start[slot_base(b) + p] = the offset of pack p's first record, with slot_base(b) = base(b) / W + b (disjoint per bin).
__global__ void __launch_bounds__(32) split_rank_kernel(const uint32_t* __restrict__ rec_start, const uint32_t* __restrict__ rec_end,
	const uint32_t* __restrict__ rec_bin, const uint64_t* __restrict__ hist, uint32_t k, uint32_t n_bins, const uint64_t* __restrict__ state,
	uint64_t* __restrict__ rec_dst, uint64_t* __restrict__ pack_start, uint64_t* __restrict__ bin_packs)
{
	extern __shared__ uint32_t s_cur[];                                // [n_bins]
	const uint64_t n_rec = state[kStRecords];
	const uint64_t n_rt = (n_rec + kSplitRecTile - 1) / kSplitRecTile;
	const uint32_t tile = blockIdx.x, lane = threadIdx.x;
	if (tile >= n_rt) return;
	for (uint32_t b = lane; b < n_bins; b += 32) s_cur[b] = 0;
	__syncwarp();
	const uint64_t r0 = (uint64_t)tile * kSplitRecTile;
	const uint64_t r1 = r0 + kSplitRecTile < n_rec ? r0 + kSplitRecTile : n_rec;
	for (uint64_t rb = r0; rb < r1; rb += 32) {
		const uint64_t r = rb + lane;
		const bool active = r < r1;
		const uint32_t b = active ? rec_bin[r] : 0xffffffffu;
		const uint32_t bytes = active ? split_rec_bytes(rec_start[r], rec_end[r], k) : 0u;
		const uint32_t peers = __match_any_sync(0xffffffffu, b);
		uint32_t pre = 0, tot = 0;
#pragma unroll
		for (int j = 0; j < 32; ++j) {
			const uint32_t v = __shfl_sync(0xffffffffu, bytes, j);
			if ((peers >> j) & 1u) { tot += v; if (j < (int)lane) pre += v; }
		}
		const uint32_t cur = active ? s_cur[b] : 0u;
		__syncwarp();
		if (active && lane == (uint32_t)(__ffs(peers) - 1)) s_cur[b] = cur + tot;
		__syncwarp();
		if (!active) continue;
		const uint64_t dst = hist[(uint64_t)b * n_rt + tile] + cur + pre;
		rec_dst[r] = dst;
		const uint64_t base = split_bin_base(hist, n_rt, b, n_bins, state);
		const uint64_t bin_bytes = split_bin_base(hist, n_rt, b + 1, n_bins, state) - base;
		const uint64_t s = dst - base, e = s + bytes;
		const uint64_t slot = base / kSplitPackWindow + b;
		if (s == 0) pack_start[slot] = 0;
		if (e < bin_bytes && e / kSplitPackWindow != s / kSplitPackWindow) pack_start[slot + e / kSplitPackWindow] = e;
		if (e == bin_bytes) bin_packs[b] = s / kSplitPackWindow + 1;
	}
}

// ------------------------------------------------------------------------------------------------ fragments, packs, capacity
// One CTA.  pack0[b] = exclusive scan of bin_packs; state[kStPacks] = total packs; the capacity flag; the fragments (only when the
// outputs fit: a capacity error leaves every output untouched); result[0..4] = bytes, packs, capacity error, super-k-mers, k-mers.
__global__ void __launch_bounds__(kSplitThreads) split_frag_kernel(const uint64_t* __restrict__ hist, const unsigned long long* __restrict__ bin_kmers,
	const unsigned long long* __restrict__ bin_recs, const uint64_t* __restrict__ bin_packs, uint32_t n_bins, uint64_t* __restrict__ state,
	uint64_t out_capacity, uint64_t pack_capacity, uint64_t* __restrict__ pack0, kmcb200_bin_fragment* __restrict__ frags, uint64_t* __restrict__ result)
{
	__shared__ uint64_t s_warp[kSplitThreads / 32];
	__shared__ uint64_t s_tot[3];
	const uint64_t n_rt = (state[kStRecords] + kSplitRecTile - 1) / kSplitRecTile;
	uint64_t carry = 0, sk = 0, km = 0;
	for (uint32_t c = 0; c < n_bins; c += kSplitThreads) {
		const uint32_t b = c + threadIdx.x;
		const uint64_t v = b < n_bins ? bin_packs[b] : 0;
		uint64_t tot;
		const uint64_t ex = split_block_excl<0>(v, s_warp, &tot);
		if (b < n_bins) { pack0[b] = carry + ex; sk += bin_recs[b]; km += bin_kmers[b]; }
		carry += tot;
	}
	uint64_t tsk, tkm;
	split_block_excl<0>(sk, s_warp, &tsk);
	split_block_excl<0>(km, s_warp, &tkm);
	if (threadIdx.x == 0) {
		const uint64_t bytes = n_rt ? state[kStBytes] : 0;
		const uint64_t err = bytes > out_capacity || carry > pack_capacity;
		state[kStBytes] = bytes; state[kStPacks] = carry; state[kStCapErr] = err; state[kStSuperKmers] = tsk; state[kStKmers] = tkm;
		s_tot[0] = err;
		if (result) { result[0] = bytes; result[1] = carry; result[2] = err; result[3] = tsk; result[4] = tkm; }
	}
	__syncthreads();
	if (s_tot[0] || !frags) return;
	for (uint32_t b = threadIdx.x; b < n_bins; b += blockDim.x) {
		kmcb200_bin_fragment f;
		f.byte_off = n_rt ? hist[(uint64_t)b * n_rt] : 0;
		f.bytes = (n_rt ? split_bin_base(hist, n_rt, b + 1, n_bins, state) : 0) - f.byte_off;
		f.n_rec = bin_kmers[b];
		f.n_super_kmers = bin_recs[b];
		f.pack0 = (uint32_t)pack0[b];
		f.n_packs = (uint32_t)bin_packs[b];
		frags[b] = f;
	}
}

// pack j of the batch: its bin by binary search over pack0, its length from the next pack start (or the bin's end)
__global__ void __launch_bounds__(kSplitThreads) split_pack_bytes_kernel(const uint64_t* __restrict__ hist, const uint64_t* __restrict__ pack0,
	const uint64_t* __restrict__ bin_packs, const uint64_t* __restrict__ pack_start, uint32_t n_bins, const uint64_t* __restrict__ state,
	uint64_t* __restrict__ pack_bytes)
{
	if (state[kStCapErr]) return;
	const uint64_t n_packs = state[kStPacks];
	const uint64_t n_rt = (state[kStRecords] + kSplitRecTile - 1) / kSplitRecTile;
	for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_packs; j += (uint64_t)gridDim.x * blockDim.x) {
		uint32_t lo = 0, hi = n_bins;                                   // first bin with pack0 > j
		while (lo < hi) { const uint32_t mid = (lo + hi) / 2; if (pack0[mid] <= j) lo = mid + 1; else hi = mid; }
		const uint32_t b = lo - 1;
		const uint64_t p = j - pack0[b];
		const uint64_t base = split_bin_base(hist, n_rt, b, n_bins, state);
		const uint64_t slot = base / kSplitPackWindow + b;
		const uint64_t end = p + 1 < bin_packs[b] ? pack_start[slot + p + 1] : split_bin_base(hist, n_rt, b + 1, n_bins, state) - base;
		pack_bytes[j] = end - pack_start[slot + p];
	}
}

// one thread per record: the length byte and the packed symbols at rec_dst
__global__ void __launch_bounds__(kSplitThreads) split_emit_kernel(const uint8_t* __restrict__ seq, const uint32_t* __restrict__ rec_start,
	const uint32_t* __restrict__ rec_end, const uint64_t* __restrict__ rec_dst, uint32_t k, const uint64_t* __restrict__ state, uint8_t* __restrict__ out)
{
	if (state[kStCapErr]) return;
	const uint64_t n_rec = state[kStRecords];
	for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rec; r += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t s = rec_start[r];
		const uint32_t n = rec_end[r] - s + k;
		uint8_t* o = out + rec_dst[r];
		o[0] = (uint8_t)(n - k);
		const uint8_t* p = seq + s;
		for (uint32_t i = 0; i < n; i += 4) {
			uint32_t v = 0;
#pragma unroll
			for (uint32_t q = 0; q < 4; ++q) v = (v << 2) | (i + q < n ? (split_code(p[i + q]) & 3u) : 0u);
			o[1 + i / 4] = (uint8_t)v;
		}
	}
}

}  // namespace kmcb
