// kmc_b200 — histogram estimation on the GPU: the ntHash sampling of KMC's CntHashEstimator (kmc_core/libs/ntHash/ntHashWrapper.h:97-454),
// which `kmc -e` and `kmc --opt-out-size` run over every sequence of the input.  Included by kmc_b200.cu.
//
// The batch format is kmcb200_split's: every byte other than ACGTacgt separates, so a k-mer is sampled exactly when its k bases are all
// ACGT.  Its hash is canonical ntHash, min(fh, rh), with R the split rotation (the high 31 bits and the low 33 bits each rotated left by
// one within themselves):
//     fh = XOR_i R^(k-1-i)(seed[c_i]),  rh = XOR_i R^i(seed[3 - c_i])
// A hash h is sampled into table 0 when h >> (63 - s) == 1 and into table 1 when h >> (64 - s) == 2^(s-1) - 1 (CntHashEstimator::try_insert,
// :306-316), each at counter h mod 2^27.
// Kernels:
//   estimate_hash_kernel   a tile of kEstTile k-mer end positions per CTA; thread j rolls the hash over positions 16 j .. 16 j + 15 of it,
//                          starting k - 1 bases before them (the same steps as the reference's Process), and adds 1 to the counter of a
//                          sampled hash with a u32 atomic (about 1.5 * 2^-s of the hashes)
//   estimate_hist_kernel   one pass over the 2 x 2^27 counters with 16-byte loads: the histograms of min(65536, c) of the two tables and
//                          the largest counter.  Zeros are counted in registers, values below kEstSharedBins in shared memory, and only the
//                          rare larger ones go to global atomics.
// The recursion that turns the two histograms into the estimate runs on the host (estimate.inl).
#pragma once
#include "split.cuh"

namespace kmcb {

constexpr uint32_t kEstMaxK = 256;
constexpr uint32_t kEstThreads = 256;
constexpr uint32_t kEstPer = 16;                                        // consecutive k-mer end positions per thread
constexpr uint32_t kEstTile = kEstThreads * kEstPer;
constexpr uint32_t kEstHalo = kEstMaxK - 1;
constexpr uint32_t kEstR = 27;                                          // log2 of the counters per table (CntHashEstimator's r)
constexpr uint64_t kEstTable = 1ull << kEstR;
constexpr uint32_t kEstMaxOcc = 65536;                                  // max_occ_value
constexpr uint32_t kEstHistLen = kEstMaxOcc + 1;                        // bins of one table's histogram
constexpr uint32_t kEstSharedBins = 2048;                               // counter values the histogram kernel bins in shared memory

// the four ntHash seeds of A, C, G, T (ntHash.hpp:189-192)
constexpr uint64_t kNtSeed[4] = {0x3c8bfbb395c60474ull, 0x3193c18562a02b4cull, 0x20323ed082572324ull, 0x295549f54be24456ull};

// R: rol1 then swapbits033 (ntHash.hpp:350-381)
__host__ __device__ __forceinline__ uint64_t nt_rot(uint64_t v)
{
	v = (v << 1) | (v >> 63);
	const uint64_t x = (v ^ (v >> 33)) & 1u;
	return v ^ (x | (x << 33));
}

// R^-1: ror1 then swapbits3263
__host__ __device__ __forceinline__ uint64_t nt_unrot(uint64_t v)
{
	v = (v >> 1) | (v << 63);
	const uint64_t x = ((v >> 32) ^ (v >> 63)) & 1u;
	return v ^ ((x << 32) | (x << 63));
}

// seed[c] and R^k(seed[c]), the two tables the rolling step reads (the reference's M_seedTab and P_msTab)
struct EstTabs {
	uint64_t seed[4];
	uint64_t rk[4];
};

// counters[t * 2^27 + (h mod 2^27)] += 1 for every sampled hash h of the batch (t = the table that samples it)
__global__ void __launch_bounds__(kEstThreads) estimate_hash_kernel(const uint8_t* __restrict__ seq, uint64_t len, uint32_t k, uint32_t s,
	EstTabs tabs, uint32_t* __restrict__ counters)
{
	__shared__ uint8_t s_code[kEstTile + kEstHalo + 1];
	__shared__ uint64_t s_seed[4], s_rk[4];
	const uint32_t tid = threadIdx.x;
	const uint64_t t0 = (uint64_t)blockIdx.x * kEstTile;
	if (tid == 0) {                                                     // constant indices: the parameters stay out of local memory
#pragma unroll
		for (uint32_t i = 0; i < 4; ++i) {
			s_seed[i] = tabs.seed[i];
			s_rk[i] = tabs.rk[i];
		}
	}
	// s_code[i] = code of base t0 - kEstHalo + i (4 outside the batch)
	for (uint32_t i = tid; i < kEstTile + kEstHalo; i += kEstThreads) {
		const int64_t b = (int64_t)t0 - (int64_t)kEstHalo + (int64_t)i;
		s_code[i] = (b >= 0 && (uint64_t)b < len) ? (uint8_t)split_code(seq[b]) : (uint8_t)4;
	}
	__syncthreads();
	const uint8_t* c = s_code + kEstHalo + tid * kEstPer - (k - 1);
	uint64_t fh = 0, rh = 0;
	uint32_t run = 0;                                                   // ACGT bases since the last separator
	// the k - 1 bases before the first end position: never a whole k-mer, so no outgoing base (M_NTC64_N)
	for (uint32_t j = 0; j + 1 < k; ++j) {
		const uint32_t b = c[j];
		if (b > 3) {
			fh = rh = 0;
			run = 0;
			continue;
		}
		fh = nt_rot(fh) ^ s_seed[b];
		rh = nt_unrot(rh ^ s_rk[3 - b]);
		++run;
	}
	const uint64_t first = t0 + (uint64_t)tid * kEstPer;
	const uint64_t top_mask = (1ull << (s - 1)) - 1;
#pragma unroll
	for (uint32_t e = 0; e < kEstPer; ++e) {
		const uint32_t b = c[k - 1 + e];
		if (b > 3) {
			fh = rh = 0;
			run = 0;
			continue;
		}
		if (run >= k) {                                                 // M_NTC64: base c[e - 1] leaves the window
			const uint32_t o = c[e - 1];
			fh = nt_rot(fh) ^ s_rk[o] ^ s_seed[b];
			rh = nt_unrot(rh ^ s_rk[3 - b] ^ s_seed[3 - o]);
		} else {
			fh = nt_rot(fh) ^ s_seed[b];
			rh = nt_unrot(rh ^ s_rk[3 - b]);
		}
		++run;
		if (run >= k && first + e < len) {
			const uint64_t h = rh < fh ? rh : fh;
			const uint64_t pref = h >> (63 - s);
			const uint32_t idx = (uint32_t)(h & (kEstTable - 1));
			if (pref == 1) atomicAdd(&counters[idx], 1u);
			if ((pref >> 1) == top_mask) atomicAdd(&counters[kEstTable + idx], 1u);
		}
	}
}

// blockIdx.y = table.  hist[table * kEstHistLen + min(65536, c)] += 1 for every counter c of the table; hist[2 * kEstHistLen] = max(c)
// over both tables.  hist must be zero before the launch.
__global__ void __launch_bounds__(kEstThreads) estimate_hist_kernel(const uint32_t* __restrict__ counters, uint32_t* __restrict__ hist)
{
	__shared__ uint32_t s_hist[kEstSharedBins];
	const uint32_t tid = threadIdx.x;
	const uint32_t table = blockIdx.y;
	const uint4* src = reinterpret_cast<const uint4*>(counters + table * kEstTable);
	uint32_t* out = hist + table * kEstHistLen;
	for (uint32_t i = tid; i < kEstSharedBins; i += kEstThreads) s_hist[i] = 0;
	__syncthreads();
	uint32_t zeros = 0, mx = 0;
	auto add = [&](uint32_t c) {
		if (c == 0) {
			++zeros;
			return;
		}
		mx = c > mx ? c : mx;
		if (c < kEstSharedBins) atomicAdd(&s_hist[c], 1u);
		else atomicAdd(&out[c < kEstMaxOcc ? c : kEstMaxOcc], 1u);
	};
	constexpr uint32_t n_vec = (uint32_t)(kEstTable / 4);
	for (uint32_t i = blockIdx.x * kEstThreads + tid; i < n_vec; i += gridDim.x * kEstThreads) {
		const uint4 v = __ldcs(src + i);
		add(v.x);
		add(v.y);
		add(v.z);
		add(v.w);
	}
	for (int o = 16; o; o >>= 1) {
		zeros += __shfl_xor_sync(0xffffffffu, zeros, o);
		const uint32_t m = __shfl_xor_sync(0xffffffffu, mx, o);
		mx = m > mx ? m : mx;
	}
	if ((tid & 31) == 0) {
		if (zeros) atomicAdd(&s_hist[0], zeros);
		if (mx) atomicMax(&hist[2 * kEstHistLen], mx);
	}
	__syncthreads();
	for (uint32_t i = tid; i < kEstSharedBins; i += kEstThreads)
		if (s_hist[i]) atomicAdd(&out[i], s_hist[i]);
}

}  // namespace kmcb
