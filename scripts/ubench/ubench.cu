// Micro-benchmarks of the primitives the radix kernels lean on: shared atomics, match.any, ballots, shuffles.
// Each test runs ITER dependent-free repetitions per warp on all SMs and reports cycles per warp-instruction per SM-subpartition.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int ITER = 4096;

__device__ __forceinline__ uint32_t lcg(uint32_t& s) { s = s * 1664525u + 1013904223u; return s; }

template <int MODE>
__global__ void k(uint32_t* out, int unused)
{
	__shared__ uint32_t sh[8 * 256];
	for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) sh[i] = 0;
	__syncthreads();
	uint32_t s = threadIdx.x * 2654435761u + blockIdx.x * 40503u + 1;
	uint32_t acc = 0;
	const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	long long t0 = clock64();
#pragma unroll 4
	for (int i = 0; i < ITER; ++i) {
		uint32_t d = (lcg(s) >> 13) & 255u;           // random digit
		if (MODE == 0) acc += d;                                                     // baseline (lcg only)
		if (MODE == 1) atomicAdd(&sh[d], 1u);                                        // CTA-shared histogram, no return
		if (MODE == 2) acc += atomicAdd(&sh[d], 1u);                                 // with return
		if (MODE == 3) atomicAdd(&sh[(warp & 7) * 256 + d], 1u);                     // warp-private histogram
		if (MODE == 4) acc += __match_any_sync(0xffffffffu, d);                      // match.any on 8-bit value
		if (MODE == 5) { uint32_t m = 0xffffffffu;                                   // 8 ballots
#pragma unroll
			for (int b = 0; b < 8; ++b) { uint32_t v = __ballot_sync(0xffffffffu, (d >> b) & 1); m &= ((d >> b) & 1) ? v : ~v; }
			acc += m; }
		if (MODE == 6) acc += __shfl_sync(0xffffffffu, d, (lane + 1) & 31);          // shuffle
		if (MODE == 7) { uint32_t dd = d & 3u; atomicAdd(&sh[dd], 1u); }             // 4 distinct addresses (heavy same-address)
		if (MODE == 8) { uint32_t m = __match_any_sync(0xffffffffu, d); if ((int)lane == __ffs(m) - 1) sh[(warp & 7) * 256 + d] += __popc(m); __syncwarp(); }   // match + leader RMW
		if (MODE == 9) { sh[(warp & 7) * 256 + ((d + lane) & 255)] += 1; }            // plain LDS+STS RMW (conflict-free-ish)
		if (MODE == 10) acc += __popc(__ballot_sync(0xffffffffu, d & 1));            // single ballot
		if (MODE == 11) { uint32_t dd = (d & 0xF0u) | (lane & 15u); atomicAdd(&sh[dd], 1u); }  // 2 lanes per address
		if (MODE == 12) { atomicAdd(&sh[lane * 8 + (d & 7)], 1u); }                  // conflict-free banks, distinct addresses
		if (MODE == 13) { unsigned long long* p = reinterpret_cast<unsigned long long*>(sh) + ((d * 3 + lane) & 1023); acc += (uint32_t)atomicCAS(p, 0xFFFFFFFFFFFFFFFFull, (unsigned long long)d); }   // CAS.64 random
		if (MODE == 14) { acc += atomicCAS(&sh[(d * 3 + lane) & 2047], 0xFFFFFFFFu, d); }                              // CAS.32 random
		if (MODE == 15) { unsigned long long* p = reinterpret_cast<unsigned long long*>(sh) + ((d * 3 + lane) & 1023); acc += (uint32_t)atomicMin(p, (unsigned long long)d * 7919ull); }      // MIN.64
		if (MODE == 16) { unsigned long long* p = reinterpret_cast<unsigned long long*>(sh) + ((d * 3 + lane) & 1023); atomicAdd(p, 1ull); }      // ADD.64
		if (MODE == 17) { acc += atomicMin(&sh[(d * 3 + lane) & 2047], d * 7919u); }                                    // MIN.32
		if (MODE == 18) { acc += atomicExch(&sh[(d * 3 + lane) & 2047], d); }                                           // EXCH.32
		if (MODE == 20) { unsigned long long* p = reinterpret_cast<unsigned long long*>(sh) + ((acc + d) & 1023); acc += (uint32_t)atomicCAS(p, 0xFFFFFFFFFFFFFFFFull, (unsigned long long)d); }   // CAS.64, address depends on the previous result: latency
		if (MODE == 21) { const unsigned long long* p = reinterpret_cast<const unsigned long long*>(sh) + ((acc + d) & 1023); acc += (uint32_t)*reinterpret_cast<const volatile unsigned long long*>(p); }   // LDS.64 dependent chain
		if (MODE == 22) { acc += atomicAdd(&sh[(acc + d) & 2047], 1u); }                                                // ADD.32 with return, dependent chain
		if (MODE == 23) { unsigned long long* p = reinterpret_cast<unsigned long long*>(sh) + ((d * 3 + lane) & 1023); const unsigned long long v = *reinterpret_cast<volatile unsigned long long*>(p); if ((uint32_t)v != 12345u) atomicAdd(reinterpret_cast<uint32_t*>(p), 1u); }   // LDS.64 + ADD.32 (the 'copy of a known k-mer' path without CAS)
		if (MODE == 19) { unsigned long long* p = reinterpret_cast<unsigned long long*>(sh) + ((d * 3 + lane) & 1023); acc += (uint32_t)atomicExch(p, (unsigned long long)d); }  // EXCH.64
	}
	long long t1 = clock64();
	if (threadIdx.x == 0) out[blockIdx.x * 2] = (uint32_t)(t1 - t0);
	out[blockIdx.x * 2 + 1] = acc + sh[threadIdx.x & 255];
}

template <int MODE>
void run(const char* name, int threads, int blocks_per_sm)
{
	int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
	uint32_t* out; cudaMalloc(&out, sms * blocks_per_sm * 8);
	k<MODE><<<sms * blocks_per_sm, threads>>>(out, 0);
	cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
	cudaEventRecord(a);
	k<MODE><<<sms * blocks_per_sm, threads>>>(out, 0);
	cudaEventRecord(b); cudaEventSynchronize(b);
	float ms; cudaEventElapsedTime(&ms, a, b);
	uint32_t h[2]; cudaMemcpy(h, out, 8, cudaMemcpyDeviceToHost);
	const double warps_per_sm = threads / 32.0 * blocks_per_sm;
	const double cyc = h[0];
	printf("%-44s thr=%4d blk/SM=%d : %8.1f cycles/iter/warp, %6.2f cycles per warp-instr per SM (all warps), kernel %.3f ms\n", name, threads, blocks_per_sm,
		cyc / ITER, cyc / ITER / warps_per_sm, ms);
	cudaFree(out);
}

int main()
{
	for (int cfg = 0; cfg < 1; ++cfg) {
		const int thr = cfg == 0 ? 512 : 1024, bps = cfg == 0 ? 2 : 2;
		run<0>("baseline lcg", thr, bps);
		run<1>("atomicAdd smem CTA-shared random (no ret)", thr, bps);
		run<2>("atomicAdd smem CTA-shared random (ret)", thr, bps);
		run<3>("atomicAdd smem warp-private random", thr, bps);
		run<12>("atomicAdd smem conflict-free distinct", thr, bps);
		run<11>("atomicAdd smem 2 lanes/address", thr, bps);
		run<7>("atomicAdd smem 4 addresses", thr, bps);
		run<4>("match.any 8-bit", thr, bps);
		run<5>("8 ballots emulating match", thr, bps);
		run<10>("single ballot + popc", thr, bps);
		run<6>("shfl", thr, bps);
		run<13>("atomicCAS 64 smem random", thr, bps);
		run<14>("atomicCAS 32 smem random", thr, bps);
		run<15>("atomicMin 64 smem random", thr, bps);
		run<16>("atomicAdd 64 smem random", thr, bps);
		run<17>("atomicMin 32 smem random", thr, bps);
		run<18>("atomicExch 32 smem random", thr, bps);
		run<19>("atomicExch 64 smem random", thr, bps);
		run<23>("LDS.64 + atomicAdd 32 (no CAS)", thr, bps);
		run<20>("atomicCAS 64 dependent chain, 1 warp/SM", 32, 1);
		run<21>("LDS.64 dependent chain, 1 warp/SM", 32, 1);
		run<22>("atomicAdd 32 ret dependent chain, 1 warp/SM", 32, 1);
		run<0>("baseline lcg, 1 warp/SM", 32, 1);
		run<8>("match + leader LDS/STS RMW + syncwarp", thr, bps);
		run<9>("plain smem RMW (LDS+IADD+STS)", thr, bps);
	}
	return 0;
}
