// kmc_b200 — device-side helpers shared by the stage-2 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace kmcb {

constexpr int kMaxWords = 4;            // records of up to 4 x 64 bit  (k <= 128)

// ---------------------------------------------------------------------------------------------
// A k-mer record: the byte image is identical to the reference's CKmer<SIZE> (kmc_core/kmer.h:22-67):
// uint64 data[SIZE], data[0] least significant, compared from data[SIZE-1] down.
template <int WORDS>
struct __align__(8) Rec {
	uint64_t w[WORDS];
};

template <int WORDS>
__device__ __forceinline__ bool rec_equal(const Rec<WORDS>& a, const Rec<WORDS>& b)
{
	bool e = true;
#pragma unroll
	for (int i = 0; i < WORDS; ++i) e = e && (a.w[i] == b.w[i]);
	return e;
}

template <int WORDS>
__device__ __forceinline__ bool rec_less(const Rec<WORDS>& a, const Rec<WORDS>& b)
{
	// most significant word first (kmer.h:271-278)
	bool lt = false, decided = false;
#pragma unroll
	for (int i = WORDS - 1; i >= 0; --i) {
		if (!decided && a.w[i] != b.w[i]) { lt = a.w[i] < b.w[i]; decided = true; }
	}
	return lt;
}

// byte `b` of the little-endian record image (kmer.h:242-245 get_byte)
template <int WORDS>
__device__ __forceinline__ uint32_t rec_byte(const Rec<WORDS>& r, uint32_t b)
{
	uint64_t x = r.w[0];
	if (WORDS > 1) {
		const uint32_t wi = b >> 3;
#pragma unroll
		for (int i = 1; i < WORDS; ++i) if (wi == (uint32_t)i) x = r.w[i];
	}
	return (uint32_t)(x >> ((b & 7u) * 8u)) & 0xFFu;
}

// ---------------------------------------------------------------------------------------------
// PTX wrappers: mbarrier + TMA 1-D bulk copy (cp.async.bulk, SASS UBLKCP) + relaxed gpu-scope ld/st
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity)
{
	uint32_t ok;
	asm volatile(
		"{\n\t.reg .pred p;\n\t"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
		"selp.u32 %0, 1, 0, p;\n\t}"
		: "=r"(ok)
		: "r"(smem_u32(bar)), "r"(parity)
		: "memory");
	return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
	while (!mbar_try_wait(bar, parity)) {}
}
// global -> shared bulk copy; dst, src and bytes must be multiples of 16
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
		"l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
		: "memory");
}

__device__ __forceinline__ uint32_t ld_relaxed(const uint32_t* p)
{
	uint32_t v;
	asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}
__device__ __forceinline__ uint64_t ld_relaxed(const uint64_t* p)
{
	uint64_t v;
	asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
	return v;
}
__device__ __forceinline__ void st_relaxed(uint32_t* p, uint32_t v) { asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_relaxed(uint64_t* p, uint64_t v) { asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }
__device__ __forceinline__ uint32_t lanemask_lt()
{
	uint32_t m;
	asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
	return m;
}

// ---------------------------------------------------------------------------------------------
// Decoupled look-back descriptors (64 bit): [63:62] state, [61:40] epoch, [39:0] value.
// The epoch makes descriptors of earlier launches read as "not ready", so the array is zeroed once at
// allocation and never again between passes/bins (the host bumps the epoch per launch).
constexpr uint64_t kDescAggregate = 1, kDescPrefix = 2;
constexpr int kDescStateShift = 62, kDescEpochShift = 40;
constexpr uint64_t kDescValueMask = (1ull << 40) - 1, kDescEpochMask = (1ull << 22) - 1;

__device__ __forceinline__ uint64_t desc_pack(uint64_t state, uint32_t epoch, uint64_t value)
{
	return (state << kDescStateShift) | ((uint64_t)epoch << kDescEpochShift) | value;
}
// state of a descriptor as seen by a launch with the given epoch (0 = not ready)
__device__ __forceinline__ uint32_t desc_state(uint64_t v, uint32_t epoch)
{
	return (((v >> kDescEpochShift) & kDescEpochMask) == epoch) ? (uint32_t)(v >> kDescStateShift) : 0u;
}

// Publishes this tile's aggregate for one chain and returns the exclusive prefix over all earlier tiles.
// desc points at this chain's slot of tile 0; consecutive tiles are `stride` slots apart.
__device__ __forceinline__ uint64_t lookback_exclusive(uint64_t* desc, uint64_t stride, uint32_t tile, uint64_t aggregate, uint32_t epoch)
{
	if (tile == 0) {
		st_relaxed(desc, desc_pack(kDescPrefix, epoch, aggregate));
		return 0;
	}
	st_relaxed(desc + (uint64_t)tile * stride, desc_pack(kDescAggregate, epoch, aggregate));
	uint64_t excl = 0;
	for (int64_t t = (int64_t)tile - 1;; --t) {
		uint64_t v;
		uint32_t st;
		do {
			v = ld_relaxed(desc + (uint64_t)t * stride);
			st = desc_state(v, epoch);
		} while (st == 0);
		excl += v & kDescValueMask;
		if (st == kDescPrefix) break;
	}
	st_relaxed(desc + (uint64_t)tile * stride, desc_pack(kDescPrefix, epoch, excl + aggregate));
	return excl;
}


// Second half of the chained scan when the aggregate has already been published (radix passes publish it early):
// returns the exclusive prefix over all earlier tiles and upgrades this tile's descriptor to an inclusive prefix.
__device__ __forceinline__ uint64_t lookback_resolve(uint64_t* desc, uint64_t stride, uint32_t tile, uint64_t aggregate, uint32_t epoch)
{
	uint64_t excl = 0;
	for (int64_t t = (int64_t)tile - 1;; --t) {
		uint64_t v;
		uint32_t st;
		do {
			v = ld_relaxed(desc + (uint64_t)t * stride);
			st = desc_state(v, epoch);
		} while (st == 0);
		excl += v & kDescValueMask;
		if (st == kDescPrefix) break;
	}
	st_relaxed(desc + (uint64_t)tile * stride, desc_pack(kDescPrefix, epoch, excl + aggregate));
	return excl;
}

}  // namespace kmcb
