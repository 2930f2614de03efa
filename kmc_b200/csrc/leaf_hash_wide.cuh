// kmc_b200 — leaves of WIDER records (k > 32: 2..4 words), the design of leaf_hash.cuh: one hash table over the whole leaf, probes that miss
// are deferred into a queue and drained by straight-line code, rounds read the leaf with a predicate, the order is restored at the emission
// by virtual groups.  (The job of CompactKmers / CompactKxmers + kxmer_set.h, kmc_core/kb_sorter.h:937-1281,
// fused with the lower levels of the sort.)
//
// What differs from the one-word kernel: a k-mer does not fit into a table entry, so the entry holds
//     [ index of the first copy inside the leaf (16) | hash tag (16) | count (32) ]          EMPTY = all ones
// and "is this my k-mer?" is answered by the tag first and, when the tags agree, by comparing with that first copy (a global load that hits
// L2: the leaf was just streamed).  A queue item is [ probes done (16) | index of the record (16) | its 32-bit hash ]: a deferred probe
// reloads its record only if it meets an entry with its tag.
#pragma once
#include "leaf_hash.cuh"

namespace kmcb {

template <int SLOT_BITS>
struct LhwRound {
	uint32_t s_main, s_surv, s_over, s_dummy;
	uint64_t* queue;
	uint32_t cmin, cmax1;
	bool never, has_max;
};

template <int WORDS>
__device__ __forceinline__ uint32_t lhw_hash(const Rec<WORDS>& r)
{
	uint64_t x = r.w[0];
#pragma unroll
	for (int i = 1; i < WORDS; ++i) x = (x ^ (x >> 29)) * 0xBF58476D1CE4E5B9ull + r.w[i];
	x = (x ^ (x >> 31)) * 0x9E3779B97F4A7C15ull;
	return (uint32_t)(x >> 32);
}

// one probe of the k-mer `key` (record j of the leaf, hash h) at `slot`; returns true when the slot belongs to another k-mer
template <int WORDS, int SLOT_BITS, bool SIMPLE>
__device__ __forceinline__ bool lhw_probe(const LhwRound<SLOT_BITS>& t, bool act, const Rec<WORDS>& key, uint32_t j, uint32_t h, uint32_t slot,
	const Rec<WORDS>* __restrict__ g, uint32_t& r_claim, uint32_t& r_max)
{
	const uint32_t tag = h & 0xFFFFu;
	const uint32_t saddr = t.s_main + slot * 8u;
	unsigned long long cur;
	asm volatile("ld.shared.u64 %0, [%1];" : "=l"(cur) : "r"(saddr) : "memory");
	const bool was_empty = cur == kLwEmpty;
	const unsigned long long mine = ((unsigned long long)j << 48) | ((unsigned long long)tag << 32) | 1ull;          // j <= 65533: never the EMPTY pattern
	const unsigned long long got = lh_cas64(act && was_empty, saddr, t.s_dummy, mine);
	const unsigned long long eff = was_empty ? got : cur;          // (a slot that was EMPTY may have been taken in between: then the CAS returns its owner)
	const bool claimed = act && was_empty && got == kLwEmpty;
	bool same = false;
	if (act && !claimed && ((uint32_t)(eff >> 32) & 0xFFFFu) == tag) same = rec_equal<WORDS>(lw_load<WORDS>(g + (uint32_t)(eff >> 48)), key);
	const uint32_t newc = lh_add32(same, saddr) + 1u;          // low word = count
	r_claim += claimed ? 1u : 0u;
	const uint32_t bit = 1u << (slot & 31u), woff = (slot >> 5) * 4u;
	if (SIMPLE) {
		lh_or32(same && newc == t.cmin, t.s_surv + woff, bit);
	} else {
		const bool at_min = (same && newc == t.cmin) || (claimed && t.cmin == 1u);
		if (t.never) r_max += at_min ? 1u : 0u;
		else lh_or32(at_min, t.s_surv + woff, bit);
		if (t.has_max) {
			const bool at_max = !t.never && ((same && newc == t.cmax1) || (claimed && t.cmax1 == 1u));
			lh_or32(at_max, t.s_over + woff, bit);
			r_max += at_max ? 1u : 0u;
		}
	}
	return act && !claimed && !same;
}

template <int WORDS, int SLOT_BITS, bool SIMPLE>
__global__ void __launch_bounds__(32 * kLwWarps, KMCB200_LH_MINBLOCKS) leaf_hash_wide_kernel(const LeafArgs a)
{
	using R = Rec<WORDS>;
	using SM = LhSmem<SLOT_BITS>;
	constexpr int SLOTS = SM::kSlots;
	constexpr int NW = SLOTS / 32;
	constexpr uint32_t FULL = 0xffffffffu;
	constexpr uint32_t SM1 = (uint32_t)SLOTS - 1u;
	constexpr int V = 2;                                 // records per lane and step
	static_assert(WORDS >= 2 && NW <= 32 && NW >= 4, "");
	extern __shared__ __align__(16) uint8_t lhw_dsm[];
	SM& S = reinterpret_cast<SM*>(lhw_dsm)[threadIdx.x >> 5];
	if (*a.flags & kMsdFlagStop) return;
	const uint32_t lane = threadIdx.x & 31u, lt = lanemask_lt();
	S.dummy[lane] = 0ull;
	__syncwarp();
	const uint32_t CAP = max((uint32_t)SLOTS * a.fill_pct / 100u, 32u);
	const uint32_t LIMIT = (uint32_t)SLOTS - (uint32_t)SLOTS / 8u;
	const R* __restrict__ recs = reinterpret_cast<const R*>(a.recs);
	const uint32_t ob = a.suffix_bytes + a.counter_bytes;
	const uint32_t padw = (ob + 7) >> 3;
	const uint32_t prefix_shift = 2u * (a.k - a.lut_prefix_len);
	const bool one_prefix = prefix_shift >= a.low_bits;
	const LwCut cut{a.cutoff_min > 1u ? a.cutoff_min : 1u, a.cutoff_max + 1u, a.cutoff_max < (a.cutoff_min > 1u ? a.cutoff_min : 1u)};
	uint64_t* const tmp64 = reinterpret_cast<uint64_t*>(a.tmp);
	uint16_t* const list = S.list();
	uint32_t t_unique = 0, t_max = 0, t_emit = 0;
	uint32_t ratio_q8 = min(max(a.ratio0_q8, 8u), 256u);
	bool failed = false;

	uint32_t work = 0;
	if (lane == 0) work = atomicAdd(a.ticket, 1u);
	work = __shfl_sync(FULL, work, 0);
	while (work < a.n_leaves) {
		uint32_t next_t = 0;
		if (lane == 0) next_t = atomicAdd(a.ticket, 1u);
		const uint32_t leaf = work;
		const uint64_t lo = a.start[leaf];
		const uint32_t m = (uint32_t)min(a.start[leaf + 1] - lo, (uint64_t)0xffffffffu);
		uint32_t emit_base = 0;
		bool prefetched = false;
		if (m > kLwMaxLeaf) failed = true;          // (the entry's index field: the LSD fallback takes the bin)
		else if (m > 0) {
			const uint32_t round_recs = max(CAP * 256u / ratio_q8, 32u);
			uint32_t e0 = 0;
			while ((m >> e0) > round_recs && e0 < 8 && e0 < a.low_bits) ++e0;
			uint32_t e = e0, r = 0, leaf_claims = 0;
			const R* __restrict__ g = recs + lo;
			while (true) {
				// ================================================================ one round: the k-mers whose next e bits are r
				const uint32_t sub_shift = a.low_bits - e;
				const uint32_t emask = (1u << e) - 1u;
				{
					const uint4 ev = make_uint4(~0u, ~0u, ~0u, ~0u), zv = make_uint4(0, 0, 0, 0);
#pragma unroll
					for (int i = 0; i < SLOTS * 8 / 16 / 32; ++i) reinterpret_cast<uint4*>(S.main)[i * 32 + lane] = ev;
					if (lane < 2 * NW / 4) reinterpret_cast<uint4*>(S.surv)[lane] = zv;
				}
				__syncwarp();
				const LhwRound<SLOT_BITS> T{smem_u32(S.main), smem_u32(S.surv), smem_u32(S.over), smem_u32(&S.dummy[lane]), S.queue,
					cut.cmin, cut.cmax1, cut.never, cut.cmax1 != 0u && cut.cmax1 <= kLwMaxLeaf + 1u};
				uint32_t r_claim = 0, r_max = 0, head = 0, tail = 0;
				bool ok = true;
				// ---- insertion: V records per lane and step; misses are queued as [probes | record | hash]
				for (uint32_t j0 = 0; j0 < m; j0 += V * 32) {
					R key[V];
					uint32_t h[V];
					bool act[V];
#pragma unroll
					for (int u = 0; u < V; ++u) {
						const uint32_t j = j0 + u * 32 + lane;
						act[u] = j < m;
						if (act[u]) key[u] = lw_load<WORDS>(g + j);
						else {
#pragma unroll
							for (int i = 0; i < WORDS; ++i) key[u].w[i] = 0;
						}
						if (e && rec_bits<WORDS>(key[u], sub_shift, emask) != r) act[u] = false;          // another round's k-mer
						h[u] = lhw_hash<WORDS>(key[u]);
					}
#pragma unroll
					for (int u = 0; u < V; ++u) {
						const uint32_t j = j0 + u * 32 + lane;
						const bool miss = lhw_probe<WORDS, SLOT_BITS, SIMPLE>(T, act[u], key[u], j, h[u], h[u] >> (32 - SLOT_BITS), g, r_claim, r_max);
						const uint32_t bal = __ballot_sync(FULL, miss);
						if (miss) S.queue[(tail + __popc(bal & lt)) & (kLhQueue - 1)] = (1ull << 48) | ((uint64_t)j << 32) | h[u];
						tail += __popc(bal);
					}
					if (__reduce_add_sync(FULL, r_claim) > LIMIT) ok = false;          // (a table that fills up must end the round here)
					while (ok && tail - head >= 32u) {
						__syncwarp();
						const bool pend = true;
						const uint64_t item = S.queue[(head + lane) & (kLhQueue - 1)];
						head += 32u;
						const uint32_t hh = (uint32_t)item, jj = (uint32_t)(item >> 32) & 0xFFFFu, pc = (uint32_t)(item >> 48);
						const R kk = lw_load<WORDS>(g + jj);
						const bool miss = lhw_probe<WORDS, SLOT_BITS, SIMPLE>(T, pend, kk, jj, hh, ((hh >> (32 - SLOT_BITS)) + pc) & SM1, g, r_claim, r_max);
						const uint32_t bal = __ballot_sync(FULL, miss);
						if (miss) S.queue[(tail + __popc(bal & lt)) & (kLhQueue - 1)] = ((uint64_t)(pc + 1u) << 48) | (item & 0x0000FFFFFFFFFFFFull);
						tail += __popc(bal);
						if (__reduce_add_sync(FULL, r_claim) > LIMIT) ok = false;
					}
					if (!ok) break;
				}
				// what is left in the queue: every lane follows one probe to its slot
				while (ok && tail != head) {
					__syncwarp();
					const uint32_t take = min(tail - head, 32u);
					bool pend = lane < take;
					const uint64_t item = pend ? S.queue[(head + lane) & (kLhQueue - 1)] : 0ull;
					head += take;
					const uint32_t hh = (uint32_t)item, jj = (uint32_t)(item >> 32) & 0xFFFFu;
					R kk;
					if (pend) kk = lw_load<WORDS>(g + jj);
					else {
#pragma unroll
						for (int i = 0; i < WORDS; ++i) kk.w[i] = 0;
					}
					uint32_t slot = ((hh >> (32 - SLOT_BITS)) + (uint32_t)(item >> 48)) & SM1;
					while (true) {
						pend = lhw_probe<WORDS, SLOT_BITS, SIMPLE>(T, pend, kk, jj, hh, slot, g, r_claim, r_max);
						slot = (slot + 1u) & SM1;
						if (__reduce_add_sync(FULL, r_claim) > LIMIT) { ok = false; break; }
						if (!__any_sync(FULL, pend)) break;
					}
				}
				if (!prefetched) {
					prefetched = true;
					const uint32_t nl = __shfl_sync(FULL, next_t, 0);
					if (nl < a.n_leaves) {
						const uint64_t nlo = a.start[nl];
						const uint32_t nm = (uint32_t)min(a.start[nl + 1] - nlo, (uint64_t)kLwMaxLeaf);
						for (uint32_t i = lane * (128 / (8 * WORDS)); i < nm; i += 32 * (128 / (8 * WORDS))) asm volatile("prefetch.global.L2 [%0];" ::"l"(recs + nlo + i));
					}
				}
				__syncwarp();
				if (!ok) {
					if (e < a.low_bits && e < e0 + kLwMaxSplit) { ++e; r <<= 1; continue; }
					failed = true;
					break;
				}
				t_unique += r_claim;
				t_max += r_max;
				leaf_claims += r_claim;
				// ---- reached & ~over is the result; the k-mer of an entry is its first copy
				const uint32_t w_main = lane < (uint32_t)NW ? (S.surv[lane] & ~S.over[lane]) : 0u;
				const uint32_t n_main = __reduce_add_sync(FULL, (uint32_t)__popc(w_main));
				if (n_main) {
					const uint32_t vbits = min(sub_shift, kLhVgBits);          // virtual group = the top 6 bits below the round's prefix
					const uint32_t vshift = sub_shift - vbits, vmask = (1u << vbits) - 1u;
					auto key_of = [&](uint32_t s) -> R { return lw_load<WORDS>(g + (uint32_t)(S.main[s] >> 48)); };
					__syncwarp();
					S.vcur[lane] = 0; S.vcur[lane + 32] = 0;
					__syncwarp();
					for (uint32_t w = w_main; w; w &= w - 1) {
						const uint32_t s = lane * 32 + (uint32_t)(__ffs(w) - 1);
						atomicAdd(&S.vcur[rec_bits<WORDS>(key_of(s), vshift, vmask)], 1u);
					}
					__syncwarp();
					{
						const uint32_t c0 = S.vcur[2 * lane], c1 = S.vcur[2 * lane + 1];
						uint32_t inc = c0 + c1;
#pragma unroll
						for (int o = 1; o < 32; o <<= 1) {
							const uint32_t x = __shfl_up_sync(FULL, inc, o);
							if (lane >= (uint32_t)o) inc += x;
						}
						const uint32_t ex = inc - c0 - c1;
						__syncwarp();
						S.vbase[2 * lane] = ex; S.vbase[2 * lane + 1] = ex + c0;
						S.vcur[2 * lane] = ex; S.vcur[2 * lane + 1] = ex + c0;
						if (lane == 31) S.vbase[kLhVg] = inc;
					}
					__syncwarp();
					for (uint32_t w = w_main; w; w &= w - 1) {
						const uint32_t s = lane * 32 + (uint32_t)(__ffs(w) - 1);
						list[atomicAdd(&S.vcur[rec_bits<WORDS>(key_of(s), vshift, vmask)], 1u)] = (uint16_t)s;
					}
					__syncwarp();
					for (uint32_t q = lane; q < n_main; q += 32) {
						const uint32_t s = list[q];
						const uint64_t ent = S.main[s];
						const R kk = lw_load<WORDS>(g + (uint32_t)(ent >> 48));
						const uint32_t vg = rec_bits<WORDS>(kk, vshift, vmask);
						const uint32_t q_lo = S.vbase[vg], q_hi = S.vbase[vg + 1];
						uint32_t pos = q_lo;
						for (uint32_t j = q_lo; j < q_hi; ++j) pos += rec_less<WORDS>(key_of(list[j]), kk) ? 1u : 0u;
						const uint32_t c = (uint32_t)ent;
						const uint32_t value = c > a.counter_max ? a.counter_max : c;          // kb_sorter.h:1190
						uint64_t* dst = tmp64 + (lo + emit_base + pos) * padw;
						for (uint32_t w = 0; w < padw; ++w) dst[w] = lw_out_word<WORDS>(kk, value, a.suffix_bytes, w);
						if (!one_prefix) atomicAdd(reinterpret_cast<unsigned long long*>(a.lut) + rec_prefix<WORDS>(kk, prefix_shift), 1ull);     // kb_sorter.h:1203
					}
					emit_base += n_main;
				}
				__syncwarp();
				while (e > e0 && (r & 1u)) { r >>= 1; --e; }
				++r;
				if (e == e0 && r == (1u << e0)) break;
			}
			if (!failed && m >= 256u) {
				const uint32_t q8 = min(max(__reduce_add_sync(FULL, leaf_claims) * 256u / m, 8u), 256u);
				ratio_q8 = (ratio_q8 + q8 + 1u) >> 1;
			}
		}
		if (lane == 0) {
			a.leaf_emit[leaf] = failed ? 0u : emit_base;
			if (emit_base && !failed) atomicAdd(&a.group_sum[leaf >> 10], emit_base);
			t_emit += emit_base;
			if (one_prefix && emit_base && !failed)
				atomicAdd(reinterpret_cast<unsigned long long*>(a.lut) + ((a.leaf_prefix | leaf) >> (prefix_shift - a.low_bits)), (unsigned long long)emit_base);
		}
		if (failed) break;
		work = __shfl_sync(FULL, next_t, 0);
	}
	failed = __any_sync(FULL, failed);
	if (failed) { if (lane == 0) atomicOr(a.flags, kMsdFlagFallback); return; }
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		t_unique += __shfl_down_sync(FULL, t_unique, o);
		t_max += __shfl_down_sync(FULL, t_max, o);
	}
	if (lane == 0) {
		if (t_unique) atomicAdd(reinterpret_cast<unsigned long long*>(a.result), (unsigned long long)t_unique);
		if (t_unique - t_emit - t_max) atomicAdd(reinterpret_cast<unsigned long long*>(a.result) + 1, (unsigned long long)(t_unique - t_emit - t_max));
		if (t_max) atomicAdd(reinterpret_cast<unsigned long long*>(a.result) + 2, (unsigned long long)t_max);
	}
}

}  // namespace kmcb
