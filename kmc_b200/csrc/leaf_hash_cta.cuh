// kmc_b200 — leaves of one-word records, third design: ONE HASH TABLE PER CTA, ONE LEAF PER CTA.
//
// Same job and interface as leaf_hash_kernel (leaf_hash.cuh: LeafArgs, the leaf's distinct k-mers in key order with their counts at
// tmp + (start[leaf] + position) * pad, leaf_emit, group_sum, LUT, the three statistics, the heavy-leaf list, the fallback flag), and the
// same insertion: the slot is a hash of all key bits below the round's prefix, a plain load before the CAS, probes that miss are deferred
// to a per-warp queue drained 64 at a time (lh_insert / lh_drain).  What changes is who owns the table:
//   * the NWARPS warps of a CTA share ONE table of 2^SLOT_BITS slots (4 warps x 1024 slots before, the same shared memory) and count ONE
//     leaf together, striding over its records.  A round is planned for ~62 % load, i.e. ~8 K records of a 30x bin in 4096 slots: nearly
//     every leaf of the workload (8 + 8 partition bits over bins of 2^25 .. 2^28 k-mers: means of 512 .. 4096 records, spread over 0 .. 2x)
//     is ONE round, every record is read and hashed once, with all lanes active - where a warp-owned 1024-slot table needed 2 .. 4
//     predicated rounds over the same leaf, each reading all of it;
//   * the claim count of a round is CTA-wide (shared memory: every warp adds what it claimed after each step); the warp whose addition
//     passes the limit raises the "full" flag, which ends the round for every warp at its next step, and the split on the next bit is
//     decided by all threads after a barrier.  The CAS / add protocol of the table is safe between warps as it is between lanes;
//   * the emission builds the survivor bitmap over the whole table, counts the survivors into 256 virtual groups (their next 8 key bits),
//     and ranks a survivor by comparison inside its group - every step spread over the CTA.
//
// Leaves beyond kLwHeavy records still go to the HEAVY launch of leaf_warp_kernel; leaf_scan / leaf_gather are unchanged.
#pragma once
#include "leaf_hash.cuh"

namespace kmcb {

constexpr uint32_t kLcVgBits = 8;                        // virtual groups of the emission: 2^8 (a few survivors each)
constexpr uint32_t kLcVg = 1u << kLcVgBits;
constexpr uint32_t kSmemPerSm = 228 * 1024, kSmemPerCta = 1024;      // sm_90: shared memory of an SM, and what the runtime reserves per CTA

template <int NWARPS, int SLOT_BITS>
struct LcSmem {
	static constexpr int kSlots = 1 << SLOT_BITS;
	uint64_t main[kSlots];                    // the table
	uint64_t queue[NWARPS][kLhQueue];         // deferred probes of each warp; during the emission: the u16 list of survivors, in group order
	uint32_t surv[kSlots / 32];               // entries whose count reached cutoff_min ...
	uint32_t over[kSlots / 32];               // ... whose count went past cutoff_max
	uint32_t vbase[kLcVg + 4];                // emission: first list position of every virtual group (+ end)
	uint32_t vcur[kLcVg];                     // emission: counters / cursors of the virtual groups
	uint64_t dummy[32];                       // one word per lane, always 0 (lh_cas64)
	uint32_t claims;                          // slots claimed in the round, over all warps
	uint32_t full;                            // the round's claims passed the limit: every warp stops inserting
	uint32_t failed;                          // the heavy-leaf list overflowed
	uint32_t stat_max;                        // n_cutoff_max of the CTA, summed at the end
	uint32_t ticket[2];                       // this leaf / the next one (alternating)
	__device__ __forceinline__ uint16_t* list() { return reinterpret_cast<uint16_t*>(&queue[0][0]); }       // [kSlots]
};

// CTAs per SM the kernel is compiled for: as many as shared memory allows, but no fewer than 96 registers per thread (the insertion's
// four probe chains and the drain's two need about that many; fewer spill)
template <int NWARPS, int SLOT_BITS>
constexpr int lc_min_blocks()
{
	constexpr int by_smem = (int)(kSmemPerSm / (sizeof(LcSmem<NWARPS, SLOT_BITS>) + kSmemPerCta));
	constexpr int by_regs = 65536 / (96 * 32 * NWARPS);
	return by_smem < by_regs ? by_smem : by_regs;
}

// round control of the CTA kernel: the claims since the warp's last step go into the CTA-wide count, and the round ends for every warp
// once one of them has seen that count pass the limit.  (Every claim is published before lh_insert returns: its loops end on a full().)
template <int NWARPS>
struct LcCtaCtl {
	static constexpr uint32_t kStride = 128 * NWARPS;    // the warps take turns at 128-record steps
	uint32_t* claims;
	volatile uint32_t* full_flag;
	uint32_t limit, lane;
	__device__ __forceinline__ bool full(uint32_t& r_claim) const
	{
		const uint32_t part = __reduce_add_sync(0xffffffffu, r_claim);
		r_claim = 0;
		uint32_t stop = 0;
		if (lane == 0) {
			if (part && atomicAdd(claims, part) + part > limit) *full_flag = 1u;
			stop = *full_flag;
		}
		return __shfl_sync(0xffffffffu, stop, 0) != 0u;
	}
};

template <int NWARPS, int SLOT_BITS, bool SIMPLE>
__global__ void __launch_bounds__(32 * NWARPS, lc_min_blocks<NWARPS, SLOT_BITS>()) leaf_hash_cta_kernel(const LeafArgs a)
{
	using R = Rec<1>;
	using SM = LcSmem<NWARPS, SLOT_BITS>;
	constexpr uint32_t SLOTS = SM::kSlots, NW = SLOTS / 32, NT = 32 * NWARPS;
	constexpr uint32_t FULL = 0xffffffffu;
	static_assert(NW % 4 == 0, "the bitmaps are cleared 16 bytes at a time");
	static_assert(NWARPS * kLhQueue * 8 >= SLOTS * 2, "the u16 list of survivors lives in the queues");
	static_assert(SLOTS <= 65536, "list entries and probe counts are 16 bits");
	static_assert(kLcVg == 8 * 32, "the scan of the virtual groups takes eight counters per lane");
	static_assert(kLhQueue >= 192 && (kLhQueue & (kLhQueue - 1)) == 0, "a step adds up to 128 deferred probes to up to 63 left over");
	extern __shared__ __align__(16) uint8_t lc_dsm[];
	SM& S = *reinterpret_cast<SM*>(lc_dsm);
	if (*a.flags & kMsdFlagStop) return;
	const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5, lt = lanemask_lt();
	if (tid < 32) S.dummy[tid] = 0ull;
	if (tid == 0) { S.stat_max = 0; S.failed = 0; S.ticket[0] = atomicAdd(a.ticket, 1u); }
	__syncthreads();
	const uint32_t CAP = max(SLOTS * a.fill_pct / 100u, 32u);                   // distinct k-mers a round is planned for
	const uint32_t LIMIT = SLOTS - SLOTS / 8u;                                   // ... and where it gives up (the table gets too crowded to probe)
	const unsigned long long* __restrict__ recs = reinterpret_cast<const unsigned long long*>(a.recs);
	const uint32_t ob = a.suffix_bytes + a.counter_bytes;
	const uint32_t padw = (ob + 7) >> 3;                                   // temporary records: padw 64-bit words
	const uint32_t prefix_shift = 2u * (a.k - a.lut_prefix_len);
	const bool one_prefix = prefix_shift >= a.low_bits;                    // every k-mer of a leaf has the same LUT prefix
	const LwCut cut{a.cutoff_min > 1u ? a.cutoff_min : 1u, a.cutoff_max + 1u, a.cutoff_max < (a.cutoff_min > 1u ? a.cutoff_min : 1u)};
	uint64_t* const tmp64 = reinterpret_cast<uint64_t*>(a.tmp);
	uint16_t* const list = S.list();
	uint32_t t_unique = 0, t_emit = 0;                    // thread 0; n_cutoff_min = unique - emitted - n_cutoff_max
	uint32_t t_max = 0;                                   // per thread
	uint32_t ratio_q8 = min(max(a.ratio0_q8, 8u), 256u);          // distinct k-mers per record (x 256): running estimate of this CTA
	bool failed = false;

	uint32_t par = 0;
	uint32_t work = S.ticket[0];
	while (work < a.n_leaves) {
		// (the other ticket word was last read before the previous leaf's closing barrier)
		if (tid == 0) S.ticket[par ^ 1u] = atomicAdd(a.ticket, 1u);        // the next leaf: in flight while this one is counted
		const uint32_t leaf = work;
		const uint64_t lo = a.start[leaf];
		const uint32_t m = (uint32_t)min(a.start[leaf + 1] - lo, (uint64_t)0xffffffffu);
		uint32_t emit_base = 0;
		if (m > kLwHeavy) {          // a large leaf: noted for the HEAVY launch of leaf_warp_kernel (its emitted count and LUT share are written there)
			if (tid == 0) {
				const uint32_t slot = atomicAdd(a.heavy_count, 1u);
				if (slot < a.heavy_cap) a.heavy_list[slot] = leaf;
				else S.failed = 1u;          // (more large leaves than the list holds: the LSD fallback takes the bin)
			}
		} else {
			if (m > 0) {
				bool prefetched = false;
				const uint32_t round_recs = max(CAP * 256u / ratio_q8, 32u);          // records of a round: their distinct k-mers should load the table to fill_pct
				uint32_t e0 = 0;
				while (((m >> e0) > round_recs && e0 < 8 && e0 < a.low_bits) || a.low_bits - e0 > kLhKeyBits) ++e0;      // (an entry holds <= 48 key bits)
				uint32_t e = e0, r = 0, leaf_claims = 0;
				const unsigned long long* __restrict__ g = recs + lo;
				while (true) {
					// ================================================================ one round: the k-mers whose next e bits are r
					const uint32_t kb = a.low_bits - e;                                    // key bits below the round's prefix (<= 48)
					const uint32_t cb = min(64u - kb, 32u);                                // bits of the count field (>= 16)
					const uint64_t rem_mask = (1ull << kb) - 1ull;
					const uint32_t cmask = cb >= 32 ? 0xffffffffu : ((1u << cb) - 1u);
					const uint32_t emask = (1u << e) - 1u;
					// ---- clear (the previous round is done with everything: barrier at its end)
					{
						const uint4 ev = make_uint4(~0u, ~0u, ~0u, ~0u), zv = make_uint4(0, 0, 0, 0);
						for (uint32_t i = tid; i < SLOTS / 2; i += NT) reinterpret_cast<uint4*>(S.main)[i] = ev;
						for (uint32_t i = tid; i < NW / 2; i += NT) reinterpret_cast<uint4*>(S.surv)[i] = zv;            // surv, over (contiguous)
						for (uint32_t i = tid; i < kLcVg; i += NT) S.vcur[i] = 0u;
						if (tid == 0) { S.claims = 0u; S.full = 0u; }
					}
					__syncthreads();
					// ---- insertion: warp w takes the 128-record steps w, w + NWARPS, ...
					const LhRound T{smem_u32(S.main), smem_u32(S.queue[warp]), smem_u32(S.surv), smem_u32(S.over), smem_u32(&S.dummy[lane]), S.queue[warp], cb, cmask,
						rem_mask, 1ull << cb, cut.cmin, cut.cmax1, cut.never, cut.cmax1 != 0u && cut.cmax1 <= kLwHeavy + 1u};
					const LcCtaCtl<NWARPS> ctl{&S.claims, &S.full, LIMIT, lane};
					uint32_t r_claim = 0, r_max = 0;
					if (e == 0) lh_insert<SLOT_BITS, SIMPLE, false>(T, ctl, g, warp * 128u, m, kb, emask, r, lane, lt, r_claim, r_max);
					else lh_insert<SLOT_BITS, SIMPLE, true>(T, ctl, g, warp * 128u, m, kb, emask, r, lane, lt, r_claim, r_max);
					if (!prefetched) {        // the next leaf: towards L2 while this one is counted
						prefetched = true;
						const uint32_t nl = S.ticket[par ^ 1u];          // (written before the clear's barrier)
						if (nl < a.n_leaves) {
							const uint64_t nlo = a.start[nl];
							const uint32_t nm = (uint32_t)min(a.start[nl + 1] - nlo, (uint64_t)kLwHeavy);
							for (uint32_t i = tid * 16; i < nm; i += NT * 16) asm volatile("prefetch.global.L2 [%0];" ::"l"(recs + nlo + i));
						}
					}
					__syncthreads();
					const bool ok = S.full == 0u;
					const uint32_t claims = S.claims;
					if (!ok) {        // this range does not fit: split it on the next bit (nothing of it has been emitted)
						__syncthreads();          // (everyone has read the flag before the next round clears it)
						if (e < a.low_bits && e < e0 + kLwMaxSplit) { ++e; r <<= 1; continue; }
						failed = true;
						break;
					}
					if (tid == 0) t_unique += claims;
					t_max += r_max;
					leaf_claims += claims;
					// ---- reached & ~over is the result: survivors per virtual group (= the top 8 key bits of the entry)
					const uint64_t key_hi = (((uint64_t)(a.leaf_prefix | leaf) << e) | (uint64_t)r) << kb;          // (low_bits + bits of the leaf index <= 64)
					const uint32_t vgs = cb + (kb > kLcVgBits ? kb - kLcVgBits : 0u);
					const uint32_t vgm = kb >= kLcVgBits ? kLcVg - 1u : ((1u << kb) - 1u);
					for (uint32_t wi = tid; wi < NW; wi += NT)
						for (uint32_t w = S.surv[wi] & ~S.over[wi]; w; w &= w - 1) {
							const uint32_t s = wi * 32 + (uint32_t)(__ffs(w) - 1);
							atomicAdd(&S.vcur[(uint32_t)(S.main[s] >> vgs) & vgm], 1u);
						}
					__syncthreads();
					if (warp == 0) {
						uint32_t c[kLcVg / 32], sum = 0;
#pragma unroll
						for (int i = 0; i < (int)(kLcVg / 32); ++i) { c[i] = S.vcur[lane * (kLcVg / 32) + i]; sum += c[i]; }
						uint32_t inc = sum;
#pragma unroll
						for (int o = 1; o < 32; o <<= 1) {
							const uint32_t t = __shfl_up_sync(FULL, inc, o);
							if (lane >= (uint32_t)o) inc += t;
						}
						uint32_t ex = inc - sum;
#pragma unroll
						for (int i = 0; i < (int)(kLcVg / 32); ++i) { S.vbase[lane * (kLcVg / 32) + i] = ex; S.vcur[lane * (kLcVg / 32) + i] = ex; ex += c[i]; }
						if (lane == 31) S.vbase[kLcVg] = inc;
					}
					__syncthreads();
					const uint32_t n_main = S.vbase[kLcVg];
					if (n_main) {
						for (uint32_t wi = tid; wi < NW; wi += NT)          // the list of survivors, group by group
							for (uint32_t w = S.surv[wi] & ~S.over[wi]; w; w &= w - 1) {
								const uint32_t s = wi * 32 + (uint32_t)(__ffs(w) - 1);
								list[atomicAdd(&S.vcur[(uint32_t)(S.main[s] >> vgs) & vgm], 1u)] = (uint16_t)s;
							}
						__syncthreads();
						// inside its group a k-mer is placed by comparing it with the other survivors of the group
						for (uint32_t q = tid; q < n_main; q += NT) {
							const uint64_t ent = S.main[list[q]];
							const uint64_t rem = (ent >> cb) & rem_mask;
							const uint32_t vg = (uint32_t)(ent >> vgs) & vgm;
							const uint32_t q_lo = S.vbase[vg], q_hi = S.vbase[vg + 1];
							uint32_t pos = q_lo;
							for (uint32_t j = q_lo; j < q_hi; ++j) pos += (((S.main[list[j]] >> cb) & rem_mask) < rem) ? 1u : 0u;
							R kk; kk.w[0] = key_hi | rem;
							const uint32_t c = (uint32_t)ent & cmask;
							const uint32_t value = c > a.counter_max ? a.counter_max : c;          // kb_sorter.h:1190
							uint64_t* dst = tmp64 + (lo + emit_base + pos) * padw;
							for (uint32_t w = 0; w < padw; ++w) dst[w] = lw_out_word<1>(kk, value, a.suffix_bytes, w);
							if (!one_prefix) atomicAdd(reinterpret_cast<unsigned long long*>(a.lut) + rec_prefix<1>(kk, prefix_shift), 1ull);     // kb_sorter.h:1203
						}
						emit_base += n_main;
					}
					__syncthreads();          // (the emission is done with the table, the bitmaps and the list before the next round clears them)
					// ---- next round: back up from finished halves of a split, then one step to the right
					while (e > e0 && (r & 1u)) { r >>= 1; --e; }
					++r;
					if (e == e0 && r == (1u << e0)) break;
				}
				if (!failed && m >= 256u) {          // distinct k-mers per record of this leaf -> the estimate the next leaves are planned with
					const uint32_t q8 = min(max(leaf_claims * 256u / m, 8u), 256u);
					ratio_q8 = (ratio_q8 + q8 + 1u) >> 1;
				}
			}
			if (tid == 0) {
				a.leaf_emit[leaf] = failed ? 0u : emit_base;
				if (emit_base && !failed) atomicAdd(&a.group_sum[leaf >> 10], emit_base);          // for leaf_scan_kernel
				t_emit += emit_base;
				if (one_prefix && emit_base && !failed)
					atomicAdd(reinterpret_cast<unsigned long long*>(a.lut) + ((a.leaf_prefix | leaf) >> (prefix_shift - a.low_bits)), (unsigned long long)emit_base);      // leaf = k-mer >> low_bits
			}
		}
		__syncthreads();          // (the next ticket and the heavy-list flag are visible)
		if (failed || S.failed) { failed = true; break; }
		par ^= 1u;
		work = S.ticket[par];
	}
	// ---- statistics of this CTA
	if (failed) { if (tid == 0) atomicOr(a.flags, kMsdFlagFallback); return; }
	t_max = __reduce_add_sync(FULL, t_max);
	if (lane == 0 && t_max) atomicAdd(&S.stat_max, t_max);
	__syncthreads();
	if (tid == 0) {
		const uint32_t tm = S.stat_max;
		if (t_unique) atomicAdd(reinterpret_cast<unsigned long long*>(a.result), (unsigned long long)t_unique);
		if (t_unique - t_emit - tm) atomicAdd(reinterpret_cast<unsigned long long*>(a.result) + 1, (unsigned long long)(t_unique - t_emit - tm));
		if (tm) atomicAdd(reinterpret_cast<unsigned long long*>(a.result) + 2, (unsigned long long)tm);
	}
}

}  // namespace kmcb
