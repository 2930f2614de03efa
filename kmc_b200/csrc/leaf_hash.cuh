// kmc_b200 — leaves of one-word records, second design (round 2): ONE HASH TABLE OVER THE WHOLE LEAF, PROBES THAT MISS ARE DEFERRED,
// THE ORDER IS RESTORED AT THE EMISSION.
//
// Same job as leaf_warp_kernel (leaf_warp.cuh: the sorted list of a leaf's DISTINCT k-mers with their multiplicities = CompactKmers,
// kmc_core/kb_sorter.h:1128-1281, fused with the lower levels of the sort), same interface (LeafArgs), same one-warp-per-leaf
// organisation.  What the profile of leaf_warp_kernel said (DESIGN 3.2): most of its warp instructions went to the insertion (the warp
// iterates its probe loop as often as its unluckiest lane) and to the ring that compacts the k-mers of one of several table rounds - and
// on the target workload nearly every record sits in a leaf of several rounds, because
//   * canonical k-mers are not uniform: the leaf sizes of a bin are spread over 0 .. 2x the mean (the density of canonical k-mers
//     falls linearly over the key space), and
//   * the ordered groups of 64 slots overflow long before the table is full: a real k-mer and its ~10 error variants differ in one
//     late symbol, share their leading bits and therefore their group (6 real k-mers in one group fill it), so a round could only be
//     planned for as many RECORDS as the table has slots although only 30 % of them are distinct.
// Here:
//   * the slot is a hash of ALL key bits below the leaf's prefix, linear probing runs over the whole table: clumps of neighbours
//     scatter, a round holds as many records as give ~60 % load (~2100 records of a 30x bin in a 1024-slot table);
//   * a probe that finds another k-mer in its slot is not retried on the spot (lanes would diverge and the warp would wait for the
//     longest probe sequence): the k-mer goes, with its probe count, into a small queue in shared memory, and the queue is drained
//     32 entries at a time by the same straight-line code.  Every probe of every k-mer costs the same few instructions, executed by
//     full warps;
//   * the rounds of a large leaf (sub-ranges of its next e bits) read the leaf with a predicate instead of compacting it;
//   * the cutoffs are applied on the way (two bitmaps, as before); the survivors are brought into key order by a counting sort on their
//     next 6 bits ("virtual groups": no capacity, so no overflow) and a rank by comparison inside the group.
// A round whose table fills up (more distinct k-mers than planned) is split in two on the next bit, as before; each warp keeps a
// running estimate of distinct k-mers per record and plans its rounds with it, so bins of low coverage do not pay for optimism twice.
//
// Entry (64 bit, EMPTY = all ones): [ key bits below the leaf/round prefix (KB <= 48) | count (min(64 - KB, 32) bits) ].
// Queue item (64 bit): [ probes done (16) | key bits (48) ].
#pragma once
#include "leaf_warp.cuh"

namespace kmcb {

#ifndef KMCB200_LH_QUEUE
#define KMCB200_LH_QUEUE 256
#endif
#ifndef KMCB200_LH_MINBLOCKS
#define KMCB200_LH_MINBLOCKS 5
#endif
#ifndef KMCB200_LH_VGBITS
#define KMCB200_LH_VGBITS 6
#endif
constexpr uint32_t kLhQueue = KMCB200_LH_QUEUE;          // deferred probes (a step adds <= 128 to <= 63 left over)
constexpr uint32_t kLhVgBits = KMCB200_LH_VGBITS;        // virtual groups of the emission: 2^6
constexpr uint32_t kLhVg = 1u << kLhVgBits;
constexpr uint32_t kLhKeyBits = 48;                      // key bits of an entry / a queue item
static_assert(kLhVg == 64, "the scan of the virtual groups takes two counters per lane");

template <int SLOT_BITS>
struct LhSmem {
	static constexpr int kSlots = 1 << SLOT_BITS;
	uint64_t main[kSlots];           // the table
	uint64_t queue[kLhQueue];        // deferred probes; during the emission: the u16 list of survivors, in group order
	uint32_t surv[kSlots / 32];      // entries whose count reached cutoff_min ...
	uint32_t over[kSlots / 32];      // ... whose count went past cutoff_max
	uint32_t vbase[kLhVg + 4];       // emission: first list position of every virtual group (+ end)
	uint32_t vcur[kLhVg];            // emission: counters / cursors of the virtual groups
	uint64_t dummy[32];              // one word per lane, always 0: where the CAS of a lane with nothing to insert goes
	__device__ __forceinline__ uint16_t* list() { return reinterpret_cast<uint16_t*>(queue); }       // [kSlots]
};

__device__ __forceinline__ uint32_t lh_hash(uint64_t rem) { return ((uint32_t)rem ^ (uint32_t)(rem >> 27)) * 0x9E3779B1u; }

// Shared-memory atomics on 32-bit shared addresses (inline PTX).  ptxas turns a predicated ATOMS into a branch around it (BSSY / BRA / BSYNC),
// and those reconvergence points fence the four probe chains of a step off from each other; an UNCONDITIONAL atomic keeps the code
// straight-line - a lane with nothing to do aims its CAS at a dummy word of its own (holds 0: the compare with EMPTY fails, nothing is written),
// adds 0 to a count, ORs 0 into a bitmap - but occupies the shared-memory atomic unit for all 32 lanes, and the ORs of 32 lanes into a
// 32-word bitmap collide: everything predicated is the faster default.
#ifndef KMCB200_LH_UNCOND_CAS
#define KMCB200_LH_UNCOND_CAS 0
#endif
#ifndef KMCB200_LH_UNCOND_ADD
#define KMCB200_LH_UNCOND_ADD 0
#endif
#ifndef KMCB200_LH_UNCOND_OR
#define KMCB200_LH_UNCOND_OR 0
#endif
__device__ __forceinline__ unsigned long long lh_cas64(bool p, uint32_t saddr, uint32_t sdummy, unsigned long long val)
{
#if KMCB200_LH_UNCOND_CAS
	unsigned long long old;
	asm volatile("atom.shared.cas.b64 %0, [%1], %2, %3;" : "=l"(old) : "r"(p ? saddr : sdummy), "l"((unsigned long long)kLwEmpty), "l"(val) : "memory");
#else
	unsigned long long old = 0ull;
	asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p atom.shared.cas.b64 %0, [%2], %3, %4;\n\t}"
		: "+l"(old) : "r"((uint32_t)p), "r"(saddr), "l"((unsigned long long)kLwEmpty), "l"(val) : "memory");
#endif
	return old;
}
// KMCB200_LH_LDS_FIRST: look at the slot with a plain load first; only a lane that finds it EMPTY tries to claim it with the (5x more expensive)
// CAS.64 - three of four records of a 30x bin are copies of a k-mer that is in the table already
#ifndef KMCB200_LH_LDS_FIRST
#define KMCB200_LH_LDS_FIRST 1
#endif
__device__ __forceinline__ unsigned long long lh_probe(bool p, uint32_t saddr, uint32_t sdummy, unsigned long long val)
{
#if KMCB200_LH_LDS_FIRST
	unsigned long long cur;
	asm volatile("ld.shared.u64 %0, [%1];" : "=l"(cur) : "r"(saddr) : "memory");
	const bool empty = cur == kLwEmpty;
	const unsigned long long got = lh_cas64(p && empty, saddr, sdummy, val);
	return empty ? got : cur;          // (a slot that was EMPTY may have been taken in between: then the CAS returns its owner)
#else
	return lh_cas64(p, saddr, sdummy, val);
#endif
}
__device__ __forceinline__ uint32_t lh_add32(bool p, uint32_t saddr)
{
#if KMCB200_LH_UNCOND_ADD
	uint32_t old;
	asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(saddr), "r"(p ? 1u : 0u) : "memory");
#else
	uint32_t old = 0u;
	asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p atom.shared.add.u32 %0, [%2], 1;\n\t}" : "+r"(old) : "r"((uint32_t)p), "r"(saddr) : "memory");
#endif
	return old;
}
__device__ __forceinline__ void lh_or32(bool p, uint32_t saddr, uint32_t bits)
{
#if KMCB200_LH_UNCOND_OR
	asm volatile("red.shared.or.b32 [%0], %1;" :: "r"(saddr), "r"(p ? bits : 0u) : "memory");
#else
	asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %0, 0;\n\t@p red.shared.or.b32 [%1], %2;\n\t}" :: "r"((uint32_t)p), "r"(saddr), "r"(bits) : "memory");
#endif
}

struct LhRound {
	uint32_t s_main, s_queue, s_surv, s_over;          // shared-memory addresses of the warp's table, queue and bitmaps
	uint32_t s_dummy;                                  // ... and of this LANE's dummy word (always 0)
	uint64_t* queue;
	uint32_t cb, cmask;
	uint64_t rem_mask, key_unit;                       // key_unit = 1 << cb: two entries hold the same k-mer iff (a ^ b) < key_unit
	uint32_t cmin, cmax1;                              // max(cutoff_min, 1); cutoff_max + 1 (0: never reached)
	bool never, has_max;                               // never: cutoff_max < cutoff_min (whatever reaches cmin counts as n_cutoff_max); has_max: counts can reach cmax1 at all
};

// what a probe found: the slot was empty and is ours now (claimed) / holds this k-mer (one more copy, cutoffs applied on the way:
// kb_sorter.h:1174-1191) / holds another k-mer (returns true: the probe goes on, later)
// SIMPLE: cutoff_min >= 2 and a cutoff_max no count of a leaf can exceed (the usual -ci2 -cx1e9): one compare per copy, nothing per claim
template <bool SIMPLE>
__device__ __forceinline__ bool lh_settle(const LhRound& t, bool act, unsigned long long old, unsigned long long ent, uint32_t slot, uint32_t& r_claim, uint32_t& r_max)
{
	const bool empty = old == kLwEmpty;
	const bool same = !empty && (old ^ ent) < t.key_unit;
	const bool add = act && same;
	const uint32_t newc = (lh_add32(add, t.s_main + slot * 8u) & t.cmask) + 1u;      // low word = count (never carries: count < 2^cb - 1)
	const bool claimed = act && empty;
	r_claim += claimed ? 1u : 0u;
	const uint32_t bit = 1u << (slot & 31u), woff = (slot >> 5) * 4u;
	if (SIMPLE) {
		lh_or32(add && newc == t.cmin, t.s_surv + woff, bit);
	} else {
		const bool at_min = (add && newc == t.cmin) || (claimed && t.cmin == 1u);
		if (t.never) r_max += at_min ? 1u : 0u;
		else lh_or32(at_min, t.s_surv + woff, bit);
		if (t.has_max) {
			const bool at_max = !t.never && ((add && newc == t.cmax1) || (claimed && t.cmax1 == 1u));
			lh_or32(at_max, t.s_over + woff, bit);
			r_max += at_max ? 1u : 0u;
		}
	}
	return act && !empty && !same;
}

// one drain step: up to 64 deferred probes (two per lane, their chains overlap), each moved on by one slot
template <int SLOT_BITS, bool SIMPLE>
__device__ __forceinline__ void lh_drain(const LhRound& t, uint32_t& head, uint32_t& tail, uint32_t lane, uint32_t lt, uint32_t& r_claim, uint32_t& r_max)
{
	constexpr uint32_t SM1 = (1u << SLOT_BITS) - 1u;
	__syncwarp();
	const uint32_t take = min(tail - head, 64u);
	bool act[2];
	uint64_t rem[2];
	uint32_t pc[2], slot[2];
	unsigned long long ent[2], old[2];
#pragma unroll
	for (int u = 0; u < 2; ++u) {
		act[u] = u * 32 + lane < take;
		const uint64_t item = act[u] ? t.queue[(head + u * 32 + lane) & (kLhQueue - 1)] : 0ull;
		rem[u] = item & ((1ull << kLhKeyBits) - 1ull);
		pc[u] = (uint32_t)(item >> kLhKeyBits);
		slot[u] = ((lh_hash(rem[u]) >> (32 - SLOT_BITS)) + pc[u]) & SM1;
		ent[u] = (rem[u] << t.cb) | 1ull;
		old[u] = lh_probe(act[u], t.s_main + slot[u] * 8u, t.s_dummy, ent[u]);
	}
	head += take;
#pragma unroll
	for (int u = 0; u < 2; ++u) {
		const bool miss = lh_settle<SIMPLE>(t, act[u], old[u], ent[u], slot[u], r_claim, r_max);
		const uint32_t bal = __ballot_sync(0xffffffffu, miss);
		if (miss) t.queue[(tail + __popc(bal & lt)) & (kLhQueue - 1)] = ((uint64_t)(pc[u] + 1u) << kLhKeyBits) | rem[u];
		tail += __popc(bal);
	}
}

// when a round's table is full: asked after every step that may have claimed slots (a full table must end the round there, or probes
// would circulate in the queue for ever).  The warp kernel owns its table: its lanes' claims of the round are the whole count.
struct LhWarpCtl {
	static constexpr uint32_t kStride = 128;             // records between two steps of a warp
	uint32_t limit;
	__device__ __forceinline__ bool full(uint32_t& r_claim) const { return __reduce_add_sync(0xffffffffu, r_claim) > limit; }
};

// the insertion of one round: 4 k-mers per lane and step (records first + 128 * i .. + 127, stepping by Ctl::kStride), first probes of all
// four before any result is looked at; returns false when the table fills up (more distinct k-mers than planned).  MULTI: one of several
// rounds of a leaf - only the k-mers whose next bits are r
template <int SLOT_BITS, bool SIMPLE, bool MULTI, class Ctl>
__device__ __forceinline__ bool lh_insert(const LhRound& T, const Ctl& ctl, const unsigned long long* __restrict__ g, uint32_t first, uint32_t m, uint32_t kb,
	uint32_t emask, uint32_t r, uint32_t lane, uint32_t lt, uint32_t& r_claim, uint32_t& r_max)
{
	constexpr uint32_t FULL = 0xffffffffu;
	uint32_t head = 0, tail = 0;
	bool ok = true;
	uint64_t nx[4];
#pragma unroll
	for (int u = 0; u < 4; ++u) { const uint32_t j = first + u * 32 + lane; nx[u] = j < m ? __ldg(g + j) : 0ull; }
	for (uint32_t j0 = first; j0 < m; j0 += Ctl::kStride) {
		uint64_t rem[4];
		uint32_t slot[4];
		unsigned long long ent[4], old[4];
		bool act[4];
#pragma unroll
		for (int u = 0; u < 4; ++u) {
			const uint64_t cur = nx[u];
			act[u] = j0 + u * 32 + lane < m;
			if (MULTI) act[u] = act[u] && (((uint32_t)(cur >> kb) & emask) == r);
			rem[u] = cur & T.rem_mask;
			slot[u] = lh_hash(rem[u]) >> (32 - SLOT_BITS);
			ent[u] = (rem[u] << T.cb) | 1ull;
			old[u] = lh_probe(act[u], T.s_main + slot[u] * 8u, T.s_dummy, ent[u]);
		}
#pragma unroll
		for (int u = 0; u < 4; ++u) { const uint32_t j = j0 + Ctl::kStride + u * 32 + lane; nx[u] = j < m ? __ldg(g + j) : 0ull; }
#pragma unroll
		for (int u = 0; u < 4; ++u) {
			const bool miss = lh_settle<SIMPLE>(T, act[u], old[u], ent[u], slot[u], r_claim, r_max);
			const uint32_t bal = __ballot_sync(FULL, miss);
			if (miss) T.queue[(tail + __popc(bal & lt)) & (kLhQueue - 1)] = (1ull << kLhKeyBits) | rem[u];
			tail += __popc(bal);
		}
		if (ctl.full(r_claim)) ok = false;          // more distinct k-mers than planned: the round is split
		while (ok && tail - head >= 64u) {
			lh_drain<SLOT_BITS, SIMPLE>(T, head, tail, lane, lt, r_claim, r_max);
			if (ctl.full(r_claim)) ok = false;
		}
		if (!ok) break;
	}
	// what is left in the queue at the end of the leaf (< 64 probes): every lane takes one and FOLLOWS it to its slot - a short loop
	// (a few probes) instead of drain steps that each move a handful of probes by one slot and queue them again
	while (ok && tail != head) {
		__syncwarp();
		const uint32_t take = min(tail - head, 32u);
		bool pend = lane < take;
		const uint64_t item = pend ? T.queue[(head + lane) & (kLhQueue - 1)] : 0ull;
		head += take;
		const uint64_t rem = item & ((1ull << kLhKeyBits) - 1ull);
		const unsigned long long ent = (rem << T.cb) | 1ull;
		uint32_t slot = ((lh_hash(rem) >> (32 - SLOT_BITS)) + (uint32_t)(item >> kLhKeyBits)) & ((1u << SLOT_BITS) - 1u);
		while (true) {
			const unsigned long long old = lh_probe(pend, T.s_main + slot * 8u, T.s_dummy, ent);
			pend = lh_settle<SIMPLE>(T, pend, old, ent, slot, r_claim, r_max);
			slot = (slot + 1u) & ((1u << SLOT_BITS) - 1u);
			if (ctl.full(r_claim)) { ok = false; break; }          // (a full table would keep the loop going for ever)
			if (!__any_sync(FULL, pend)) break;
		}
	}
	return ok;
}

template <int SLOT_BITS, bool SIMPLE>
__global__ void __launch_bounds__(32 * kLwWarps, KMCB200_LH_MINBLOCKS) leaf_hash_kernel(const LeafArgs a)
{
	using R = Rec<1>;
	using SM = LhSmem<SLOT_BITS>;
	constexpr int SLOTS = SM::kSlots;
	constexpr int NW = SLOTS / 32;                       // bitmap words (<= 32: one per lane)
	constexpr uint32_t FULL = 0xffffffffu;
	static_assert(NW <= 32 && NW >= 4, "one bitmap word per lane");
	static_assert(kLhQueue * 8 >= (uint32_t)SLOTS * 2, "the u16 list of survivors lives in the queue");
	static_assert(kLhQueue >= 192 && (kLhQueue & (kLhQueue - 1)) == 0, "a step adds up to 128 deferred probes to up to 63 left over");
	extern __shared__ __align__(16) uint8_t lh_dsm[];
	SM& S = reinterpret_cast<SM*>(lh_dsm)[threadIdx.x >> 5];
	if (*a.flags & kMsdFlagStop) return;
	const uint32_t lane = threadIdx.x & 31u, lt = lanemask_lt();
	S.dummy[lane] = 0ull;
	__syncwarp();
	const uint32_t CAP = max((uint32_t)SLOTS * a.fill_pct / 100u, 32u);         // distinct k-mers a round is planned for
	const uint32_t LIMIT = (uint32_t)SLOTS - (uint32_t)SLOTS / 8u;               // ... and where it gives up (the table gets too crowded to probe)
	const unsigned long long* __restrict__ recs = reinterpret_cast<const unsigned long long*>(a.recs);
	const uint32_t ob = a.suffix_bytes + a.counter_bytes;
	const uint32_t padw = (ob + 7) >> 3;                                   // temporary records: padw 64-bit words
	const uint32_t prefix_shift = 2u * (a.k - a.lut_prefix_len);
	const bool one_prefix = prefix_shift >= a.low_bits;                    // every k-mer of a leaf has the same LUT prefix
	const LwCut cut{a.cutoff_min > 1u ? a.cutoff_min : 1u, a.cutoff_max + 1u, a.cutoff_max < (a.cutoff_min > 1u ? a.cutoff_min : 1u)};
	uint64_t* const tmp64 = reinterpret_cast<uint64_t*>(a.tmp);
	uint16_t* const list = S.list();
	uint32_t t_unique = 0, t_max = 0, t_emit = 0;        // per lane; n_cutoff_min = unique - emitted - n_cutoff_max
	uint32_t ratio_q8 = min(max(a.ratio0_q8, 8u), 256u);          // distinct k-mers per record (x 256): running estimate of this warp
	bool failed = false;

	uint32_t work = 0;
	if (lane == 0) work = atomicAdd(a.ticket, 1u);
	work = __shfl_sync(FULL, work, 0);
	while (work < a.n_leaves) {
		uint32_t next_t = 0;
		if (lane == 0) next_t = atomicAdd(a.ticket, 1u);                   // the next leaf: in flight while this one is counted
		const uint32_t leaf = work;
		const uint64_t lo = a.start[leaf];
		const uint32_t m = (uint32_t)min(a.start[leaf + 1] - lo, (uint64_t)0xffffffffu);
		uint32_t emit_base = 0;
		bool prefetched = false;
		if (m > kLwHeavy) {          // a large leaf: noted for the HEAVY launch of leaf_warp_kernel (dominant-k-mer path; its emitted count and LUT share are written there)
			if (lane == 0) {
				const uint32_t slot = atomicAdd(a.heavy_count, 1u);
				if (slot < a.heavy_cap) a.heavy_list[slot] = leaf;
				else failed = true;          // (more large leaves than the list holds: the LSD fallback takes the bin)
			}
			failed = __any_sync(FULL, failed);
			if (failed) break;
			work = __shfl_sync(FULL, next_t, 0);
			continue;
		}
		if (m > 0) {
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
				// ---- clear
				{
					const uint4 ev = make_uint4(~0u, ~0u, ~0u, ~0u), zv = make_uint4(0, 0, 0, 0);
#pragma unroll
					for (int i = 0; i < SLOTS * 8 / 16 / 32; ++i) reinterpret_cast<uint4*>(S.main)[i * 32 + lane] = ev;
					if (lane < 2 * NW / 4) reinterpret_cast<uint4*>(S.surv)[lane] = zv;            // surv, over (contiguous)
				}
				__syncwarp();
				// ---- insertion
				const LhRound T{smem_u32(S.main), smem_u32(S.queue), smem_u32(S.surv), smem_u32(S.over), smem_u32(&S.dummy[lane]), S.queue, cb, cmask, rem_mask, 1ull << cb,
					cut.cmin, cut.cmax1, cut.never, cut.cmax1 != 0u && cut.cmax1 <= kLwHeavy + 1u};
				uint32_t r_claim = 0, r_max = 0;
				const LhWarpCtl ctl{LIMIT};
				const bool ok = e == 0 ? lh_insert<SLOT_BITS, SIMPLE, false>(T, ctl, g, 0u, m, kb, emask, r, lane, lt, r_claim, r_max)
				                       : lh_insert<SLOT_BITS, SIMPLE, true>(T, ctl, g, 0u, m, kb, emask, r, lane, lt, r_claim, r_max);
				if (!prefetched) {        // the next leaf: towards L2 while this one is counted
					prefetched = true;
					const uint32_t nl = __shfl_sync(FULL, next_t, 0);
					if (nl < a.n_leaves) {
						const uint64_t nlo = a.start[nl];
						const uint32_t nm = (uint32_t)min(a.start[nl + 1] - nlo, (uint64_t)kLwHeavy);
						for (uint32_t i = lane * 16; i < nm; i += 32 * 16) asm volatile("prefetch.global.L2 [%0];" ::"l"(recs + nlo + i));
					}
				}
				__syncwarp();
				if (!ok) {        // this range does not fit: split it on the next bit (nothing of it has been emitted)
					if (e < a.low_bits && e < e0 + kLwMaxSplit) { ++e; r <<= 1; continue; }
					failed = true;
					break;
				}
				t_unique += r_claim;
				t_max += r_max;
				leaf_claims += r_claim;
				// ---- reached & ~over is the result
				const uint32_t w_main = lane < (uint32_t)NW ? (S.surv[lane] & ~S.over[lane]) : 0u;
				const uint32_t n_main = __reduce_add_sync(FULL, (uint32_t)__popc(w_main));
				if (n_main) {
					// the k-mer of an entry = prefix of the leaf and the round | its key bits
					const uint64_t key_hi = (((uint64_t)(a.leaf_prefix | leaf) << e) | (uint64_t)r) << kb;          // (low_bits + bits of the leaf index <= 64)
					const uint32_t vgs = cb + (kb > kLhVgBits ? kb - kLhVgBits : 0u);          // virtual group = the top 6 key bits of the entry
					const uint32_t vgm = kb >= kLhVgBits ? kLhVg - 1u : ((1u << kb) - 1u);
					__syncwarp();
					S.vcur[lane] = 0; S.vcur[lane + 32] = 0;
					__syncwarp();
					for (uint32_t w = w_main; w; w &= w - 1) {          // how many survivors per group
						const uint32_t s = lane * 32 + (uint32_t)(__ffs(w) - 1);
						atomicAdd(&S.vcur[(uint32_t)(S.main[s] >> vgs) & vgm], 1u);
					}
					__syncwarp();
					{
						const uint32_t c0 = S.vcur[2 * lane], c1 = S.vcur[2 * lane + 1];
						uint32_t inc = c0 + c1;
#pragma unroll
						for (int o = 1; o < 32; o <<= 1) {
							const uint32_t t = __shfl_up_sync(FULL, inc, o);
							if (lane >= (uint32_t)o) inc += t;
						}
						const uint32_t ex = inc - c0 - c1;
						__syncwarp();
						S.vbase[2 * lane] = ex; S.vbase[2 * lane + 1] = ex + c0;
						S.vcur[2 * lane] = ex; S.vcur[2 * lane + 1] = ex + c0;
						if (lane == 31) S.vbase[kLhVg] = inc;
					}
					__syncwarp();
					for (uint32_t w = w_main; w; w &= w - 1) {          // the list of survivors, group by group
						const uint32_t s = lane * 32 + (uint32_t)(__ffs(w) - 1);
						list[atomicAdd(&S.vcur[(uint32_t)(S.main[s] >> vgs) & vgm], 1u)] = (uint16_t)s;
					}
					__syncwarp();
					// inside its group a k-mer is placed by comparing it with the other survivors of the group; emitted lane-dense
					for (uint32_t q = lane; q < n_main; q += 32) {
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
				__syncwarp();          // (the emission is done with the table, the bitmaps and the list before the next round clears them)
				// ---- next round: back up from finished halves of a split, then one step to the right
				while (e > e0 && (r & 1u)) { r >>= 1; --e; }
				++r;
				if (e == e0 && r == (1u << e0)) break;
			}
			if (!failed && m >= 256u) {          // distinct k-mers per record of this leaf -> the estimate the next leaves are planned with
				const uint32_t q8 = min(max(__reduce_add_sync(FULL, leaf_claims) * 256u / m, 8u), 256u);
				ratio_q8 = (ratio_q8 + q8 + 1u) >> 1;
			}
		}
		if (lane == 0) {
			a.leaf_emit[leaf] = failed ? 0u : emit_base;
			if (emit_base && !failed) atomicAdd(&a.group_sum[leaf >> 10], emit_base);          // for leaf_scan_kernel
			t_emit += emit_base;
			if (one_prefix && emit_base && !failed)
				atomicAdd(reinterpret_cast<unsigned long long*>(a.lut) + ((a.leaf_prefix | leaf) >> (prefix_shift - a.low_bits)), (unsigned long long)emit_base);      // leaf = k-mer >> low_bits
		}
		if (failed) break;
		work = __shfl_sync(FULL, next_t, 0);
	}
	// ---- statistics of this warp
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
