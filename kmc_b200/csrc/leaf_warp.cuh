// kmc_b200 — what the leaf kernels of the hybrid MSD path share, the kernel for one-word leaves with a DOMINANT k-mer, and the two
// kernels that pack the counted leaves into the output.
//
// What stage 2 needs from a leaf bucket (records that share their top 8+b2 bits, ~1 K records) is the sorted list of its DISTINCT
// k-mers with their multiplicities (CompactKmers, kmc_core/kb_sorter.h:1128-1281; for k % 32 != 0 the same result comes out of
// CompactKxmers :937-1122 + kxmer_set.h).  The leaf kernels (leaf_hash.cuh, leaf_hash_cta.cuh, leaf_hash_wide.cuh) count a leaf in a
// hash table instead of sorting every copy, apply the cutoffs (kb_sorter.h:1174-1191) and emit the survivors lane-dense (record bytes /
// clamp / lut[prefix]++ as kb_sorter.h:1190-1203) into the leaf's region of a temporary buffer; leaf_scan_kernel + leaf_gather_kernel
// pack the regions into the output.  This file holds their interface (LeafArgs) and the helpers they share.
//
// leaf_warp_kernel counts the one-word leaves of more than kLwHeavy records, which the leaf kernels only note (LeafArgs::heavy_list).
// A leaf gets that large when ONE k-mer has 10^5..10^6 copies (poly-A, satellite repeats): its copies are counted by comparison and
// enter the table once, with their number.  The rest of the leaf is counted by one warp in a hash table whose GROUPS are ordered:
//   * the table is groups of 64 slots; the group of a k-mer is its next bits (monotone: group order is k-mer order),
//     the slot inside the group is a hash of the remaining bits, linear probing stays inside the group.  (A fully
//     order-preserving table does not work: a sequencing error late in a k-mer leaves its leading bits untouched, so a real
//     k-mer and its error variants would all fight for one slot - measured: 1/3 of the records collided.)
//     The first copy claims a slot with one 64-bit atomicCAS, every other copy is one 32-bit atomicAdd on the count;
//   * the cutoffs are applied ON THE WAY: the add that lifts a count to cutoff_min sets the entry's bit in a bitmap (one word per
//     group), the add that lifts it past cutoff_max sets it in a second one.  When the last record is in, reached & ~over IS the set
//     of survivors: prefix popcounts of the words are the output positions of the groups, and inside a group (a handful of
//     survivors) a k-mer is placed by comparing it with the other survivors of its word.
// The leaf is counted in 2^e rounds over sub-ranges of its next e bits (a cheap scan compacts the round's k-mers into a ring in shared
// memory, the ring is inserted densely); a round in which a group fills up is split in two on the next bit (binary descent, nothing of
// it has been emitted yet).  Only a leaf beyond kLwMaxHeavyLeaf records, a rest beyond kLwMaxLeaf records, or a k-mer range that cannot
// be split any further raises the device flag: the LSD passes + count_emit_kernel behind then redo the bin.
//
// Entry format (64 bit, EMPTY = all ones): [ key bits below the group bits (<= 47) | count ]; the k-mer is rebuilt from leaf, round,
// group and entry.
#pragma once
#include "common.cuh"
#include "expand.cuh"
#include "msd_sort.cuh"
#include "count.cuh"

namespace kmcb {

constexpr int kLwWarps = 4;                      // warps per CTA (independent of each other)
constexpr uint32_t kLwGroupBits = 6;             // slots per group = 64: a real k-mer and its error variants share a group, groups must absorb such clumps
constexpr int kLwList = 256;                     // u16 list of survivors, one step of the emission
constexpr uint32_t kLwRing = 256;                // ring of the compacted k-mers of a round
constexpr int kLwMinBlocks = 7;                  // leaf_warp_kernel: CTAs per SM it is compiled for
constexpr uint32_t kLwMaxLeaf = 65534;           // records of a warp-counted leaf (count field >= 16 bits)
constexpr uint32_t kLwHeavy = 16384;             // one-word records: a leaf beyond this is first relieved of the copies of ONE dominant k-mer (poly-A,
                                                 // satellite repeats: a k-mer with 10^5..10^6 copies makes its leaf that large); what remains must fit kLwMaxLeaf
constexpr uint32_t kLwMaxHeavyLeaf = 1u << 22;   // ... and the whole leaf must stay below this (one warp streams it a few times)
constexpr uint32_t kLwMaxSplit = 12;             // extra split bits a round may descend
constexpr uint64_t kLwEmpty = ~0ull;

struct LeafArgs {
	const void* recs;            // partitioned records
	const uint64_t* start;       // [n_leaves + 1]
	uint32_t n_leaves;
	uint32_t low_bits;           // bits below the partition digits
	uint32_t heavy_cap;          // one-word records: entries of heavy_list (below).  In this slot the u32 fields after it keep their 8-byte pairing,
	                             // which the leaf kernels' code depends on (moved one word apart, leaf_hash_wide_kernel took 1-2 registers more)
	uint32_t fill_pct;           // leaf_hash_kernel: distinct k-mers a round of the table is planned for, in percent of its slots
	uint32_t ratio0_q8;          // leaf_hash_kernel: first estimate of distinct k-mers per record, x 256 (every warp then follows what it sees)
	uint32_t leaf_prefix;        // key block of an oversized bin: (block prefix << log2(n_leaves)), so that (leaf_prefix | leaf) = k-mer >> low_bits; else 0
	uint32_t k, lut_prefix_len, cutoff_min, cutoff_max, counter_max, counter_bytes, suffix_bytes;
	uint8_t* tmp;                // leaf L writes its records, padded to a multiple of 8 bytes, at tmp + start[L] * pad
	uint32_t* leaf_emit;         // [n_leaves] emitted records
	uint32_t* group_sum;         // [n_leaves / 1024] their sums (zero-initialised)
	uint64_t* lut;
	uint64_t* result;            // [0] n_unique [1] n_cutoff_min [2] n_cutoff_max
	uint32_t* ticket;
	uint32_t* flags;
	// one-word records: leaves beyond kLwHeavy records are noted by the leaf kernel and counted by leaf_warp_kernel (dominant-k-mer path)
	uint32_t* heavy_list; uint32_t* heavy_count; uint32_t* heavy_ticket;
};

template <int SLOT_BITS>
struct LwSmem {
	static constexpr int kSlots = 1 << SLOT_BITS;
	uint64_t main[kSlots];           // the table: ordered groups of 64 hashed slots
	uint64_t ring[kLwRing];          // k-mers of the current round, compacted; during the emission the u16 list lives here
	uint32_t surv[kSlots / 32];      // per group: entries whose count reached cutoff_min (later: the survivors) ...
	uint32_t over[kSlots / 32];      // ... whose count went past cutoff_max (later: survivors in earlier groups)
	__device__ __forceinline__ uint16_t* list() { return reinterpret_cast<uint16_t*>(ring); }       // [kLwList]
};
static_assert(kLwRing * 8 >= kLwList * 2, "the u16 list lives in the ring");

template <int WORDS>
__device__ __forceinline__ Rec<WORDS> lw_load(const Rec<WORDS>* p)
{
	Rec<WORDS> r;
	if (WORDS == 2) {
		const ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2*>(p));
		r.w[0] = v.x; r.w[WORDS - 1] = v.y;
	} else if (WORDS == 4) {
		const ulonglong2 v0 = __ldg(reinterpret_cast<const ulonglong2*>(p)), v1 = __ldg(reinterpret_cast<const ulonglong2*>(p) + 1);
		r.w[0] = v0.x; r.w[1 % WORDS] = v0.y; r.w[2 % WORDS] = v1.x; r.w[3 % WORDS] = v1.y;
	} else {
#pragma unroll
		for (int i = 0; i < WORDS; ++i) r.w[i] = __ldg(reinterpret_cast<const unsigned long long*>(p) + i);
	}
	return r;
}

// 64 bits of the record starting at bit `pos` (multiple of 8, < 64 * WORDS)
template <int WORDS>
__device__ __forceinline__ uint64_t lw_extract64(const Rec<WORDS>& r, uint32_t pos)
{
	const uint32_t wi = pos >> 6, off = pos & 63u;
	uint64_t lo = r.w[0], hi = 0;
#pragma unroll
	for (int i = 1; i < WORDS; ++i) {
		if (wi == (uint32_t)i) lo = r.w[i];
		if (wi + 1 == (uint32_t)i) hi = r.w[i];
	}
	if (WORDS == 1 || wi + 1 >= (uint32_t)WORDS) hi = 0;
	uint64_t v = lo >> off;
	if (off) v |= hi << (64u - off);
	return v;
}

// word w of the emitted record: (k-p)/4 suffix bytes most significant first, then the counter least significant first
// (kb_sorter.h:1198-1201), as little-endian 64-bit words (byte 0 of the record = bits 0-7 of word 0)
template <int WORDS>
__device__ __forceinline__ uint64_t lw_out_word(const Rec<WORDS>& key, uint32_t value, uint32_t sb, uint32_t w)
{
	const int nkb = (int)sb - 8 * (int)w;          // suffix bytes still to go out from this word on
	if (nkb >= 8) return bswap64(lw_extract64<WORDS>(key, 8u * (uint32_t)(nkb - 8)));
	if (nkb > 0) return bswap64(key.w[0] << (8 * (8 - nkb))) | ((uint64_t)value << (8 * nkb));
	const int sh = -nkb;
	return sh < 4 ? (uint64_t)(value >> (8 * sh)) : 0ull;
}

// cutoffs applied on the way (kb_sorter.h:1174-1191): what happens when a count goes from c-1 to c
struct LwCut {
	uint32_t cmin;               // max(cutoff_min, 1): reaching it makes a survivor ...
	uint32_t cmax1;              // ... reaching cutoff_max + 1 unmakes it (0 = never: cutoff_max is 2^32 - 1)
	bool never;                  // cutoff_max < cutoff_min: nothing survives, whatever reaches cmin counts as n_cutoff_max
};
// (two bitmaps, both only ever OR-ed: the result does not depend on the order in which lanes get to run)
__device__ __forceinline__ void lw_transition(const LwCut& c, uint32_t newc, uint32_t* reached, uint32_t* over, uint32_t idx, uint32_t& r_max)
{
	if (newc != c.cmin && newc != c.cmax1) return;          // almost every add
	if (newc == c.cmin) {
		if (c.never) ++r_max;
		else atomicOr(&reached[idx >> 5], 1u << (idx & 31u));
	}
	if (newc == c.cmax1 && !c.never) { atomicOr(&over[idx >> 5], 1u << (idx & 31u)); ++r_max; }
}

// ---- V k-mers per lane into the warp's table.  The first probes of all V are issued before any result is looked at (their latencies
// overlap); further probes (the slot belongs to another k-mer) walk the 32 slots of the group.
struct LwRound {
	uint64_t* main; uint32_t* surv; uint32_t* over;
	uint32_t gshift, gmask, cb, cmask;
	uint64_t rem_mask;
	LwCut cut;
};

// slot of a k-mer: its group (the bits above gshift), then a hash of the bits below
__device__ __forceinline__ uint32_t lw_slot(uint64_t kmer, uint64_t rem, uint32_t gshift, uint32_t gmask)
{
	return ((((uint32_t)(kmer >> gshift)) & gmask) << kLwGroupBits) | ((((uint32_t)rem ^ (uint32_t)(rem >> 27)) * 0x9E3779B1u) >> (32 - kLwGroupBits));
}

template <int V>
__device__ __forceinline__ void lw_insert1(const LwRound& t, const uint64_t (&kk)[V], uint32_t vmask, uint32_t& r_claim, uint32_t& r_max, bool& ok)
{
	constexpr uint32_t GM = (1u << kLwGroupBits) - 1u;
	uint32_t slot[V];
	unsigned long long old[V], ent[V];
#pragma unroll
	for (int v = 0; v < V; ++v) {
		const uint64_t rem = kk[v] & t.rem_mask;
		slot[v] = lw_slot(kk[v], rem, t.gshift, t.gmask);
		ent[v] = (rem << t.cb) | 1ull;
		old[v] = kLwEmpty;
		if ((vmask >> v) & 1u) old[v] = atomicCAS(reinterpret_cast<unsigned long long*>(&t.main[slot[v]]), (unsigned long long)kLwEmpty, ent[v]);
	}
	// The probe loop only LOOKS for the k-mer's slot: lanes diverge here (the warp iterates as often as its unluckiest lane), so it is
	// kept to a handful of instructions; what happens to the slot comes after it, converged.
#pragma unroll
	for (int v = 0; v < V; ++v) {
		const bool act = (vmask >> v) & 1u;
		const unsigned long long tag = ent[v] >> t.cb;
		uint32_t s = slot[v];
		unsigned long long o = old[v];
		uint32_t probe = 0;
		while (o != kLwEmpty && (o >> t.cb) != tag) {
			if (++probe > GM) break;                                  // the group is full
			s = (s & ~GM) | ((s + 1u) & GM);
			o = atomicCAS(reinterpret_cast<unsigned long long*>(&t.main[s]), (unsigned long long)kLwEmpty, ent[v]);
		}
		if (probe > GM) ok = false;
		else if (act) {
			uint32_t newc = 1u;
			if (o == kLwEmpty) ++r_claim;
			else newc = (atomicAdd(reinterpret_cast<uint32_t*>(&t.main[s]), 1u) & t.cmask) + 1u;      // low word = count
			lw_transition(t.cut, newc, t.surv, t.over, s, r_max);
		}
	}
}

// The one-word leaves the leaf kernels noted (a.heavy_list: more than kLwHeavy records), in a launch of their own after theirs - none in a
// typical bin, so the launch returns at once.  (With the dominant-k-mer path compiled into the main leaf kernel the common case was
// markedly slower: that kernel is sensitive to registers and code layout.)
template <int SLOT_BITS>
__global__ void __launch_bounds__(32 * kLwWarps, kLwMinBlocks) leaf_warp_kernel(const LeafArgs a)
{
	using R = Rec<1>;
	using SM = LwSmem<SLOT_BITS>;
	constexpr int SLOTS = SM::kSlots;
	constexpr int NW = SLOTS / 32;                       // groups = bitmap words (<= 32)
	constexpr int NG = SLOTS >> kLwGroupBits;           // groups
	constexpr uint32_t GB = SLOT_BITS - kLwGroupBits;    // group bits
	constexpr uint32_t GM = (1u << kLwGroupBits) - 1u;
	constexpr uint32_t ROUND = SLOTS;                    // a round that overflows a group is split on the next bit: optimism costs one wasted round
	constexpr uint32_t FULL = 0xffffffffu;
	static_assert(NW <= 32 && NW >= 4, "one bitmap word per lane");
	extern __shared__ __align__(16) uint8_t lw_dsm[];
	SM& S = reinterpret_cast<SM*>(lw_dsm)[threadIdx.x >> 5];
	if (*a.flags & kMsdFlagStop) return;
	const uint32_t lane = threadIdx.x & 31u, lt = lanemask_lt();
	const R* __restrict__ recs = reinterpret_cast<const R*>(a.recs);
	const uint32_t ob = a.suffix_bytes + a.counter_bytes;
	const uint32_t padw = (ob + 7) >> 3;                                   // temporary records: padw 64-bit words
	const uint32_t prefix_shift = 2u * (a.k - a.lut_prefix_len);
	const bool one_prefix = prefix_shift >= a.low_bits;                    // every k-mer of a leaf has the same LUT prefix
	const LwCut cut{a.cutoff_min > 1u ? a.cutoff_min : 1u, a.cutoff_max + 1u, a.cutoff_max < (a.cutoff_min > 1u ? a.cutoff_min : 1u)};
	uint64_t* const tmp64 = reinterpret_cast<uint64_t*>(a.tmp);
	uint16_t* const list = S.list();
	uint32_t t_unique = 0, t_max = 0, t_emit = 0;        // per lane; n_cutoff_min = unique - emitted - n_cutoff_max
	bool failed = false;

	const uint32_t n_work = min(*a.heavy_count, a.heavy_cap);
	uint32_t work = 0;
	if (lane == 0) work = atomicAdd(a.heavy_ticket, 1u);
	work = __shfl_sync(FULL, work, 0);
	while (work < n_work) {
		uint32_t next_t = 0;
		if (lane == 0) next_t = atomicAdd(a.heavy_ticket, 1u);
		const uint32_t leaf = a.heavy_list[work];
		const uint64_t lo = a.start[leaf];
		const uint32_t m = (uint32_t)min(a.start[leaf + 1] - lo, (uint64_t)0xffffffffu);
		uint32_t emit_base = 0;
		// ---- a dominant k-mer?  Its copies are counted by comparison - one ballot per 32 records - and enter the table once, with their
		// number; the table rounds are sized for what remains.  Without this a single k-mer of >= 65535 copies would send the whole bin to
		// the LSD fallback.
		bool heavy = false;
		uint64_t cand = 0;
		uint32_t n_eq = 0, m_rest = m;
		const unsigned long long* __restrict__ g = reinterpret_cast<const unsigned long long*>(recs) + lo;
		if (m > kLwHeavy && m <= kLwMaxHeavyLeaf) {
			// the candidate: the most frequent of 32 evenly spaced records (a k-mer that holds more than a quarter of the leaf is very likely to
			// be it, whatever the order of the leaf's records - level 1 reserves its runs in no fixed order; if not, nothing is lost but this scan)
			{
				const uint64_t smp = __ldg(g + (uint64_t)lane * m / 32);
				uint32_t votes = 0;
				for (int i = 0; i < 32; ++i) votes += __shfl_sync(FULL, smp, i) == smp;
				uint32_t best = (votes << 5) | (31u - lane);          // (ties: the lowest lane)
#pragma unroll
				for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(FULL, best, o));
				cand = __shfl_sync(FULL, smp, 31u - (best & 31u));
			}
			for (uint32_t j0 = 0; j0 < m; j0 += 128) {
				uint64_t v[4];
#pragma unroll
				for (int u = 0; u < 4; ++u) { const uint32_t j = j0 + u * 32 + lane; v[u] = j < m ? __ldg(g + j) : ~cand; }
#pragma unroll
				for (int u = 0; u < 4; ++u) n_eq += __popc(__ballot_sync(FULL, v[u] == cand));
			}
			heavy = n_eq > m / 4;
			if (heavy) m_rest = m - n_eq; else n_eq = 0;
		}
		if (m_rest > kLwMaxLeaf) failed = true;
		else if (m > 0) {
			uint32_t e0 = 0;
			while (((m_rest >> e0) > ROUND && e0 < 8 && e0 < a.low_bits) || a.low_bits - e0 > GB + 47u) ++e0;      // (an entry holds <= 47 key bits)
			uint32_t e = e0, r = 0;
			while (true) {
				// ================================================================ one round: the k-mers whose next e bits are r
				const uint32_t sub_shift = a.low_bits - e;
				const uint32_t gshift = sub_shift > GB ? sub_shift - GB : 0;                      // bits below the group bits
				const uint32_t cb = min(64u - gshift, 32u);                                      // bits of the count field
				const uint64_t rem_mask = (1ull << gshift) - 1ull;                                // gshift <= 47
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
				// ---- insertion: a cheap scan compacts this round's k-mers (but the dominant one) into a ring, the ring is inserted 64 at a time
				uint32_t r_claim = 0, r_max = 0;
				bool ok = true;
				{
					const LwRound T{S.main, S.surv, S.over, gshift, (uint32_t)NG - 1u, cb, cmask, rem_mask, cut};
					uint32_t head = 0, tail = 0;
					uint64_t nx[4];
#pragma unroll
					for (int u = 0; u < 4; ++u) { const uint32_t j = u * 32 + lane; nx[u] = j < m ? __ldg(g + j) : 0ull; }
					for (uint32_t j0 = 0; j0 < m && ok; j0 += 128) {
						uint64_t cur[4];
						bool in[4];
#pragma unroll
						for (int u = 0; u < 4; ++u) { cur[u] = nx[u]; in[u] = (j0 + u * 32 + lane < m) && ((uint32_t)(cur[u] >> sub_shift) & emask) == r && !(heavy && cur[u] == cand); }
#pragma unroll
						for (int u = 0; u < 4; ++u) { const uint32_t j = j0 + 128 + u * 32 + lane; nx[u] = j < m ? __ldg(g + j) : 0ull; }
#pragma unroll
						for (int u = 0; u < 4; ++u) {
							const uint32_t bal = __ballot_sync(FULL, in[u]);
							if (in[u]) S.ring[(tail + __popc(bal & lt)) & (kLwRing - 1)] = cur[u];
							tail += __popc(bal);
						}
						const bool last = j0 + 128 >= m;
						while (tail - head >= 64 || (last && tail != head)) {
							const uint32_t avail = tail - head;
							__syncwarp();
							const uint64_t kk[2] = {S.ring[(head + lane) & (kLwRing - 1)], S.ring[(head + 32 + lane) & (kLwRing - 1)]};
							__syncwarp();
							head += min(avail, 64u);
							lw_insert1<2>(T, kk, (lane < avail ? 1u : 0u) | (32 + lane < avail ? 2u : 0u), r_claim, r_max, ok);
							ok = __all_sync(FULL, ok);
							if (!ok) break;                            // a group is full: the round is split
						}
					}
				}
				// the dominant k-mer enters the table of its round once, with the number of its copies
				if (heavy && ok && ((uint32_t)(cand >> sub_shift) & emask) == r) {
					if (cb < 32 && (n_eq >> cb)) ok = false;          // (the count field of this round is too narrow: split the round - or give up)
					else if (lane == 0) {
						const uint64_t rem = cand & rem_mask;
						uint32_t sl = lw_slot(cand, rem, gshift, (uint32_t)NG - 1u);
						const unsigned long long ent = (rem << cb) | (unsigned long long)n_eq;
						uint32_t probe = 0;
						while (atomicCAS(reinterpret_cast<unsigned long long*>(&S.main[sl]), (unsigned long long)kLwEmpty, ent) != kLwEmpty) {          // (no copy of it is in the table: a free slot of its group is all it needs)
							if (++probe > GM) break;
							sl = (sl & ~GM) | ((sl + 1u) & GM);
						}
						if (probe > GM) ok = false;
						else {
							++r_claim;
							if (n_eq >= cut.cmin) { if (cut.never) ++r_max; else atomicOr(&S.surv[sl >> 5], 1u << (sl & 31u)); }
							if (!cut.never && cut.cmax1 != 0u && n_eq >= cut.cmax1) { atomicOr(&S.over[sl >> 5], 1u << (sl & 31u)); ++r_max; }
						}
					}
				}
				__syncwarp();
				ok = __all_sync(FULL, ok);
				if (!ok) {        // this range does not fit: split it on the next bit (nothing of it has been emitted)
					if (e < a.low_bits && e < e0 + kLwMaxSplit) { ++e; r <<= 1; continue; }
					failed = true;
					break;
				}
				t_unique += r_claim;
				t_max += r_max;
				// the k-mer of an entry
				const uint64_t key_hi = (gshift + GB) >= 64 ? 0ull
					: (((((uint64_t)(a.leaf_prefix | leaf) << a.low_bits) | ((uint64_t)r << sub_shift)) >> (gshift + GB)) << (gshift + GB));
				auto entry_key = [&](uint32_t s, uint64_t ent) -> R {
					R kk;
					kk.w[0] = key_hi | ((uint64_t)(s >> kLwGroupBits) << gshift) | ((ent >> cb) & rem_mask);
					return kk;
				};
				// ---- reached & ~over is the result: prefix popcounts of the words = positions of the groups
				const uint32_t w_main = lane < (uint32_t)NW ? (S.surv[lane] & ~S.over[lane]) : 0u;
				uint32_t inc = __popc(w_main);
#pragma unroll
				for (int o = 1; o < 32; o <<= 1) {
					const uint32_t t = __shfl_up_sync(FULL, inc, o);
					if (lane >= (uint32_t)o) inc += t;
				}
				const uint32_t w_excl = inc - __popc(w_main);
				const uint32_t n_main = __shfl_sync(FULL, inc, 31);
				__syncwarp();
				if (lane < (uint32_t)NW) { S.surv[lane] = w_main; S.over[lane] = w_excl; }
				// ---- survivors: listed group by group (kLwList positions at a time); inside its group a k-mer is placed by comparing it
				// with the other survivors of the word; emitted lane-dense
				for (uint32_t q0 = 0; q0 < n_main; q0 += kLwList) {
					__syncwarp();
					{
						uint32_t w = w_main, q = w_excl;
						while (w) {
							const uint32_t b = __ffs(w) - 1;
							w &= w - 1;
							if (q - q0 < (uint32_t)kLwList) list[q - q0] = (uint16_t)(lane * 32 + b);
							++q;
						}
					}
					__syncwarp();
					const uint32_t q1 = min(n_main, q0 + (uint32_t)kLwList);
					for (uint32_t q = q0 + lane; q < q1; q += 32) {
						const uint32_t s = list[q - q0];
						const uint64_t ent = S.main[s];
						const R kk = entry_key(s, ent);
						const uint32_t w0 = (s >> kLwGroupBits) << (kLwGroupBits - 5);          // first bitmap word of the group
						uint32_t pos = S.over[w0];
#pragma unroll
						for (uint32_t wi = 0; wi < (1u << (kLwGroupBits - 5)); ++wi) {
							uint32_t others = S.surv[w0 + wi];
							if (w0 + wi == (s >> 5)) others &= ~(1u << (s & 31u));
							while (others) {
								const uint32_t s2 = ((w0 + wi) << 5) | (uint32_t)(__ffs(others) - 1);
								others &= others - 1;
								pos += rec_less<1>(entry_key(s2, S.main[s2]), kk) ? 1u : 0u;
							}
						}
						const uint32_t c = (uint32_t)ent & cmask;
						const uint32_t value = c > a.counter_max ? a.counter_max : c;          // kb_sorter.h:1190
						uint64_t* dst = tmp64 + (lo + emit_base + pos) * padw;
						for (uint32_t w = 0; w < padw; ++w) dst[w] = lw_out_word<1>(kk, value, a.suffix_bytes, w);
						if (!one_prefix) atomicAdd(reinterpret_cast<unsigned long long*>(a.lut) + rec_prefix<1>(kk, prefix_shift), 1ull);     // kb_sorter.h:1203
					}
				}
				emit_base += n_main;
				__syncwarp();          // (racecheck, round 2: a lane that leaves the emission early must not clear the table / bitmaps under the lanes still reading them)
				// ---- next round: back up from finished halves of a split, then one step to the right
				while (e > e0 && (r & 1u)) { r >>= 1; --e; }
				++r;
				if (e == e0 && r == (1u << e0)) break;
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

// exclusive scan of the per-leaf record counts: one CTA per group of 1024 leaves; the groups' sums were accumulated by the leaf kernel
// (one atomicAdd per leaf), so a CTA's base is a sum over <= 64 numbers.  total -> result[4], capacity check -> result[5]
__global__ void __launch_bounds__(1024) leaf_scan_kernel(const uint32_t* leaf_emit, const uint32_t* group_sum, uint32_t n_leaves, uint64_t* leaf_off,
	uint64_t* result, uint64_t out_capacity, uint32_t ob, const uint32_t* flags, const uint64_t* out_base)
{
	__shared__ uint32_t s_w[32];
	__shared__ unsigned long long s_base;
	if (*flags & kMsdFlagStop) return;
	const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = blockIdx.x, n_groups = gridDim.x;
	if (warp == 0) {
		unsigned long long b = 0, t = 0;
		for (uint32_t j = lane; j < n_groups; j += 32) { const uint32_t v = group_sum[j]; t += v; if (j < g) b += v; }
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) { b += __shfl_xor_sync(0xffffffffu, b, o); t += __shfl_xor_sync(0xffffffffu, t, o); }
		if (lane == 0) {
			s_base = b;
			if (g == 0) { result[4] = t; if (t * ob > out_capacity) result[5] = 1; }
		}
	}
	const uint32_t i = g * 1024 + tid;
	const uint32_t v = i < n_leaves ? leaf_emit[i] : 0u;
	uint32_t inc = v;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
		if (lane >= (uint32_t)o) inc += t;
	}
	if (lane == 31) s_w[warp] = inc;
	__syncthreads();
	unsigned long long base = s_base;
	for (uint32_t w = 0; w < warp; ++w) base += s_w[w];
	if (i < n_leaves) leaf_off[i] = base + inc - v;
}

// one warp per leaf: its padded temporary records -> packed records at their final place
__global__ void __launch_bounds__(256) leaf_gather_kernel(const uint8_t* tmp, const uint64_t* start, const uint32_t* leaf_emit, const uint64_t* leaf_off,
	uint32_t n_leaves, uint32_t ob, uint8_t* out, const uint64_t* result, const uint32_t* flags, const uint64_t* out_base)
{
	if (*flags & kMsdFlagStop) return;
	if (result[5]) return;                        // capacity error: nothing is written
	const uint32_t leaf = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
	if (leaf >= n_leaves) return;
	const uint32_t pad = ((ob + 7) >> 3) << 3;
	const uint32_t nbytes = leaf_emit[leaf] * ob;
	const uint8_t* src = tmp + start[leaf] * pad;
	uint8_t* dst = out + ((out_base ? *out_base : 0ull) + leaf_off[leaf]) * ob;      // out_base: records of earlier key blocks (oversized bins)
	if (ob <= 8) {
		// records of up to 8 bytes (k - p <= 28 with a one-byte counter: the usual case): a lane takes a whole padded record with one 8-byte load
		// and stores its bytes (per store instruction the warp writes 32 bytes spread over 32 * ob: a few sectors); half the instructions of
		// the byte-by-byte loop below, and wide loads
		const uint32_t n = leaf_emit[leaf];
		const unsigned long long* src8 = reinterpret_cast<const unsigned long long*>(src);
		for (uint32_t r0 = 0; r0 < n; r0 += 64) {
			unsigned long long v[2];
#pragma unroll
			for (int u = 0; u < 2; ++u) { const uint32_t r = r0 + u * 32 + lane; v[u] = r < n ? __ldg(src8 + r) : 0ull; }
#pragma unroll
			for (int u = 0; u < 2; ++u) {
				const uint32_t r = r0 + u * 32 + lane;
				if (r < n) {
					uint8_t* d = dst + (size_t)r * ob;
					for (uint32_t b = 0; b < ob; ++b) d[b] = (uint8_t)(v[u] >> (8 * b));
				}
			}
		}
		return;
	}
	const uint32_t magic = 0xFFFFFFFFu / ob + 1;          // p / ob == umulhi(p, magic) for p < 2^16 ... checked: larger leaves take the division
	const bool use_magic = nbytes < 65536u && ob > 1;     // (ob == 1: magic wraps to 0, and p / 1 needs no trick)
	// (4 independent byte loads in flight per lane: the loop is bound by the latency of its loads)
	for (uint32_t p0 = lane; p0 < nbytes; p0 += 128) {
		uint8_t v[4];
#pragma unroll
		for (int i = 0; i < 4; ++i) {
			const uint32_t p = p0 + 32 * i;
			const uint32_t r = use_magic ? __umulhi(p, magic) : p / ob;
			v[i] = p < nbytes ? __ldg(src + (size_t)r * pad + (p - r * ob)) : (uint8_t)0;
		}
#pragma unroll
		for (int i = 0; i < 4; ++i) {
			const uint32_t p = p0 + 32 * i;
			if (p < nbytes) dst[p] = v[i];
		}
	}
}

}  // namespace kmcb
