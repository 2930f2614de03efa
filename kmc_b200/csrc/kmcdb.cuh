// kmc_b200 — KMC database input (`kmc -fkmc`, include/kmc_b200.h "KMC database input"): whole .kmc_suf records -> the reads the
// reference makes of them (CBinaryFilesReader::ProcessKMC, binary_reader.h:238-304, through CKMCFile::ReadNextKmer, kmc_file.cpp:427-499):
// every record whose counter passes the database's own cutoffs becomes its k symbols in ACGT and one '\n', in file order.
//
// A record is sb = (k - lp) / 4 suffix bytes, most significant symbol first, then cs counter bytes, little-endian.  Its lp prefix symbols
// are not stored: record g (counted from the start of the file) has the prefix #{ j >= 1 : lut[j] <= g } & (4^lp - 1)
// (CPrefixFileBufferForListingMode::GetPrefix).  Records are fixed width, so one CTA takes a tile of kKdTile records:
//   kmcdb_count   kept records per tile (the counter filter)
//   scan          split_scan_launch: the tiles' exclusive offsets and the total
//   kmcdb_decode  the tile staged in shared memory, the LUT window of its first and last record found once, each kept record's prefix
//                 by a binary search inside that window, then the output written 16 aligned bytes per thread
// That is 5 launches per call whatever the size.  Record indices are 64-bit throughout: first_record may exceed 2^32.

#pragma once

namespace kmcb {

constexpr uint32_t kKdThreads = 256;
constexpr uint32_t kKdTile = kKdThreads;                                // records per CTA, one per thread
constexpr uint32_t kKdMaxRec = 64 + 4;                                  // (256 - 0) / 4 suffix bytes and a 4-byte counter
constexpr uint32_t kKdAcgt = 0x54474341u;                               // "ACGT", symbol s in byte s
static_assert(kKdThreads == kSplitThreads, "kmcdb_decode scans with split_block_excl");

struct KdGeom {
	uint32_t k, lp, sb, cs, rec;                                        // k-mer length, LUT prefix length, suffix / counter / record bytes
	uint64_t min_count, max_count;                                      // the database's cutoffs
};

// CKMCFile::ReadNextKmer's filter: the counter accumulated into a uint32, not applied when the database stores no counters
__device__ __forceinline__ bool kd_kept(const uint8_t* r, const KdGeom& g)
{
	if (g.cs == 0) return true;
	uint32_t c = 0;
	for (uint32_t b = 0; b < g.cs; ++b) c |= (uint32_t)r[g.sb + b] << (8 * b);
	return !((uint64_t)c < g.min_count || (uint64_t)c > g.max_count);
}

// the smallest j in [lo, hi) with lut[j] > v, or hi
__device__ __forceinline__ uint64_t kd_upper(const uint64_t* __restrict__ lut, uint64_t lo, uint64_t hi, uint64_t v)
{
	while (lo < hi) {
		const uint64_t mid = lo + (hi - lo) / 2;
		if (lut[mid] <= v) lo = mid + 1; else hi = mid;
	}
	return lo;
}

__global__ void __launch_bounds__(kKdThreads) kmcdb_count_kernel(const uint8_t* __restrict__ suf, uint64_t n, KdGeom g,
	uint64_t* __restrict__ tile_kept)
{
	const uint64_t r = (uint64_t)blockIdx.x * kKdTile + threadIdx.x;
	const int kept = __syncthreads_count(r < n && kd_kept(suf + r * g.rec, g));
	if (threadIdx.x == 0) tile_kept[blockIdx.x] = (uint64_t)kept;
}

// result[0] = output bytes, result[1] = kept records; nothing is written to seq when the output exceeds capacity
__global__ void __launch_bounds__(kKdThreads) kmcdb_decode_kernel(const uint8_t* __restrict__ suf, uint64_t n, uint64_t first, KdGeom g,
	const uint64_t* __restrict__ lut, uint64_t lut_entries, const uint64_t* __restrict__ tile_off, const uint64_t* __restrict__ total,
	uint8_t* __restrict__ seq, uint64_t capacity, uint64_t* __restrict__ result)
{
	__shared__ uint4 s_rec4[kKdTile * kKdMaxRec / 16];
	__shared__ uint32_t s_tab[256];                                     // suffix byte -> its 4 symbols, the first in the low byte
	__shared__ uint32_t s_prefix[kKdTile];                              // by kept index
	__shared__ uint16_t s_src[kKdTile];                                 // by kept index: the record's place in the tile
	__shared__ uint64_t s_warp[kKdThreads / 32];
	__shared__ uint64_t s_win[2];
	const uint32_t K1 = g.k + 1;
	const uint64_t kept_all = *total, out_bytes = kept_all * K1;
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		result[0] = out_bytes;
		result[1] = kept_all;
	}
	const uint64_t r0 = (uint64_t)blockIdx.x * kKdTile;
	if (out_bytes > capacity || r0 >= n) return;                        // uniform over the CTA
	const uint32_t m_rec = n - r0 < kKdTile ? (uint32_t)(n - r0) : kKdTile;
	const uint8_t* src = suf + r0 * g.rec;
	const uint32_t bytes = m_rec * g.rec;
	uint8_t* s_rec = reinterpret_cast<uint8_t*>(s_rec4);
	uint32_t head = 0;
	if ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
		head = bytes / 16 * 16;
		for (uint32_t c = threadIdx.x; c < bytes / 16; c += kKdThreads) s_rec4[c] = reinterpret_cast<const uint4*>(src)[c];
	}
	for (uint32_t i = head + threadIdx.x; i < bytes; i += kKdThreads) s_rec[i] = src[i];
	{
		const uint32_t b = threadIdx.x;
		s_tab[b] = (kKdAcgt >> (8 * (b >> 6)) & 255u) | (kKdAcgt >> (8 * ((b >> 4) & 3u)) & 255u) << 8 |
			(kKdAcgt >> (8 * ((b >> 2) & 3u)) & 255u) << 16 | (kKdAcgt >> (8 * (b & 3u)) & 255u) << 24;
	}
	if (threadIdx.x == 0) {                                             // the prefixes of the tile's first and last record
		const uint64_t a = kd_upper(lut, 1, lut_entries, first + r0) - 1;
		s_win[0] = a;
		s_win[1] = kd_upper(lut, a + 1, lut_entries, first + r0 + m_rec - 1) - 1;
	}
	__syncthreads();
	const uint32_t t = threadIdx.x;
	const bool keep = t < m_rec && kd_kept(s_rec + t * g.rec, g);
	uint64_t m = 0;
	const uint32_t local = (uint32_t)split_block_excl<0>(keep ? 1 : 0, s_warp, &m);
	if (keep) {
		const uint64_t a = s_win[0], b = s_win[1];
		const uint64_t cnt = b > a ? kd_upper(lut, a + 1, b + 1, first + r0 + t) - 1 : a;
		s_prefix[local] = (uint32_t)(cnt & ((1ull << (2 * g.lp)) - 1));
		s_src[local] = (uint16_t)t;
	}
	__syncthreads();
	// the tile's output is seq[o0, o0 + m * K1); thread c takes the 16-byte aligned piece c of it, whole pieces in one store
	const uint64_t o0 = tile_off[blockIdx.x] * K1;
	const uint32_t len = (uint32_t)m * K1;
	if (len == 0) return;
	const uintptr_t p0 = reinterpret_cast<uintptr_t>(seq + o0), a0 = p0 & ~(uintptr_t)15;
	const uint64_t n_pieces = (p0 + len - a0 + 15) / 16;
	for (uint64_t c = threadIdx.x; c < n_pieces; c += kKdThreads) {
		const uintptr_t pa = a0 + 16 * c;
		const uint32_t j0 = pa < p0 ? (uint32_t)(p0 - pa) : 0u;          // the piece's first byte of this tile
		uint32_t ob = (uint32_t)(pa + j0 - p0);                            // < kKdTile * 257: 32 bits
		uint32_t rec = ob / K1, pos = ob % K1;
		uint32_t pre = s_prefix[rec];
		const uint8_t* rp = s_rec + s_src[rec] * g.rec;
		uint64_t lo = 0, hi = 0;                                        // the piece's bytes 0-7 and 8-15
		auto put = [&](uint32_t j) {
			uint32_t sym;
			if (pos == g.k) sym = '\n';
			else if (pos < g.lp) sym = kKdAcgt >> (8 * ((pre >> (2 * (g.lp - 1 - pos))) & 3u)) & 255u;
			else {
				const uint32_t q = pos - g.lp;
				sym = s_tab[rp[q >> 2]] >> (8 * (q & 3u)) & 255u;
			}
			if (j < 8) lo |= (uint64_t)sym << (8 * j); else hi |= (uint64_t)sym << (8 * (j - 8));
			if (++pos == K1 && ob + 1 < len) {
				pos = 0;
				++rec;
				pre = s_prefix[rec];
				rp = s_rec + s_src[rec] * g.rec;
			}
			++ob;
		};
		if (j0 == 0 && ob + 16 <= len) {                                  // a whole piece: one 16-byte store
#pragma unroll
			for (uint32_t j = 0; j < 16; ++j) put(j);
			*reinterpret_cast<uint4*>(pa) = make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
		} else {
			uint32_t j = j0;
			for (; j < 16 && ob < len; ++j) put(j);
			for (uint32_t i = j0; i < j; ++i) reinterpret_cast<uint8_t*>(pa)[i] = (uint8_t)((i < 8 ? lo : hi) >> (8 * (i & 7u)));
		}
	}
}

}  // namespace kmcb
