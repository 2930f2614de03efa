// kmc_b200 — BGZF members inflated on the GPU (RFC 1951 DEFLATE inside RFC 1952 gzip members, as `bgzip` / `samtools` write them).
// Included by kmc_b200.cu; the host side (member table, handle, entry points) is gunzip.inl.
//
// A BGZF file is a series of independent gzip members of at most 64 KiB of text each, whose header carries the member's compressed size
// (the 'BC' extra subfield).  No member refers to another, so one warp inflates one member, grid-stride over the members of a call:
//   block headers   lane 0 reads the bit stream (stored, fixed Huffman and dynamic Huffman blocks);
//   decode tables   built by the whole warp in shared memory: code-length counts and canonical order by __match_any_sync, then every
//                   entry of a 2^10 (literal/length) or 2^8 (distance) lookup table decoded from its own index; longer codes are decoded
//                   bit by bit from the canonical counts (gz_slow);
//   tokens          lane 0 decodes up to kGzLits literals / kGzMatches matches into a shared queue; the warp then stores the literals in
//                   parallel and runs the matches in order, each copy lane-parallel: out[p + i] = out[p - d + i % d] reads only bytes
//                   written before the match, so overlapping copies (d < length) need no rounds.  __syncwarp orders the warp's own
//                   global stores before the loads that depend on them.
//   trailer         CRC32 of the output, per-lane slices combined by the GF(2) shift x^(8n) mod P, and ISIZE, as zlib's gzip mode checks.
// Output goes straight into the member's slice of the text buffer; back-references read that slice only.
//
// Validation (a bad member sets the call's error word to min(member << 8 | code), and the call returns KMCB200_ERR_INVALID):
//   every input byte read is inside the member's deflate data (past its end the bit reader shifts in zeros, and a stream that consumed
//   them is truncated, whatever error those zeros would give), every output byte and every back-reference inside [0, ISIZE) of the
//   member's slice; invalid block types, stored lengths whose complement does not match, over-subscribed code sets and the incomplete
//   ones zlib's inflate_table rejects, codes with no symbol, length / distance symbols 286-287 / 30-31, a repeat with no previous length,
//   a dynamic header without end-of-block, a stream that ends before its final block or leaves bytes before the trailer, and CRC32 /
//   ISIZE mismatches.  Each error is the one zlib reports for the same deflate data.
#pragma once
#include <cstdint>

namespace kmcb {

constexpr uint32_t kGzThreads = 128;                                    // 4 warps, 4 members at a time per CTA
constexpr uint32_t kGzWarps = kGzThreads / 32;
constexpr uint32_t kGzLBits = 10;                                       // literal/length lookup: codes of <= 10 bits
constexpr uint32_t kGzDBits = 8;                                        // distance lookup: codes of <= 8 bits
constexpr uint32_t kGzLits = 128;                                       // token queue: literals ...
constexpr uint32_t kGzMatches = 64;                                     // ... and matches per decode round
constexpr uint32_t kGzMaxText = 65536;                                  // BGZF: at most 64 KiB of text per member
constexpr uint32_t kGzTrailer = 8;                                      // CRC32, ISIZE

// error codes of the error word's low byte (gz_error_name)
enum : uint32_t {
	kGzErrMember = 1, kGzErrBlockType, kGzErrStored, kGzErrCodeSet, kGzErrCode, kGzErrDistance, kGzErrOutput, kGzErrTruncated,
	kGzErrIsize, kGzErrCrc, kGzErrTrailing, kGzErrRepeat, kGzErrNoEob
};

__host__ __device__ inline const char* gz_error_name(uint32_t code)
{
	switch (code) {
	case kGzErrMember: return "not a BGZF member inside the buffer (header, sizes or output slice)";
	case kGzErrBlockType: return "invalid block type";
	case kGzErrStored: return "stored block length does not match its complement";
	case kGzErrCodeSet: return "over-subscribed or incomplete code set";
	case kGzErrCode: return "invalid literal/length or distance code";
	case kGzErrDistance: return "distance too far back";
	case kGzErrOutput: return "more output than the member's ISIZE";
	case kGzErrTruncated: return "deflate data ends before its final block";
	case kGzErrIsize: return "ISIZE does not match the inflated length";
	case kGzErrCrc: return "CRC32 mismatch";
	case kGzErrTrailing: return "bytes between the deflate stream and the trailer";
	case kGzErrRepeat: return "invalid code-length repeat";
	case kGzErrNoEob: return "no end-of-block code";
	default: return "unknown error";
	}
}

__constant__ uint16_t c_gz_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_gz_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_gz_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
	6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_gz_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_gz_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// one BGZF member of a call (kmcb200_bgzf_member)
struct GzMember {
	uint64_t in_off, out_off;
	uint32_t in_bytes, isize;
};

// a decode table: counts per code length, symbols in canonical order, and the lookup of the short codes ((symbol << 4) | length, 0: none)
struct GzTable {
	uint32_t count[16];
	uint16_t sym[288];
};

// one warp's shared state
struct GzWarp {
	GzTable lt, dt;
	uint16_t ltab[1u << kGzLBits];
	uint16_t dtab[1u << kGzDBits];
	uint32_t offs[16];
	uint32_t lit_pos[kGzLits];
	uint32_t m_pos[kGzMatches];
	uint32_t m_ld[kGzMatches];                                          // length | distance << 16
	uint8_t lit[kGzLits];
	uint8_t lens[320];                                                  // literal/length code lengths, then the distance ones
	uint8_t cl_lens[20];
	uint32_t n_lit, n_match, err, btype, last, eob, fixed;
	uint32_t copy_dst, copy_len, out_len;
	uint64_t copy_src;
};

// lens[0, n) -> t (counts and canonical order) and tab[1 << bits]; the whole warp calls it.  Returns 0, or kGzErrCodeSet for the sets
// zlib's inflate_table rejects: over-subscribed, or incomplete, except a literal/length or distance set that is a single code of length 1
// (an empty set is accepted: every code of it is then invalid).
__device__ uint32_t gz_build(GzWarp& s, const uint8_t* lens, uint32_t n, GzTable& t, uint16_t* tab, uint32_t bits, bool code_lengths, uint32_t lane)
{
	if (lane < 16) t.count[lane] = 0;
	__syncwarp();
	const uint32_t lt_mask = (1u << lane) - 1;
	for (uint32_t b = 0; b < n; b += 32) {
		const uint32_t L = b + lane < n ? lens[b + lane] : 0;
		const uint32_t peers = __match_any_sync(0xffffffffu, L);
		if (L && (peers & lt_mask) == 0) t.count[L] += __popc(peers);
		__syncwarp();
	}
	uint32_t err = 0;
	if (lane == 0) {
		uint32_t max = 0;
		int left = 1;
		for (uint32_t L = 1; L < 16; ++L) {
			if (t.count[L]) max = L;
			left = (left << 1) - (int)t.count[L];
			if (left < 0) err = kGzErrCodeSet;
		}
		if (max && left > 0 && (code_lengths || max != 1)) err = kGzErrCodeSet;
		uint32_t o = 0;
		for (uint32_t L = 0; L < 16; ++L) { s.offs[L] = o; o += L ? t.count[L] : 0; }
	}
	err = __shfl_sync(0xffffffffu, err, 0);
	if (err) return err;
	__syncwarp();
	for (uint32_t b = 0; b < n; b += 32) {
		const uint32_t L = b + lane < n ? lens[b + lane] : 0;
		const uint32_t peers = __match_any_sync(0xffffffffu, L);
		if (L) t.sym[s.offs[L] + __popc(peers & lt_mask)] = (uint16_t)(b + lane);
		__syncwarp();
		if (L && (peers & lt_mask) == 0) s.offs[L] += __popc(peers);
		__syncwarp();
	}
	for (uint32_t idx = lane; idx < (1u << bits); idx += 32) {
		int code = 0, first = 0, index = 0;
		uint16_t e = 0;
		for (uint32_t L = 1; L <= bits; ++L) {
			code |= (idx >> (L - 1)) & 1;
			const int c = (int)t.count[L];
			if (code - first < c) { e = (uint16_t)((t.sym[index + code - first] << 4) | L); break; }
			index += c;
			first = (first + c) << 1;
			code <<= 1;
		}
		tab[idx] = e;
	}
	__syncwarp();
	return 0;
}

// lane 0's bit reader over raw[ip, end): bytes past `end` read as 0; consumed() past end * 8 means the data was truncated
struct GzBits {
	const uint8_t* raw;
	uint64_t ip, end, bb;
	uint32_t nb;
	__device__ void refill()
	{
		while (nb <= 56) {
			const uint64_t b = ip < end ? raw[ip] : 0;
			++ip;
			bb |= b << nb;
			nb += 8;
		}
	}
	__device__ uint32_t peek(uint32_t n) const { return (uint32_t)(bb & ((1ull << n) - 1)); }
	__device__ void drop(uint32_t n) { bb >>= n; nb -= n; }
	__device__ uint32_t take(uint32_t n) { const uint32_t v = peek(n); drop(n); return v; }
	__device__ uint64_t consumed() const { return ip * 8 - nb; }
};

// a symbol of table t (lookup of `bits` bits, then code by code up to 15 bits); needs >= 15 bits in the reader.  ~0u: no such code, which
// only an empty set or a single 1-bit code has; the one bit is consumed, as zlib's table for such a set consumes it.
__device__ __forceinline__ uint32_t gz_decode(GzBits& r, const GzTable& t, const uint16_t* tab, uint32_t bits)
{
	const uint16_t e = tab[r.peek(bits)];
	if (e & 15) { r.drop(e & 15); return e >> 4; }
	int code = 0, first = 0, index = 0;
	for (uint32_t L = 1; L < 16; ++L) {
		code |= (int)((r.bb >> (L - 1)) & 1);
		const int c = (int)t.count[L];
		if (code - first < c) { r.drop(L); return t.sym[index + code - first]; }
		index += c;
		first = (first + c) << 1;
		code <<= 1;
	}
	r.drop(1);
	return ~0u;
}

// the reflected CRC-32 polynomial arithmetic: a * b mod P, and x^(8n) mod P (1u << 31 is x^0)
__device__ __forceinline__ uint32_t gz_mulmodp(uint32_t a, uint32_t b)
{
	uint32_t p = 0;
	for (uint32_t m = 1u << 31; m; m >>= 1) {
		if (a & m) p ^= b;
		b = (b & 1) ? (b >> 1) ^ 0xedb88320u : b >> 1;
	}
	return p;
}

__device__ uint32_t gz_x8n(uint32_t n)
{
	uint32_t p = 1u << 31, base = 1u << 23;                              // x^0, x^8
	for (; n; n >>= 1) {
		if (n & 1) p = gz_mulmodp(base, p);
		base = gz_mulmodp(base, base);
	}
	return p;
}

// lane 0: the dynamic block header's code lengths into s.lens (the code-length code's table in s.ltab); returns an error code or 0
__device__ uint32_t gz_read_lengths(GzWarp& s, GzBits& r, uint32_t n)
{
	uint32_t i = 0;
	while (i < n) {
		r.refill();
		uint32_t sym = gz_decode(r, s.lt, s.ltab, 7);
		if (sym == ~0u) sym = 0;                                        // an empty code-length code: zlib reads every length as 0
		if (sym < 16) { s.lens[i++] = (uint8_t)sym; continue; }
		uint32_t rep, val = 0;
		if (sym == 16) {
			if (i == 0) return kGzErrRepeat;
			val = s.lens[i - 1];
			rep = 3 + r.take(2);
		} else if (sym == 17) {
			rep = 3 + r.take(3);
		} else {
			rep = 11 + r.take(7);
		}
		if (i + rep > n) return kGzErrRepeat;
		while (rep--) s.lens[i++] = (uint8_t)val;
	}
	return 0;
}

// lane 0: up to kGzLits literals / kGzMatches matches of the current block into the queue; s.eob at the end-of-block code
__device__ uint32_t gz_decode_round(GzWarp& s, GzBits& r, uint32_t& op, uint32_t isize)
{
	uint32_t nl = 0, nm = 0;
	s.eob = 0;
	while (nl < kGzLits && nm < kGzMatches) {
		r.refill();
		const uint32_t sym = gz_decode(r, s.lt, s.ltab, kGzLBits);
		if (sym < 256) {
			if (op >= isize) { s.n_lit = nl; s.n_match = nm; return kGzErrOutput; }
			s.lit_pos[nl] = op++;
			s.lit[nl++] = (uint8_t)sym;
			continue;
		}
		if (sym == 256) { s.eob = 1; break; }
		uint32_t err = 0;
		const uint32_t ls = sym - 257;
		if (sym == ~0u || ls >= 29) err = kGzErrCode;
		uint32_t len = 0, dist = 0;
		if (!err) {
			len = c_gz_lbase[ls] + r.take(c_gz_lext[ls]);
			const uint32_t ds = gz_decode(r, s.dt, s.dtab, kGzDBits);
			if (ds >= 30) err = kGzErrCode;
			else {
				r.refill();
				dist = c_gz_dbase[ds] + r.take(c_gz_dext[ds]);
				if (dist > op) err = kGzErrDistance;
				else if (op + len > isize) err = kGzErrOutput;
			}
		}
		if (err) { s.n_lit = nl; s.n_match = nm; return err; }
		s.m_pos[nm] = op;
		s.m_ld[nm++] = len | dist << 16;
		op += len;
	}
	s.n_lit = nl;
	s.n_match = nm;
	return 0;
}

// the warp: the queued literals, then the matches in order
__device__ __forceinline__ void gz_write_round(GzWarp& s, uint8_t* __restrict__ out, uint32_t lane)
{
	const uint32_t nl = s.n_lit, nm = s.n_match;
	for (uint32_t i = lane; i < nl; i += 32) out[s.lit_pos[i]] = s.lit[i];
	__syncwarp();
	for (uint32_t j = 0; j < nm; ++j) {
		const uint32_t p = s.m_pos[j], len = s.m_ld[j] & 0xffff, d = s.m_ld[j] >> 16;
		if (d >= len) {
			for (uint32_t i = lane; i < len; i += 32) out[p + i] = out[p - d + i];
		} else {
			for (uint32_t i = lane; i < len; i += 32) out[p + i] = out[p - d + i % d];
		}
		__syncwarp();
	}
}

// one member by one warp; returns its error code (0: the text is in out[0, isize) and its CRC32 / ISIZE match the trailer)
__device__ uint32_t gz_member(GzWarp& s, const uint32_t* s_crc, const uint8_t* __restrict__ raw, uint64_t raw_bytes, const GzMember& m,
	uint8_t* __restrict__ text, uint64_t text_capacity, uint32_t lane)
{
	// the header and the slices, checked by every lane alike
	if (m.in_off > raw_bytes || m.in_bytes > raw_bytes - m.in_off || m.in_bytes < 12 + kGzTrailer || m.isize > kGzMaxText ||
		m.out_off > text_capacity || m.isize > text_capacity - m.out_off)
		return kGzErrMember;
	const uint8_t* h = raw + m.in_off;
	const uint32_t xlen = h[10] | (uint32_t)h[11] << 8;
	if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || h[3] != 4 || 12 + xlen + kGzTrailer > m.in_bytes) return kGzErrMember;
	const uint8_t* tr = h + m.in_bytes - kGzTrailer;
	const uint32_t crc_want = tr[0] | (uint32_t)tr[1] << 8 | (uint32_t)tr[2] << 16 | (uint32_t)tr[3] << 24;
	const uint32_t isize_want = tr[4] | (uint32_t)tr[5] << 8 | (uint32_t)tr[6] << 16 | (uint32_t)tr[7] << 24;
	if (isize_want != m.isize) return kGzErrIsize;
	uint8_t* out = text + m.out_off;
	const uint32_t isize = m.isize;

	GzBits r{raw, m.in_off + 12 + xlen, m.in_off + m.in_bytes - kGzTrailer, 0, 0};
	uint32_t op = 0;
	// lane 0's verdict on an error: one found after the reader consumed bits past the member's data came from the zeros shifted in there,
	// so the data ended early (zlib reports such a stream unfinished, whatever those zeros decode to).  The reader stops where an error is
	// found, so consumed() is what the decision needed.
	const auto failed = [&](uint32_t e) { return lane == 0 && r.consumed() > r.end * 8 ? (uint32_t)kGzErrTruncated : e; };
	if (lane == 0) { s.err = 0; s.fixed = 0; }
	__syncwarp();
	for (;;) {
		if (lane == 0) {                                                // the block header
			uint32_t err = r.consumed() > r.end * 8 ? kGzErrTruncated : 0;
			r.refill();
			s.last = r.take(1);
			s.btype = r.take(2);
			if (!err && s.btype == 3) err = kGzErrBlockType;
			if (!err && s.btype == 0) {
				r.drop(r.nb & 7);
				const uint32_t len = r.take(16), nlen = r.take(16);
				const uint64_t at = r.ip - r.nb / 8;                    // the first data byte
				if (len != (~nlen & 0xffff)) err = kGzErrStored;
				else if (at + len > r.end) err = kGzErrTruncated;
				else if (op + len > isize) err = kGzErrOutput;
				if (!err) {
					s.copy_src = at;
					s.copy_dst = op;
					s.copy_len = len;
					r.ip = at + len;
					r.nb = 0;
					r.bb = 0;
					op += len;
				}
			} else if (!err && s.btype == 2) {
				r.refill();
				const uint32_t hlit = r.take(5) + 257, hdist = r.take(5) + 1, hclen = r.take(4) + 4;
				if (hlit > 286 || hdist > 30) err = kGzErrCodeSet;
				for (uint32_t i = 0; i < 19; ++i) s.cl_lens[i] = 0;
				for (uint32_t i = 0; !err && i < hclen; ++i) {
					r.refill();
					s.cl_lens[c_gz_clorder[i]] = (uint8_t)r.take(3);
				}
				s.copy_len = hlit;
				s.copy_dst = hdist;
			}
			s.err = err;
		}
		__syncwarp();
		if (s.err) return failed(s.err);
		const uint32_t btype = s.btype;
		if (btype == 0) {
			const uint64_t src = s.copy_src;
			const uint32_t dst = s.copy_dst, len = s.copy_len;
			for (uint32_t i = lane; i < len; i += 32) out[dst + i] = raw[src + i];
			__syncwarp();
		} else {
			if (btype == 1 && !s.fixed) {
				for (uint32_t i = lane; i < 320; i += 32) s.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : i < 288 ? 8 : 5;
				__syncwarp();
				gz_build(s, s.lens, 288, s.lt, s.ltab, kGzLBits, false, lane);
				gz_build(s, s.lens + 288, 32, s.dt, s.dtab, kGzDBits, false, lane);
				if (lane == 0) s.fixed = 1;
				__syncwarp();
			} else if (btype == 2) {
				const uint32_t hlit = s.copy_len, hdist = s.copy_dst;
				uint32_t err = gz_build(s, s.cl_lens, 19, s.lt, s.ltab, 7, true, lane);
				if (!err) {
					if (lane == 0) {
						err = gz_read_lengths(s, r, hlit + hdist);
						if (!err && s.lens[256] == 0) err = kGzErrNoEob;
						s.err = err;
						s.fixed = 0;
					}
					__syncwarp();
					err = s.err;
				}
				if (!err) err = gz_build(s, s.lens, hlit, s.lt, s.ltab, kGzLBits, false, lane);
				if (!err) err = gz_build(s, s.lens + hlit, hdist, s.dt, s.dtab, kGzDBits, false, lane);
				if (err) return failed(err);
			}
			for (;;) {                                                  // the block's tokens, round by round
				if (lane == 0) s.err = gz_decode_round(s, r, op, isize);
				__syncwarp();
				gz_write_round(s, out, lane);
				const uint32_t err = s.err, eob = s.eob;
				__syncwarp();                                           // read before lane 0 writes the next round
				if (err) return failed(err);
				if (eob) break;
			}
		}
		const uint32_t last = s.last;
		__syncwarp();
		if (last) break;
	}
	// the stream ends on the byte before the trailer, and it gave ISIZE bytes
	if (lane == 0) {
		const uint64_t used = (r.consumed() + 7) / 8;
		s.err = used > r.end ? kGzErrTruncated : used < r.end ? kGzErrTrailing : op != isize ? kGzErrIsize : 0;
	}
	__syncwarp();
	if (s.err) return s.err;

	// CRC32 of out[0, isize): lane slices, lane 0's from the initial ~0, each shifted over the bytes after it
	const uint32_t per = (isize + 31) / 32;
	const uint32_t b0 = min(isize, lane * per), b1 = min(isize, b0 + per);
	uint32_t c = lane == 0 ? 0xffffffffu : 0u;
	for (uint32_t i = b0; i < b1; ++i) c = s_crc[(c ^ out[i]) & 0xff] ^ (c >> 8);
	if (isize - b1) c = gz_mulmodp(gz_x8n(isize - b1), c);
	for (int o = 16; o; o >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, o);
	return (c ^ 0xffffffffu) == crc_want ? 0 : kGzErrCrc;
}

// one warp per member, grid-stride; err: min over the bad members of (member << 8 | code), left as it is (~0) when every member is good
__global__ void __launch_bounds__(kGzThreads) gunzip_kernel(const uint8_t* __restrict__ raw, uint64_t raw_bytes, const GzMember* __restrict__ members,
	uint64_t n_members, uint8_t* __restrict__ text, uint64_t text_capacity, unsigned long long* __restrict__ err)
{
	__shared__ GzWarp s_warp[kGzWarps];
	__shared__ uint32_t s_crc[256];
	for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
		uint32_t c = i;
		for (int j = 0; j < 8; ++j) c = (c & 1) ? (c >> 1) ^ 0xedb88320u : c >> 1;
		s_crc[i] = c;
	}
	__syncthreads();
	const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
	for (uint64_t m = (uint64_t)blockIdx.x * kGzWarps + w; m < n_members; m += (uint64_t)gridDim.x * kGzWarps) {
		const GzMember mb = members[m];
		const uint32_t e = gz_member(s_warp[w], s_crc, raw, raw_bytes, mb, text, text_capacity, lane);
		if (e && lane == 0) atomicMin(err, (unsigned long long)(m << 8 | e));
		__syncwarp();
	}
}

}  // namespace kmcb
