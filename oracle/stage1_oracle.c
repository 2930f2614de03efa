/* Plain-C restatement of KMC's stage 1 for one batch (TEST INFRASTRUCTURE); see stage1_oracle.h. */
#include "stage1_oracle.h"

#include <stdlib.h>
#include <string.h>

#define PACK_WINDOW (65536u - 128u)

static int code_of(uint8_t c)
{
	switch (c) {
	case 'A': case 'a': return 0;
	case 'C': case 'c': return 1;
	case 'G': case 'g': return 2;
	case 'T': case 't': return 3;
	default: return -1;
	}
}

/* mmer.h:40-63, symbol by symbol: no AA pair after the first symbol, no ACA prefix, no TT? or TGT suffix */
static int allowed(uint32_t x, uint32_t m)
{
	int s[16];
	for (uint32_t i = 0; i < m; ++i) s[i] = (int)((x >> (2 * (m - 1 - i))) & 3u);
	for (uint32_t i = 1; i + 1 < m; ++i)
		if (s[i] == 0 && s[i + 1] == 0) return 0;
	if (s[0] == 0 && s[1] == 1 && s[2] == 0) return 0;
	if (s[m - 3] == 3 && s[m - 2] == 3) return 0;
	if (s[m - 3] == 3 && s[m - 2] == 2 && s[m - 1] == 3) return 0;
	return 1;
}

void kmcs_norm_table(uint32_t m, uint32_t* norm)
{
	const uint32_t special = 1u << (2 * m);
	for (uint32_t x = 0; x < special; ++x) {
		uint32_t r = 0;
		for (uint32_t i = 0; i < m; ++i) r = (r << 2) | (3u - ((x >> (2 * i)) & 3u));
		const uint32_t f = allowed(x, m) ? x : special, b = allowed(r, m) ? r : special;
		norm[x] = f < b ? f : b;
	}
}

typedef struct {
	uint8_t* data;
	uint64_t bytes, cap, n_rec, n_sk;
} bin_buf;

typedef struct {
	const kmcs_params* prm;
	const uint32_t* map;
	const uint8_t* seq;
	bin_buf* bins;
	int oom;
} ctx_t;

/* kb_collector.cpp:57-71: the byte n - k, then n symbols, 4 per byte, first symbol in bits 7-6 */
static void put_record(ctx_t* c, uint64_t first, uint32_t n, uint32_t signature)
{
	bin_buf* b = &c->bins[c->map[signature]];
	const uint64_t need = 1 + (n + 3) / 4;
	if (b->bytes + need > b->cap) {
		uint64_t nc = b->cap ? 2 * b->cap : 4096;
		while (nc < b->bytes + need) nc *= 2;
		uint8_t* p = (uint8_t*)realloc(b->data, nc);
		if (!p) { c->oom = 1; return; }
		b->data = p;
		b->cap = nc;
	}
	uint8_t* o = b->data + b->bytes;
	o[0] = (uint8_t)(n - c->prm->kmer_len);
	memset(o + 1, 0, need - 1);
	for (uint32_t i = 0; i < n; ++i) o[1 + i / 4] |= (uint8_t)(code_of(c->seq[first + i]) << (6 - 2 * (i % 4)));
	b->bytes += need;
	b->n_rec += n - c->prm->kmer_len + 1;
	b->n_sk += 1;
}

/* The sequential loop over the whole batch.  `sig` / `sig_pos` are the current signature and the start of its latest occurrence, `len`
 * the symbols of the super-k-mer under construction, which ends just before position i. */
static void split_all(ctx_t* c, const uint32_t* norm, uint64_t total)
{
	const uint32_t k = c->prm->kmer_len, m = c->prm->signature_len;
	const uint32_t mmask = (1u << (2 * m)) - 1u;
	const uint8_t* s = c->seq;
	uint64_t i = 0, len = 0;
	uint32_t sig = 0;
	uint64_t sig_pos = 0;
	while (i + k <= total) {
		/* the first m-mer of a segment */
		uint32_t str = 0;
		int bad = 0;
		for (uint32_t j = 0; j < m; ++j, ++i) {
			const int x = code_of(s[i]);
			if (x < 0) { bad = 1; break; }
			str = (str << 2) | (uint32_t)x;
		}
		if (bad) { ++i; continue; }
		sig = norm[str];
		sig_pos = i - m;
		len = m;
		int restart = 0;
		for (; i < total; ++i) {
			const int x = code_of(s[i]);
			if (x < 0) {                       /* the segment ends */
				if (len >= k) put_record(c, i - len, (uint32_t)len, sig);
				len = 0;
				++i;
				restart = 1;
				break;
			}
			str = ((str << 2) | (uint32_t)x) & mmask;
			const uint32_t v = norm[str];
			if (v < sig) {                     /* a smaller m-mer enters: the signature changes */
				if (len >= k) { put_record(c, i - len, (uint32_t)len, sig); len = k - 1; }
				sig = v;
				sig_pos = i + 1 - m;
			} else if (v == sig) {
				sig_pos = i + 1 - m;
			} else if (sig_pos + k <= i) {     /* the signature's m-mer left the k-mer ending at i: find the new minimum */
				put_record(c, i - len, (uint32_t)len, sig);
				len = k - 1;
				uint64_t q = sig_pos + 1;
				uint32_t w = 0;
				for (uint32_t j = 0; j < m; ++j) w = (w << 2) | (uint32_t)code_of(s[q + j]);
				sig = norm[w];
				sig_pos = q;
				for (uint64_t e = q + m; e <= i; ++e) {
					w = ((w << 2) | (uint32_t)code_of(s[e])) & mmask;
					if (norm[w] <= sig) { sig = norm[w]; sig_pos = e + 1 - m; }
				}
			}
			++len;
			if (len == (uint64_t)k + 255) {     /* 256 k-mers: one length byte holds no more */
				put_record(c, i + 1 - len, (uint32_t)len, sig);
				i = i + 2 - k;
				len = 0;
				restart = 1;
				break;
			}
		}
		if (!restart) break;
	}
	if (len >= k) put_record(c, i - len, (uint32_t)len, sig);
}

int kmcs_split(const kmcs_params* prm, const uint32_t* map, const uint8_t* seq, uint64_t len,
	uint8_t* out, uint64_t out_cap, uint64_t* out_bytes, uint64_t* pack_bytes, uint64_t pack_cap, uint64_t* n_packs, uint64_t* frags)
{
	if (!prm || !map || (len && !seq) || !out_bytes || !n_packs || !frags) return -1;
	const uint32_t m = prm->signature_len, k = prm->kmer_len;
	if (m < 5 || m > 11 || k <= m || k > 128 || prm->n_bins < 1) return -1;
	const uint64_t map_size = (1ull << (2 * m)) + 1;
	for (uint64_t x = 0; x < map_size; ++x)
		if (map[x] >= prm->n_bins) return -1;
	uint32_t* norm = (uint32_t*)malloc(sizeof(uint32_t) << (2 * m));
	bin_buf* bins = (bin_buf*)calloc(prm->n_bins, sizeof(bin_buf));
	if (!norm || !bins) { free(norm); free(bins); return -2; }
	kmcs_norm_table(m, norm);
	ctx_t c = {prm, map, seq, bins, 0};
	split_all(&c, norm, len);
	free(norm);
	int rc = c.oom ? -2 : 0;
	/* packs: walk every bin's records */
	uint64_t off = 0, np = 0;
	for (uint32_t b = 0; b < prm->n_bins && !rc; ++b) {
		const bin_buf* bb = &bins[b];
		uint64_t* f = frags + 6 * (uint64_t)b;
		f[0] = off; f[1] = bb->bytes; f[2] = bb->n_rec; f[3] = bb->n_sk; f[4] = np; f[5] = 0;
		uint64_t s = 0, pack_first = 0, cur = (uint64_t)-1;
		while (s < bb->bytes) {
			const uint64_t rec = 1 + ((uint64_t)bb->data[s] + k + 3) / 4;
			if (s / PACK_WINDOW != cur) {
				if (cur != (uint64_t)-1) { if (np < pack_cap && pack_bytes) pack_bytes[np] = s - pack_first; ++np; }
				cur = s / PACK_WINDOW;
				pack_first = s;
				f[5]++;
			}
			s += rec;
		}
		if (bb->bytes) { if (np < pack_cap && pack_bytes) pack_bytes[np] = bb->bytes - pack_first; ++np; }
		off += bb->bytes;
	}
	*out_bytes = off;
	*n_packs = np;
	if (!rc && (off > out_cap || np > pack_cap || (off && !out))) rc = -5;
	for (uint32_t b = 0; b < prm->n_bins; ++b) {
		if (!rc && bins[b].bytes) memcpy(out + frags[6 * (uint64_t)b], bins[b].data, bins[b].bytes);
		free(bins[b].data);
	}
	free(bins);
	return rc;
}
