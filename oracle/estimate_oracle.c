/* Plain-C restatement of KMC's histogram estimator (CntHashEstimator, kmc_core/libs/ntHash/ntHashWrapper.h:97-454): Process as the
 * sequential rolling loop, symbol by symbol, and EstimateHistogram.  Test infrastructure: tests/estimate_testlib.py binds it.
 *
 *   est_oracle_increments  the counter increments of a batch (kmcb200_split's format: every byte other than ACGTacgt resets the window, as
 *                          a code of 255 does in Process), each as table * 2^27 + index, in the order Process makes them
 *   est_oracle_histogram   EstimateHistogram from the two tables' histograms of min(65536, counter), bins 0..max_occ
 *
 * The four ntHash seeds are the published constants; the rotated seeds are derived here.  Built with -std=c11 (no FMA contraction) so
 * every product and sum rounds as in the reference. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

static const uint64_t kSeed[4] = {0x3c8bfbb395c60474ull, 0x3193c18562a02b4cull, 0x20323ed082572324ull, 0x295549f54be24456ull};

/* R: the high 31 bits and the low 33 bits each rotated left by one (rol1 + swapbits033) */
static uint64_t rot(uint64_t v)
{
	v = (v << 1) | (v >> 63);
	uint64_t x = (v ^ (v >> 33)) & 1u;
	return v ^ (x | (x << 33));
}

/* R^-1 (ror1 + swapbits3263) */
static uint64_t unrot(uint64_t v)
{
	v = (v >> 1) | (v << 63);
	uint64_t x = ((v >> 32) ^ (v >> 63)) & 1u;
	return v ^ ((x << 32) | (x << 63));
}

static int code(uint8_t c)
{
	switch (c) {
	case 'A': case 'a': return 0;
	case 'C': case 'c': return 1;
	case 'G': case 'g': return 2;
	case 'T': case 't': return 3;
	default: return -1;
	}
}

/* Returns the number of increments; out[0, min(n, cap)) receives them. */
uint64_t est_oracle_increments(const uint8_t* seq, uint64_t len, uint32_t k, uint32_t s, uint64_t* out, uint64_t cap)
{
	uint64_t rk[4];                                             /* R^k(seed[c]) */
	for (int c = 0; c < 4; ++c) {
		rk[c] = kSeed[c];
		for (uint32_t i = 0; i < k; ++i) rk[c] = rot(rk[c]);
	}
	const uint64_t accept1 = (1ull << (s - 1)) - 1ull, mask = (1ull << 27) - 1ull;
	uint8_t* ring = malloc(k);                                  /* the last k symbols */
	uint32_t n_in = 0, head = 0;                               /* symbols in the ring, position of the oldest */
	uint64_t fh = 0, rh = 0, n = 0;
	for (uint64_t i = 0; i < len; ++i) {
		int c = code(seq[i]);
		if (c < 0) {
			n_in = head = 0;
			fh = rh = 0;
			continue;
		}
		int sample;
		if (n_in == k) {                                        /* full: the oldest symbol leaves */
			int o = ring[head];
			fh = rot(fh) ^ rk[o] ^ kSeed[c];
			rh = unrot(rh ^ rk[3 - c] ^ kSeed[3 - o]);
			ring[head] = (uint8_t)c;
			head = (head + 1) % k;
			sample = 1;
		} else {
			fh = rot(fh) ^ kSeed[c];
			rh = unrot(rh ^ rk[3 - c]);
			sample = n_in == k - 1;
			ring[(head + n_in) % k] = (uint8_t)c;
			++n_in;
		}
		if (!sample) continue;
		uint64_t h = rh < fh ? rh : fh;
		uint64_t pref = h >> (63 - s);
		if (pref == 1) {
			if (n < cap) out[n] = h & mask;
			++n;
		}
		if ((pref >> 1) == accept1) {
			if (n < cap) out[n] = (1ull << 27) + (h & mask);
			++n;
		}
	}
	free(ring);
	return n;
}

/* (int64_t)x as x86-64 computes it (cvttsd2si): NaN and out-of-range values give INT64_MIN */
static int64_t to_int64(double x)
{
	if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return INT64_MIN;
	return (int64_t)x;
}

void est_oracle_histogram(const uint32_t* h0, const uint32_t* h1, uint32_t max_occ, uint32_t s, uint64_t* out)
{
	const uint32_t r = 27;
	double* v_mean = malloc(sizeof(double) * (max_occ + 1u));
	double* v_hist = calloc(max_occ + 1u, sizeof(double));
	for (uint32_t i = 0; i <= max_occ; ++i) v_mean[i] = (h0[i] + h1[i]) / 2.0;
	double c_log2 = log(2);
	double log_v_mean0 = log(v_mean[0]);
	double F0Mean = (double)to_int64(((double)r * c_log2 - log_v_mean0) * (double)(1ull << (s + r)));
	for (uint32_t i = 0; i <= max_occ; ++i) out[i] = 0;
	if (!(v_mean[0] * (log_v_mean0 - r * c_log2) == 0)) {
		v_hist[1] = -1.0 * v_mean[1] / (v_mean[0] * (log_v_mean0 - r * c_log2));
		for (uint32_t i = 2; i <= max_occ; ++i) {
			double sum = 0.0;
			for (uint32_t j = 1; j < i; ++j) sum += j * v_mean[i - j] * v_hist[j];
			v_hist[i] = -1.0 * v_mean[i] / (v_mean[0] * (log_v_mean0 - r * c_log2)) - sum / (i * v_mean[0]);
		}
		for (uint32_t i = 1; i <= max_occ; ++i) {
			int64_t v = to_int64(v_hist[i] * F0Mean);
			out[i] = v == INT64_MIN ? 1ull << 63 : (uint64_t)(v < 0 ? -v : v);       /* abs(INT64_MIN) stays INT64_MIN */
		}
	}
	free(v_mean);
	free(v_hist);
}
