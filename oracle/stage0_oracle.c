/* Plain-C restatement of KMC's stage-0 statistics and of the collector's (k+x)-mer count (TEST INFRASTRUCTURE); see stage0_oracle.h. */
#include "stage0_oracle.h"
#include "stage1_oracle.h"

#include <stdlib.h>

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

/* CSplitter::CalcStats (kmc_core/splitter.cpp:439-533), statement by statement, over the batch as one sequence in which every non-ACGT
 * byte plays the reference's 'N' (a read end ends the current k-mers the same way).  `cur` is current_signature, `end` end_mmer: the
 * m-mer ending at i and its normalised value; `sig_pos` is signature_start_pos. */
int kmcs_signature_stats(uint32_t k, uint32_t m, const uint8_t* seq, uint64_t size, uint32_t* stats)
{
	if (m < 5 || m > 11 || k <= m || k > 128 || (size && !seq) || !stats) return -1;
	uint32_t* norm = (uint32_t*)malloc(sizeof(uint32_t) << (2 * m));
	if (!norm) return -2;
	kmcs_norm_table(m, norm);
	const uint32_t mask = (1u << (2 * m)) - 1u;
	uint64_t i = 0, sig_pos = 0;
	uint32_t len = 0, cur = 0, end_str = 0, end = 0;
	while (i + k - 1 < size) {
		int contains_n = 0;
		for (uint32_t j = 0; j < m; ++j, ++i)
			if (code_of(seq[i]) < 0) { contains_n = 1; break; }
		if (contains_n) { ++i; continue; }
		len = m;
		sig_pos = i - m;
		end_str = 0;
		for (uint32_t j = 0; j < m; ++j) end_str = (end_str << 2) | (uint32_t)code_of(seq[sig_pos + j]);
		cur = end = norm[end_str];
		for (; i < size; ++i) {
			const int x = code_of(seq[i]);
			if (x < 0) {
				if (len >= k) stats[cur] += 1 + len - k;
				len = 0;
				++i;
				break;
			}
			end_str = ((end_str << 2) | (uint32_t)x) & mask;
			end = norm[end_str];
			if (end < cur) {
				if (len >= k) { stats[cur] += 1 + len - k; len = k - 1; }
				cur = end;
				sig_pos = i - m + 1;
			} else if (end == cur) {
				sig_pos = i - m + 1;
			} else if (sig_pos + k - 1 < i) {
				stats[cur] += 1 + len - k;
				len = k - 1;
				++sig_pos;
				end_str = 0;
				for (uint32_t j = 0; j < m; ++j) end_str = (end_str << 2) | (uint32_t)code_of(seq[sig_pos + j]);
				cur = end = norm[end_str];
				for (uint64_t j = sig_pos + m; j <= i; ++j) {
					end_str = ((end_str << 2) | (uint32_t)code_of(seq[j])) & mask;
					end = norm[end_str];
					if (end <= cur) { cur = end; sig_pos = j - m + 1; }
				}
			}
			++len;
		}
	}
	if (len >= k) stats[cur] += 1 + len - k;
	free(norm);
	return 0;
}

/* CKmerBinCollector::update_n_plus_x_recs (kb_collector.h:66-116) for one record of n symbols (codes 0..3) */
static uint64_t kx_canonical(const uint8_t* s, uint32_t n, uint32_t k, uint32_t divide)
{
	uint32_t kmer = (uint32_t)((s[0] << 6) + (s[1] << 4) + (s[2] << 2) + s[3]) & 0xffu;
	uint32_t rev = (uint32_t)(((3 - s[k - 1]) << 6) + ((3 - s[k - 2]) << 4) + ((3 - s[k - 3]) << 2) + (3 - s[k - 4])) & 0xffu;
	uint32_t kmer_pos = 4, rev_pos = k, x = 0;
	uint64_t total = 0;
	int state = kmer < rev ? 0 : rev < kmer ? 1 : 2;
	for (uint32_t i = 0; i < n - k; ++i) {
		rev = ((rev >> 2) + ((3u - s[rev_pos++]) << 6)) & 0xffu;
		kmer = ((kmer << 2) + s[kmer_pos++]) & 0xffu;
		const int st = kmer < rev ? 0 : rev < kmer ? 1 : 2;
		if (st == state) {
			if (state == 2) ++total;
			else ++x;
		} else {
			state = st;
			total += 1 + x / divide;
			x = 0;
		}
	}
	return total + 1 + x / divide;
}

uint64_t kmcs_kxmer_count(uint32_t k, int both_strands, const uint8_t* data, uint64_t bytes)
{
	const uint32_t max_x = k % 32 ? (31 - k % 32 < 3 ? 31 - k % 32 : 3) : 0;
	if (!max_x) return 0;
	uint8_t sym[128 + 256];
	uint64_t total = 0, pos = 0;
	while (pos < bytes) {
		const uint32_t n = k + data[pos];
		for (uint32_t i = 0; i < n; ++i) sym[i] = (uint8_t)((data[pos + 1 + i / 4] >> (6 - 2 * (i % 4))) & 3u);
		total += both_strands ? kx_canonical(sym, n, k, max_x + 1) : 1 + (uint64_t)(n - k) / (max_x + 1);
		pos += 1 + (n + 3) / 4;
	}
	return total;
}
