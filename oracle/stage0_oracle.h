/* Plain-C restatement of KMC's stage 0 (TEST INFRASTRUCTURE): the per-signature k-mer statistics of CSplitter::CalcStats
 * (kmc_core/splitter.cpp:439-533), restated literally as a second route to those counts besides the identity-map split of
 * stage1_oracle.c, and the (k+x)-mer count CKmerBinCollector keeps per bin (kb_collector.cpp:73-89, kb_collector.h:66-116).
 * Built together with stage1_oracle.c (it uses kmcs_norm_table) into a library of its own. */
#ifndef KMC_STAGE0_ORACLE_H
#define KMC_STAGE0_ORACLE_H
#include <stdint.h>

/* stats[4^m + 1] is added to (32-bit, wrapping) for the batch as one sequence in which every non-ACGT byte acts as 'N'.
 * Returns 0; -1 for bad parameters; -2 when out of memory. */
int kmcs_signature_stats(uint32_t k, uint32_t m, const uint8_t* seq, uint64_t size, uint32_t* stats);

/* the (k+x)-mers of one bin's stream of records (kmcs_split's format), with max_x = k % 32 ? min(31 - k % 32, 3) : 0; 0 when max_x = 0 */
uint64_t kmcs_kxmer_count(uint32_t k, int both_strands, const uint8_t* data, uint64_t bytes);

#endif
