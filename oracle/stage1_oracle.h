/* Plain-C restatement of KMC's stage 1 for one batch (TEST INFRASTRUCTURE): the sequential splitter loop of CSplitter::ProcessReads
 * (kmc_core/splitter.cpp:557-677) and the record format of CKmerBinCollector::PutExtendedKmer (kb_collector.cpp:34-90).
 * It follows the reference's incremental signature tracking on purpose, not the per-k-mer rule the GPU kernels use (split.cuh), so
 * that the two check each other.  The batch is one byte array; every byte other than ACGTacgt ends a segment, like N or a read end.
 * Packs follow the library's rule: in a bin, the record that starts at byte s belongs to pack s / 65408. */
#ifndef KMC_STAGE1_ORACLE_H
#define KMC_STAGE1_ORACLE_H
#include <stdint.h>

typedef struct {
	uint32_t kmer_len;
	uint32_t signature_len;     /* 5..11 */
	uint32_t n_bins;            /* every map entry is < n_bins; the identity map (n_bins = 4^m + 1) gives per-signature counts */
} kmcs_params;

/* frags[6 * b + ...] = byte_off, bytes, n_rec (k-mers), n_super_kmers, pack0, n_packs of bin b; bins are concatenated in bin order in
 * out, their packs in pack_bytes.  Returns 0; -5 when out_cap or pack_cap is too small (then *out_bytes / *n_packs are the required
 * sizes and frags is filled, nothing else); -1 for bad parameters or a map value >= n_bins; -2 when out of memory. */
int kmcs_split(const kmcs_params* prm, const uint32_t* map, const uint8_t* seq, uint64_t len,
	uint8_t* out, uint64_t out_cap, uint64_t* out_bytes, uint64_t* pack_bytes, uint64_t pack_cap, uint64_t* n_packs, uint64_t* frags);

/* the normalised value of every m-mer (4^m entries): min(m-mer if allowed, reverse complement if allowed), 4^m when neither is */
void kmcs_norm_table(uint32_t m, uint32_t* norm);

#endif
