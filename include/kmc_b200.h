/* kmc_b200 — C ABI of the H100 (sm_90a) implementation of KMC's per-bin stage 2.
 *
 * This is the drop-in boundary: a KMC build binds these entry points where its own CPU code does the
 * per-bin work today.  File:line references are to refresh-bio/KMC 3.2.4.
 *
 *   seam #2 (the drop-in)  kmcb200_process_bin / kmcb200_submit_bin + kmcb200_wait_bin
 *        replaces the body of CKmerBinSorter<SIZE>::ProcessBins  (kmc_core/kb_sorter.h:210-237):
 *        Expand (:728-752) -> Sort (:757-780) -> Compact (:1287-1293) for one bin, i.e. everything
 *        between sorters_manager->GetNext()/bd->read() and kq->push().
 *   seam #1 (sort only)    kmcb200_sort_records
 *        replaces SortFunction<CKmer<SIZE>> (kmc_core/raduls.h:19-20), i.e. RadulsSort::RadixSortMSD_*
 *        (raduls_impl.h:769-776) / RadixSort::RadixSortMSD (radix.h:845-855), as called at kb_sorter.h:775.
 *   device-level twins     kmcb200_dev_*  — same operations on buffers that already live in HBM
 *        (used by bench.py for the kernel-only numbers and by hosts that keep bins resident).
 *
 * Conventions: plain C types only; every function returns 0 on success or a negative kmcb200_status;
 * kmcb200_last_error() gives the message.  A context is bound to one GPU and may be used by one host
 * thread at a time (KMC runs one sorter thread per context).  There is NO CPU fallback: without a usable
 * sm_90 device kmcb200_create fails with KMCB200_ERR_NO_DEVICE.
 *
 * Ordering (every handle, and every slot of a stage-2 context): a device-form call (kmcb200_dev_*) is queued on the caller's
 * stream and returns at once; the handle (slot) records where that work ends, and every later call on the same handle (slot),
 * device or host form, on any stream, starts on the GPU only after it.  Host-form calls are done when they return (submit_bin:
 * once wait_bin has returned).  So the handle's own workspace is never shared by two calls at once, and the caller orders only
 * its own buffers: the inputs it fills before a device-form call and the outputs it reads after one.  Different handles and
 * different contexts are independent: each may be driven by its own host thread, all at once; one handle or context is still
 * used by one host thread at a time (its slots included).  The inflater's device twin uses no workspace of its handle.
 *
 * Environment knobs read by kmcb200_create (development / tests; the defaults are the measured best):
 *   KMCB200_SORT=lsd               plain 8-bit LSD passes instead of the hybrid MSD sort
 *   KMCB200_LEAF_KERNEL=cta|hash   one-word records always by one table per CTA (leaf_hash_cta_kernel) / one table per warp (leaf_hash_kernel);
 *                                  default: the CTA kernel in bins whose mean leaf is > 1280 records, leaf_hash_kernel below
 *   KMCB200_LEAF_CTA=4:B           leaf_hash_cta_kernel: 4 warps per CTA share one table of 2^B slots; 4:12 (default) or 4:10
 *   KMCB200_LEAF_FILL_PCT=n        the hash kernels plan a table round for this load (default 62); KMCB200_LEAF_RATIO0=n: first guess of distinct k-mers per record x 256 (default 90)
 *   KMCB200_L2_BITS=1..10          bits of the second partition level (default: from the bin size: 8 for one-word records; wider records up to 10)
 *   KMCB200_MAX_BLOCK_RECORDS=n    a bin with more k-mers is counted key block by key block (default: what 60 % of the free HBM holds, < 2^32)
 *   KMCB200_KEY_BLOCKS=filter     key blocks of an oversized bin re-expand it with a filter (default: one scattering expansion when the records fit in HBM once)
 *   KMCB200_KEY_BLOCK_RECORDS=n    preferred size of a key block in the scattering flow (default 2^28)
 *   KMCB200_MAX_CHUNK_BYTES=n      ... and expanded in chunks of at most n bytes (default 2^30)
 */
#ifndef KMC_B200_H
#define KMC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KMCB200_VERSION 1
#define KMCB200_MAX_KMER_LEN 128          /* records of up to 4 x 64 bit */
#define KMCB200_MAX_SLOTS 4

typedef enum {
	KMCB200_OK = 0,
	KMCB200_ERR_INVALID = -1,             /* bad argument */
	KMCB200_ERR_NO_DEVICE = -2,           /* no CUDA device / not sm_90 (H100) */
	KMCB200_ERR_CUDA = -3,                /* CUDA runtime error (message in last_error) */
	KMCB200_ERR_BIN_FORMAT = -4,          /* packs do not end on record boundaries / n_rec mismatch */
	KMCB200_ERR_CAPACITY = -5,            /* out_capacity too small */
	KMCB200_ERR_BUSY = -6                 /* slot already holds a submitted bin */
} kmcb200_status;

typedef struct kmcb200_ctx kmcb200_ctx;

/* Per-run parameters: the fields CKmerBinSorter's constructor takes from CKMCParams (kb_sorter.h:165-200). */
typedef struct {
	uint32_t kmer_len;                    /* Params.kmer_len, 1..KMCB200_MAX_KMER_LEN */
	uint32_t both_strands;                /* Params.both_strands: 1 = canonical k-mers */
	uint32_t cutoff_min;                  /* Params.cutoff_min */
	uint32_t cutoff_max;                  /* (uint32)Params.cutoff_max   (kb_sorter.h:186) */
	uint32_t counter_max;                 /* (uint32)Params.counter_max  (kb_sorter.h:187) */
	uint32_t lut_prefix_len;              /* Params.lut_prefix_len, >= 1, (kmer_len - lut_prefix_len) % 4 == 0 */
	int32_t device;                       /* CUDA ordinal */
	uint32_t n_slots;                     /* bins in flight per context (1..KMCB200_MAX_SLOTS); 2 overlaps copies with kernels */
} kmcb200_params;

int kmcb200_create(const kmcb200_params* params, kmcb200_ctx** out_ctx);
void kmcb200_destroy(kmcb200_ctx* ctx);
/* message of the last failure on this context (or of the last failed kmcb200_create when ctx == NULL) */
const char* kmcb200_last_error(const kmcb200_ctx* ctx);

/* bytes of one emitted database record: (k-p)/4 suffix bytes + counter bytes (kb_sorter.h:1132-1142, defs.h:154-159) */
uint32_t kmcb200_out_rec_bytes(const kmcb200_ctx* ctx);
/* size in bytes of the out buffer the reference reserves for a bin of n_rec k-mers (kb_reader.h:141-150) */
uint64_t kmcb200_out_capacity(const kmcb200_ctx* ctx, uint64_t n_rec);
/* entries of the per-bin LUT: 4^lut_prefix_len */
uint64_t kmcb200_lut_entries(const kmcb200_ctx* ctx);

/* Pinned host memory for bin / result buffers (cudaHostAlloc).  A host may instead cudaHostRegister its own arena. */
int kmcb200_host_alloc(kmcb200_ctx* ctx, uint64_t bytes, void** out_ptr);
int kmcb200_host_free(kmcb200_ctx* ctx, void* ptr);

/* ---- seam #2: one bin, host buffers --------------------------------------------------------------
 * Inputs  = what CKmerBinSorter::ProcessBins gets from sorters_manager->GetNext / bd->read / epd->pop:
 *   superkmers/size : the bin byte stream (CMemoryBins::mba_input_file)        kb_sorter.h:216
 *   n_rec           : number of k-mers in the bin (CBinDesc)                   kb_sorter.h:219
 *   n_plus_x_recs   : (k+x)-mer estimate; accepted for signature parity, unused (we never build (k,x)-mers)
 *   pack_bytes[n_packs] : byte length of every expander pack (CExpanderPackDesc, first of each pair,
 *                     queues.h:376-396); packs start on record boundaries.  pack_recs may be NULL (unused).
 *                     A pack may have 0 bytes or more than 64 KiB (the latter is walked by one warp instead of one CTA).
 * Outputs = what is handed to kq->push (kb_sorter.h:1273, queues.h:826):
 *   out_suffix[0, *out_bytes) : the emitted records (one data pack (0, out_pos))
 *   lut[4^p]                  : raw per-prefix counts (the completer does the prefix sum)
 *   stats[4]                  : n_unique, n_cutoff_min, n_cutoff_max, n_total
 * An empty bin (size == 0) is legal and yields zero output and a zero LUT (kb_reader.h:198-205).
 */
int kmcb200_process_bin(kmcb200_ctx* ctx, int32_t bin_id,
	const uint8_t* superkmers, uint64_t size, uint64_t n_rec, uint64_t n_plus_x_recs,
	const uint64_t* pack_bytes, const uint64_t* pack_recs, uint32_t n_packs,
	uint8_t* out_suffix, uint64_t out_capacity, uint64_t* out_bytes,
	uint64_t* lut, uint64_t stats[4]);

/* Asynchronous form: submit returns once the work is queued on the slot's stream; wait blocks until the
 * bin's outputs are in the host buffers given to submit.  Host buffers should be pinned for real overlap. */
int kmcb200_submit_bin(kmcb200_ctx* ctx, uint32_t slot, int32_t bin_id,
	const uint8_t* superkmers, uint64_t size, uint64_t n_rec, uint64_t n_plus_x_recs,
	const uint64_t* pack_bytes, const uint64_t* pack_recs, uint32_t n_packs,
	uint8_t* out_suffix, uint64_t out_capacity, uint64_t* lut);
int kmcb200_wait_bin(kmcb200_ctx* ctx, uint32_t slot, uint64_t* out_bytes, uint64_t stats[4]);

/* SURVEY 8f N4 - a device-friendly stage-1 output: kmcb200_submit_bin for a stage 1 that also hands over, per bin, the length byte `a` of
 * every record as a separate array (extras[n_super_kmers], stream order: the value CKmerBinCollector::PutExtendedKmer stores in front of the
 * record, kb_collector.cpp:60-66) and the number of records of every expander pack (pack_superkmers[n_packs]).  The record index is then two
 * parallel prefix sums per pack instead of the serial record walk; it is verified against the stream, a wrong array is KMCB200_ERR_BIN_FORMAT.
 * INTEGRATION.md shows the few lines a KMC collector needs for it. */
int kmcb200_submit_bin_indexed(kmcb200_ctx* ctx, uint32_t slot, int32_t bin_id,
	const uint8_t* superkmers, uint64_t size, uint64_t n_rec, const uint64_t* pack_bytes, uint32_t n_packs,
	const uint8_t* extras, uint64_t n_super_kmers, const uint32_t* pack_superkmers,
	uint8_t* out_suffix, uint64_t out_capacity, uint64_t* lut);

/* One bin over several GPUs (SURVEY 8f N2; the reference's analogue is RADULS' team sort of a big bucket, raduls_impl.h:672-745): for a bin
 * that is too large for a fair share of one GPU's time.  ctxs[0..n_ctx) are contexts with identical parameters on different (or, for
 * tests, the same) devices, none with a bin in flight; one host thread per GPU is started inside the call.  Every GPU gets a contiguous
 * share of the bin's packs from the host and counts its top 12 bits; the host cuts the key space into one range per GPU and the ranges into
 * key blocks; every GPU expands its share once, scattering the k-mers by key block; the records are exchanged with peer copies (NVLink:
 * an all-to-all of 8 B x n_rec x (N-1)/N); every GPU sorts and counts its own blocks.  Outputs are concatenated in key order:
 * byte-identical to kmcb200_process_bin on one GPU. */
int kmcb200_process_bin_multi(kmcb200_ctx* const* ctxs, uint32_t n_ctx, int32_t bin_id,
	const uint8_t* superkmers, uint64_t size, uint64_t n_rec, const uint64_t* pack_bytes, uint32_t n_packs,
	uint8_t* out_suffix, uint64_t out_capacity, uint64_t* out_bytes, uint64_t* lut, uint64_t stats[4]);

/* ---- database assembly without the reference's completer loop (SURVEY 8f N3; kmc_core/kb_completer.cpp:59-326) ------------------------
 * kmcb200_wait_bin_scanned = kmcb200_wait_bin, but the LUT arrives as the completer writes it to .kmc_pre: the exclusive prefix sum of the
 * bin's raw counts offset by lut_base (records preceding the bin in the file, kb_completer.cpp:191-201), computed on the GPU before the copy.
 * The writer owns a PINNED staging ring: kmcb200_db_reserve gives the region the next bin's records are copied into by the GPU (pass it as
 * out_suffix of kmcb200_submit_bin), kmcb200_db_commit_bin queues it for the writer thread (fwrite to .kmc_suf / .kmc_pre in commit order,
 * overlapping the GPU), kmcb200_db_close writes the footer of ProcessBinsSecondStage (:284-320).  For the same bins in the same order the
 * two files are byte-identical to the reference's. */
typedef struct kmcb200_db_writer kmcb200_db_writer;
typedef struct {
	uint32_t kmer_len, counter_size /* bytes */, lut_prefix_len, signature_len, cutoff_min, cutoff_max, both_strands;
} kmcb200_db_params;
int kmcb200_wait_bin_scanned(kmcb200_ctx* ctx, uint32_t slot, uint64_t lut_base, uint64_t* out_bytes, uint64_t stats[4]);
int kmcb200_db_open(const kmcb200_db_params* params, const char* path_prefix, uint64_t staging_bytes, kmcb200_db_writer** out_writer);
const char* kmcb200_db_last_error(const kmcb200_db_writer* w);
uint64_t kmcb200_db_records(const kmcb200_db_writer* w);           /* records committed so far = lut_base of the next bin */
int kmcb200_db_reserve(kmcb200_db_writer* w, uint64_t bytes, uint8_t** out_ptr);
int kmcb200_db_commit_bin(kmcb200_db_writer* w, uint64_t payload_bytes, const uint64_t* lut, int raw_lut, const uint64_t stats[4],
	const uint32_t* signatures, uint32_t n_signatures);
int kmcb200_db_close(kmcb200_db_writer* w, uint64_t totals[4]);

/* ---- stage 1: reads -> bins (SURVEY 8f N4: GPU super-k-mer splitting) -------------------------------------------------------------
 * The work of CSplitter::ProcessReads (kmc_core/splitter.cpp:557-677) and CKmerBinCollector::PutExtendedKmer (kb_collector.cpp:34-90) for
 * one batch of sequences, on the GPU.  A batch is one byte array: ACGTacgt are bases (splitter.cpp:43-47), every other byte ends the
 * current N-free segment, so reads are simply joined with one separator byte (e.g. '\n') between them.  Each sequence is treated as one
 * unsplit read (the reference cuts reads longer than mem_part_pmm_reads into overlapping parts, splitter.cpp:143-169: that adds
 * super-k-mer cuts but moves no k-mer to another bin).
 * Output: the bins' byte streams concatenated in bin order, the expander packs of all bins in bin order, and one fragment per bin.  Inside
 * a bin the records are in input order, byte for byte the stream of the reference run with one splitter thread.  In one batch's fragment
 * of a bin, the record that starts at byte s belongs to pack s / 65408: every pack starts on a record boundary, is non-empty and holds at
 * most 65536 bytes (so stage 2 walks every pack with one CTA).  A bin's stream over several batches is the concatenation of its fragments
 * in batch order, and so is its pack list; cut between reads, any batching gives the same bins as one batch.
 * The signature map is what CSignatureMapper::get_bin_id reads (s_mapper.h:263-266): 4^signature_len + 1 entries, the last one for the
 * special signature; every entry must be below n_bins.  A map read from a .kmc_pre (kb_completer.cpp:211-221, file positions of the bins)
 * reproduces the reference's file order when the bins are committed in order 0..n_bins-1.
 * The HBM workspace is allocated by kmcb200_splitter_create from max_batch_bytes (DESIGN.md section 3.8 gives its bytes per base).  Create
 * the splitter before the stage-2 contexts of the same GPU: kmcb200_create sizes its block limit from the HBM that is free at that moment. */
#define KMCB200_SPLIT_MAX_BINS 4096
#define KMCB200_SPLIT_MAX_BATCH (1ull << 31)
typedef struct kmcb200_splitter kmcb200_splitter;
typedef struct {
	uint32_t kmer_len;                    /* Params.kmer_len: signature_len+1 .. KMCB200_MAX_KMER_LEN */
	uint32_t signature_len;               /* Params.signature_len (-p): 5..11 */
	uint32_t n_bins;                      /* 1..KMCB200_SPLIT_MAX_BINS; every map value is < n_bins (the special signature maps like any other) */
	int32_t device;                       /* CUDA ordinal */
	uint64_t max_batch_bytes;             /* largest batch one call accepts (1..KMCB200_SPLIT_MAX_BATCH): sizes the workspace */
} kmcb200_split_params;
typedef struct {
	uint64_t byte_off;                    /* offset of the bin's bytes in the output */
	uint64_t bytes;                       /* size of the bin's stream in this batch */
	uint64_t n_rec;                       /* k-mers (CBinDesc n_rec, kb_collector.cpp:74) */
	uint64_t n_super_kmers;               /* records */
	uint32_t pack0, n_packs;              /* the bin's packs: pack_bytes[pack0 .. pack0 + n_packs) */
} kmcb200_bin_fragment;

/* KMCB200_ERR_INVALID for a bad parameter or a map value >= n_bins, KMCB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback). */
int kmcb200_splitter_create(const kmcb200_split_params* params, const uint32_t* signature_map /* host, 4^signature_len + 1 */, kmcb200_splitter** out);
void kmcb200_splitter_destroy(kmcb200_splitter* sp);
/* message of the last failure on this splitter (or of the last failed kmcb200_splitter_create when sp == NULL) */
const char* kmcb200_splitter_last_error(const kmcb200_splitter* sp);
/* Host buffers: copies the batch in and returns when out[0, *out_bytes), pack_bytes[0, *n_packs) and frags[n_bins] are filled.  When
 * out_capacity or pack_capacity is too small: KMCB200_ERR_CAPACITY, *out_bytes / *n_packs give the required sizes, nothing else is written.
 * For raw FASTQ / FASTA bytes instead of a batch, see kmcb200_split_fastx ("reads text -> batch" below). */
int kmcb200_split(kmcb200_splitter* sp, const uint8_t* seq, uint64_t bytes,
	uint8_t* out, uint64_t out_capacity, uint64_t* out_bytes,
	uint64_t* pack_bytes, uint64_t pack_capacity, uint64_t* n_packs, kmcb200_bin_fragment* frags);
/* Device twin: every pointer is a device pointer, the work is queued on `stream` (a cudaStream_t; NULL = the legacy default stream).
 * d_result receives 5 x uint64: [0] output bytes, [1] packs, [2] 1 when a capacity was too small (then only d_result is written: the
 * required sizes), [3] records (super-k-mers), [4] k-mers.  d_frags[n_bins] as in kmcb200_split.  Stage 2's device entry points read a
 * bin 32 bytes past its end: give d_out that much slack when its bins go to kmcb200_dev_process_bin in place. */
int kmcb200_dev_split(kmcb200_splitter* sp, const uint8_t* d_seq, uint64_t bytes, uint8_t* d_out, uint64_t out_capacity,
	uint64_t* d_pack_bytes, uint64_t pack_capacity, kmcb200_bin_fragment* d_frags, uint64_t* d_result, void* stream);
/* Number of kernels this splitter has launched so far. */
uint64_t kmcb200_splitter_kernel_launches(const kmcb200_splitter* sp);
/* Opt-in: from now on every split also adds, per bin, the (k+x)-mer count of its records that CKmerBinCollector keeps in n_plus_x_recs
 * (kb_collector.cpp:73-89) with max_x = k % 32 ? min(31 - k % 32, 3) : 0 (kmc.h:139-142): 1 + (n - k) / (max_x + 1) per record of n
 * symbols when both_strands == 0, the collector's strand-state walk (kb_collector.h:66-116) when it is 1; nothing when max_x = 0.  This
 * is what kmcb200_stage2_bin_order needs.  The call zeroes the totals; a split that ends in KMCB200_ERR_CAPACITY (or a capacity flag on
 * the device) adds nothing.  One more kernel per split; a splitter that never calls this launches and writes exactly as before. */
int kmcb200_splitter_count_kxmers(kmcb200_splitter* sp, int both_strands);
/* per_bin[n_bins]: the totals since kmcb200_splitter_count_kxmers (waits for the device's queued work).  KMCB200_ERR_INVALID when the
 * counting was never enabled. */
int kmcb200_splitter_kxmer_totals(kmcb200_splitter* sp, uint64_t* per_bin);
/* Homopolymer compression (`kmc -hc`, CSplitter::HomopolymerCompressSeq, splitter.cpp:424-435), opt-in, on (1) or off (0) for the calls
 * that follow.  While it is on, every batch entry point of the handle (the host batch, the device twin, the raw-chunk form after its
 * parse) first compresses the batch on the device: a byte of ACGTacgt that repeats the base before it, ignoring case, is dropped, and the
 * result is padded back to the batch's length with '\n' (no k-mer, record or count comes from a separator).  Runs never cross a
 * separator, so each read is compressed on its own, as in the reference; the caller's batch is read and never written, and *consumed /
 * *seq_bytes keep their meaning (the parsed batch).  Work: 3 more kernel launches per call with a non-empty batch, no host
 * synchronisation.  Workspace: 1 B per byte of max_batch_bytes plus 8 B per 16 KiB, allocated the first time compression is turned on
 * and kept until the handle is destroyed; a handle that never turns it on allocates, launches and writes exactly as without this call.
 * The same call exists for the signature statistics and the small-k counter.  The histogram estimator has none: the reference never
 * compresses the reads it estimates from (`kmc -e -hc` writes the file `kmc -e` writes). */
int kmcb200_splitter_set_homopolymer_compressed(kmcb200_splitter* sp, int on);

/* ---- stage 0: signature statistics (CKMC::buildSignatureMapping, kmc_core/kmc.h:974-1075) ----------------------------------------
 * Before it splits, the reference counts the k-mers of every signature over a sample of the input (CSplitter::CalcStats,
 * splitter.cpp:439-533) and groups the signatures into n_bins bins by those counts (CSignatureMapper::Init, s_mapper.h:141-235).  After
 * the split, its stage 2 with one thread (-sr1) reads the bins in descending order of their memory need (CBinDesc::get_sorted_req_sizes,
 * queues.h:499-558), and that order is the bins' order in the database and the value the .kmc_pre map stores for their signatures.
 *   kmcb200_sigstats_*        the statistics on the GPU; the batch format is kmcb200_split's (every byte other than ACGTacgt separates);
 *                             counts[sig] += 1 for every k-mer of ACGT only, sig = its least normalised m-mer (4^m: the special signature),
 *                             accumulated over calls until reset, 32-bit counters that wrap like the reference's.  Workspace: the batch
 *                             (max_batch_bytes, host path) and the 4^m + 1 counters; nothing per base.
 *   kmcb200_signature_map     Init on the host: map[sig] = bin id, -1 for a signature that is not allowed (no k-mer ever has it; the
 *                             completer stores 0 for it).  Needs no device.
 *   kmcb200_stage2_bin_order  get_sorted_req_sizes + get_req_size on the host: file_pos[bin] = the bin's position in the database.  bytes,
 *                             n_rec and n_plus_x_recs are per bin over the whole input (kmcb200_bin_fragment's bytes / n_rec summed,
 *                             kmcb200_splitter_kxmer_totals; n_plus_x_recs may be NULL when k % 32 == 0).  Needs no device.
 * Host-function failures leave their message in kmcb200_sigstats_last_error(NULL). */
typedef struct kmcb200_sigstats kmcb200_sigstats;
typedef struct {
	uint32_t kmer_len;                    /* signature_len+1 .. KMCB200_MAX_KMER_LEN */
	uint32_t signature_len;               /* 5..11 */
	int32_t device;                       /* CUDA ordinal */
	uint32_t reserved;                    /* 0 */
	uint64_t max_batch_bytes;             /* largest batch one call accepts (1..KMCB200_SPLIT_MAX_BATCH) */
} kmcb200_sigstats_params;
/* KMCB200_ERR_INVALID for a bad parameter, KMCB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback).  The counters start at 0. */
int kmcb200_sigstats_create(const kmcb200_sigstats_params* params, kmcb200_sigstats** out);
void kmcb200_sigstats_destroy(kmcb200_sigstats* h);
/* message of the last failure on this handle (or of the last failed create / host function when h == NULL) */
const char* kmcb200_sigstats_last_error(const kmcb200_sigstats* h);
/* Host batch: copied in, counted; returns when the batch buffer may be reused.  A batch over max_batch_bytes: KMCB200_ERR_INVALID. */
int kmcb200_sigstats_add(kmcb200_sigstats* h, const uint8_t* seq, uint64_t bytes);
/* Device twin: d_seq in HBM, queued on `stream` (a cudaStream_t; NULL = the legacy default stream) after the handle's earlier work. */
int kmcb200_dev_sigstats_add(kmcb200_sigstats* h, const uint8_t* d_seq, uint64_t bytes, void* stream);
/* counts[4^signature_len + 1] (host) after every call queued so far, device twin included. */
int kmcb200_sigstats_read(kmcb200_sigstats* h, uint32_t* counts);
int kmcb200_sigstats_reset(kmcb200_sigstats* h);
/* Number of kernels this handle has launched so far. */
uint64_t kmcb200_sigstats_kernel_launches(const kmcb200_sigstats* h);
/* Homopolymer compression before the statistics, as kmcb200_splitter_set_homopolymer_compressed describes (CSplitter::CalcStats,
 * splitter.cpp:457-458): 3 more launches per non-empty batch. */
int kmcb200_sigstats_set_homopolymer_compressed(kmcb200_sigstats* h, int on);
/* map[4^signature_len + 1].  KMCB200_ERR_INVALID: signature_len outside 5..11, n_bins outside 2..KMCB200_SPLIT_MAX_BINS (one bin besides
 * the special signature's is needed), or counts for which the rule would hand out an id >= n_bins. */
int kmcb200_signature_map(const uint32_t* counts, uint32_t signature_len, uint32_t n_bins, int32_t* map);
/* file_pos[n_bins]: a permutation of 0..n_bins-1.  cutoff_max / counter_max as the database's parameters; records are 8 * ceil(k / 32) bytes
 * (sizeof(CKmer<SIZE>)) and every buffer is rounded to 256 bytes (ALIGNMENT), as in the reference. */
int kmcb200_stage2_bin_order(uint32_t n_bins, const uint64_t* bytes, const uint64_t* n_rec, const uint64_t* n_plus_x_recs, uint32_t kmer_len,
	uint32_t cutoff_min, uint64_t cutoff_max, uint64_t counter_max, uint32_t lut_prefix_len, uint32_t* file_pos);

/* ---- reads text -> batch: FASTQ / FASTA parsed on the GPU ------------------------------------------------------------------------
 * kmcb200_split and kmcb200_sigstats_add take batches in which every non-ACGT byte separates; raw FASTQ cannot be passed as it is (quality
 * lines hold A, C, G, T), nor FASTA (headers hold letters).  This parser makes that batch from raw file bytes on the GPU, one chunk at a
 * time, byte for byte what kmc_b200.reads.sequences_to_batch makes of the whole file (the chunks' outputs, concatenated):
 *   FASTQ  line 1 of every 4 is kept with its '\n'; lines are counted from the chunk's start, so every chunk must start on a record;
 *   FASTA  a header line (first byte '>') becomes one '\n', every other line is kept without its '\n', blank lines vanish.
 * '\r' is an ordinary byte (a separator in the batch).  A final chunk that does not end in '\n' is parsed as if it did, so the output
 * never exceeds bytes + 1.  The format is the caller's choice (the file's first non-empty line starts with '@' or '>'); the parser reads
 * text only: gzip input is inflated before it (see "gzip input" below).
 * Records end after every 4th line (FASTQ) or where a header line starts after a '\n' (FASTA); the end of a final chunk ends one too.
 *   is_final == 0  the chunk is parsed up to its last record end, returned as `consumed`: the caller carries the rest into the next chunk.
 *                  A chunk without a record end is KMCB200_ERR_INVALID ("a record is longer than the chunk") and nothing else is written.
 *   limit < bytes  only the records that start before `limit` are parsed: the cut is the first record end at or past `limit` (where the
 *                  chunk has one; a non-final chunk without one is parsed to its last record end, so consumed < limit says "go on").
 *                  KMCB200_FASTX_NO_LIMIT (or any limit >= bytes): no cut.
 * Work per call: 9 kernel launches whatever the size, no host synchronisation inside (consumed, the cut and the error are decided on the
 * device).  Workspace: the chunk and the output of the host-buffer form (2 B per byte of max_chunk_bytes) plus 120 B per 16 KiB tile.
 *
 * BAM (`kmc -fbam`, CSplitter::GetSeq, kmc_core/splitter.cpp:326-418): the chunk is *decompressed* BAM record bytes that start on a record
 * (the caller inflates the BGZF members and skips the header: magic, l_text, text, n_ref and the references).  A record's bytes may be
 * split across calls only through `consumed` and the caller's carry, as for FASTQ.
 *   KMCB200_BAM                  every record whose FLAG has neither 0x100 (secondary) nor 0x800 (supplementary) becomes its l_seq SEQ
 *                                bases as stored, A C G T for the codes 1 2 4 8 and N for every other code ('=' and IUPAC codes
 *                                included), then one '\n'; other records add nothing.  What `kmc -fbam` counts.
 *   KMCB200_BAM_ORIGINAL_STRAND  the same, with the records of FLAG 0x10 reverse complemented back to their original strand: what
 *                                `kmc -b -fbam` counts.
 * A record is at least 36 + ceil(l_seq / 2) + l_seq bytes, so the output never exceeds `bytes`; d_result[2] counts the kept records.
 * Record ends are the ends of BAM records; is_final, limit and consumed mean what they mean above, except that a final chunk that ends
 * inside a record has no implicit terminator.  A nonzero d_result[3] (then [0..2] are 0 and d_seq is not written; the host forms return
 * KMCB200_ERR_INVALID) is 1: a non-final chunk without a whole record; 2: a final chunk that ends inside a record (truncated); 3: a
 * malformed record, block_size < 32, l_seq < 0, or 32 + l_read_name + 4 * n_cigar_op + ceil(l_seq / 2) + l_seq > block_size.
 * Work per call: 7 kernel launches whatever the size, no host synchronisation inside.  The record walk is parallel where each 16 KiB
 * tile's guessed first record holds; records that defeat the guesses (no NUL-terminated name, or crafted contents) are walked serially,
 * about 0.5 us per record on an H100 (DESIGN.md section 3.15).  Workspace: as above, plus 16 B per 36 B of
 * max_chunk_bytes (0.45 B per byte) for the kept records' starts and output offsets, allocated for a BAM parser only. */
#define KMCB200_FASTQ 1
#define KMCB200_FASTA 2
/* 3 is not a format: it stays refused, as it was before the BAM formats */
#define KMCB200_BAM 4
#define KMCB200_BAM_ORIGINAL_STRAND 5
#define KMCB200_FASTX_NO_LIMIT (~0ull)
typedef struct kmcb200_fastx kmcb200_fastx;
typedef struct {
	int32_t device;                       /* CUDA ordinal */
	uint32_t format;                      /* KMCB200_FASTQ, KMCB200_FASTA, KMCB200_BAM or KMCB200_BAM_ORIGINAL_STRAND */
	uint64_t max_chunk_bytes;             /* largest chunk one call accepts (1..KMCB200_SPLIT_MAX_BATCH): sizes the workspace */
} kmcb200_fastx_params;
/* KMCB200_ERR_INVALID for a bad parameter, KMCB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback). */
int kmcb200_fastx_create(const kmcb200_fastx_params* params, kmcb200_fastx** out);
void kmcb200_fastx_destroy(kmcb200_fastx* p);
/* message of the last failure on this parser (or of the last failed create when p == NULL) */
const char* kmcb200_fastx_last_error(const kmcb200_fastx* p);
/* Number of kernels this parser has launched so far (the _fastx entry points below count theirs here too). */
uint64_t kmcb200_fastx_kernel_launches(const kmcb200_fastx* p);
/* Records parsed by the latest host-buffer call on this parser (kmcb200_fastx_parse or a _fastx entry point below): d_result[2]. */
uint64_t kmcb200_fastx_last_records(const kmcb200_fastx* p);
/* Host buffers: copies the chunk in, returns when seq[0, *seq_bytes) holds the batch and *consumed the bytes parsed.  When the batch is
 * longer than seq_capacity: KMCB200_ERR_CAPACITY, *consumed / *seq_bytes are set and seq is not written. */
int kmcb200_fastx_parse(kmcb200_fastx* p, const uint8_t* raw, uint64_t bytes, int is_final, uint64_t limit,
	uint8_t* seq, uint64_t seq_capacity, uint64_t* consumed, uint64_t* seq_bytes);
/* Device twin: d_raw / d_seq / d_result in HBM, queued on `stream` (a cudaStream_t; NULL = the legacy default stream).  seq_capacity
 * must be at least bytes + 1 (KMCB200_ERR_INVALID otherwise).  d_result receives 4 x uint64: [0] consumed, [1] sequence bytes, [2] records
 * parsed, [3] 1 when a non-final chunk has no record end, for BAM also 2 or 3 as above (then [0..2] are 0 and d_seq is not written). */
int kmcb200_dev_fastx_parse(kmcb200_fastx* p, const uint8_t* d_raw, uint64_t bytes, int is_final, uint64_t limit,
	uint8_t* d_seq, uint64_t seq_capacity, uint64_t* d_result, void* stream);
/* kmcb200_split of a raw chunk: copies it in and parses it straight into the splitter's batch buffer, then continues exactly like
 * kmcb200_split from the size phase on (same outputs, same capacity rule).  *consumed as for kmcb200_fastx_parse; *seq_bytes (may be
 * NULL) the batch's length.  bytes + 1 > max_batch_bytes: KMCB200_ERR_INVALID.  Errors are reported on the splitter. */
int kmcb200_split_fastx(kmcb200_splitter* sp, kmcb200_fastx* p, const uint8_t* raw, uint64_t bytes, int is_final,
	uint8_t* out, uint64_t out_capacity, uint64_t* out_bytes, uint64_t* pack_bytes, uint64_t pack_capacity, uint64_t* n_packs,
	kmcb200_bin_fragment* frags, uint64_t* consumed, uint64_t* seq_bytes);
/* kmcb200_sigstats_add of a raw chunk, the same way, with the parse's limit (the statistics' sample ends on a record).  bytes + 1 >
 * max_batch_bytes: KMCB200_ERR_INVALID.  Errors are reported on the statistics handle. */
int kmcb200_sigstats_add_fastx(kmcb200_sigstats* h, kmcb200_fastx* p, const uint8_t* raw, uint64_t bytes, int is_final, uint64_t limit,
	uint64_t* consumed);

/* ---- small k: reads -> direct counts -> KMC1 database (KMC's small-k mode, kmc_core/kmc.h:677-960) -------------------------------
 * For k <= 13 the reference builds no bins: it counts every k-mer in a direct array of 4^k uint64 counters (CSplitter::ProcessReadsSmallK,
 * splitter.cpp:681-805) and writes a KMC1-format database from it (CSmallKCompleter::CompleteKMCFormat, kb_completer.h:148-308).
 *   counting  the batch format is kmcb200_split's; every k-mer of ACGT only adds 1 to counts[v], v = its 2k-bit code (first symbol most
 *             significant), or min(code, reverse complement) with both strands.  Counts add up over calls until reset.
 *   finish    n_unique (non-zero counters), n_cutoff_min (count < cutoff_min), n_cutoff_max (count > cutoff_max), n_total (sum of the
 *             counts), and the LUT prefix length lp of 1..15 with (k - lp) % 4 == 0 of least n_unique * ((k - lp) / 4 + calc_counter_size)
 *             + 8 * 4^lp (kmc.h:906-936).  Records are (k - lp) / 4 suffix bytes (most significant first) and min(count, counter_max) in
 *             counter_size bytes (least significant first), counter_size = calc_counter_size_ull (defs.h:161), 0 when counter_max == 1.
 *   emit      the records of the kept k-mers in k-mer order, and lut[4^lp]: lut[p] = kept k-mers whose prefix is below p (no sentinel).
 *   write_db  finish + emit + the two files: .kmc_suf "KMCS" records "KMCS"; .kmc_pre "KMCP" lut, the KMC1 footer (version word 0, no
 *             signature map) and "KMCP".
 * Work: 1 launch per add, 4 per finish (one synchronisation), 1 per emit.  Workspace: the batch (max_batch_bytes, host path), the 4^k
 * counters (512 MiB at k = 13), one word per 4096 counters, and the records and LUT of an emit. */
typedef struct kmcb200_smallk kmcb200_smallk;
typedef struct {
	uint32_t kmer_len;                    /* 1..13 */
	uint32_t both_strands;                /* 1: canonical k-mers, 0: as they are (-b) */
	int32_t device;                       /* CUDA ordinal */
	uint32_t reserved;                    /* 0 */
	uint64_t max_batch_bytes;             /* largest batch one call accepts (1..KMCB200_SPLIT_MAX_BATCH) */
} kmcb200_smallk_params;
/* KMCB200_ERR_INVALID for a bad parameter, KMCB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback).  The counters start at 0. */
int kmcb200_smallk_create(const kmcb200_smallk_params* params, kmcb200_smallk** out);
void kmcb200_smallk_destroy(kmcb200_smallk* h);
/* message of the last failure on this handle (or of the last failed create when h == NULL) */
const char* kmcb200_smallk_last_error(const kmcb200_smallk* h);
/* Number of kernels this handle has launched so far. */
uint64_t kmcb200_smallk_kernel_launches(const kmcb200_smallk* h);
/* Homopolymer compression before the count, as kmcb200_splitter_set_homopolymer_compressed describes (CSplitter::ProcessReadsSmallK,
 * splitter.cpp:702-703, 757-758): 3 more launches per non-empty batch. */
int kmcb200_smallk_set_homopolymer_compressed(kmcb200_smallk* h, int on);
/* Host batch: copied in, counted; returns when the batch buffer may be reused.  A batch over max_batch_bytes: KMCB200_ERR_INVALID. */
int kmcb200_smallk_add(kmcb200_smallk* h, const uint8_t* seq, uint64_t bytes);
/* Device twin: d_seq in HBM, queued on `stream` (a cudaStream_t; NULL = the legacy default stream) after the handle's earlier work. */
int kmcb200_dev_smallk_add(kmcb200_smallk* h, const uint8_t* d_seq, uint64_t bytes, void* stream);
/* kmcb200_smallk_add of a raw FASTQ / FASTA chunk parsed on the GPU straight into the handle's batch buffer (see kmcb200_fastx_parse for
 * is_final and *consumed; *seq_bytes, which may be NULL, receives the batch's length).  bytes + 1 > max_batch_bytes:
 * KMCB200_ERR_INVALID.  Errors are reported on the counter handle. */
int kmcb200_smallk_add_fastx(kmcb200_smallk* h, kmcb200_fastx* p, const uint8_t* raw, uint64_t bytes, int is_final, uint64_t* consumed,
	uint64_t* seq_bytes);
/* counts[4^k] (host) after every call queued so far, device twin included. */
int kmcb200_smallk_read(kmcb200_smallk* h, uint64_t* counts);
int kmcb200_smallk_reset(kmcb200_smallk* h);
/* The totals and the layout of the database of the current counts: *lut_prefix_len, *counter_size, *suffix_bytes (the bytes of all the
 * records), stats[4] = n_unique, n_cutoff_min, n_cutoff_max, n_total.  A k-mer is kept when cutoff_min <= count <= cutoff_max. */
int kmcb200_smallk_finish(kmcb200_smallk* h, uint32_t cutoff_min, uint64_t cutoff_max, uint64_t counter_max, uint32_t* lut_prefix_len,
	uint32_t* counter_size, uint64_t* suffix_bytes, uint64_t* stats);
/* After finish (and no add or reset since): suffix[0, suffix_bytes) the records, lut[4^lut_prefix_len] the LUT.  capacity < suffix_bytes:
 * KMCB200_ERR_CAPACITY and nothing is written; no finish: KMCB200_ERR_INVALID. */
int kmcb200_smallk_emit(kmcb200_smallk* h, uint8_t* suffix, uint64_t capacity, uint64_t* lut);
/* finish + emit + path_prefix.kmc_pre / path_prefix.kmc_suf; totals[4] as finish's stats. */
int kmcb200_smallk_write_db(kmcb200_smallk* h, const char* path_prefix, uint32_t cutoff_min, uint64_t cutoff_max, uint64_t counter_max,
	uint64_t* totals);

/* ---- histogram estimation (KMC's CntHashEstimator, kmc_core/libs/ntHash/ntHashWrapper.h:97-454: `kmc -e`, `kmc --opt-out-size`) --------
 * The batch format is kmcb200_split's; every k-mer of ACGT only is hashed with canonical ntHash, h = min(fh, rh) (64 bits), and sampled:
 * counters[0][h mod 2^27] += 1 when h >> (63 - s) == 1, counters[1][h mod 2^27] += 1 when h >> (64 - s) == 2^(s-1) - 1 (two tables of
 * 2^27 uint32).  The counters are a function of the multiset of k-mers alone, and add up over calls until reset.
 *   histogram  max_occ = min(max(largest counter, 2), 65536); hist[0..max_occ] the reference's EstimateHistogram of the two tables'
 *              histograms of min(65536, counter): hist[i] estimates the number of distinct k-mers that occur i times, hist[0] = 0.  The
 *              recursion, O(max_occ^2) in double, runs on the host in the reference's order of operations.
 * `kmc` takes s = 7, or 11 when the input files hold at least 5 * 10^10 bytes (kmc.h:1118-1121).
 * Work: 1 launch per add, 1 per histogram (one synchronisation).  Workspace: the batch (max_batch_bytes, host path) and 1 GiB of counters. */
#define KMCB200_ESTIMATE_MAX_KMER_LEN 256
typedef struct kmcb200_estimator kmcb200_estimator;
typedef struct {
	uint32_t kmer_len;                    /* 1..KMCB200_ESTIMATE_MAX_KMER_LEN */
	uint32_t s;                           /* 7 or 11 */
	int32_t device;                       /* CUDA ordinal */
	uint32_t reserved;                    /* 0 */
	uint64_t max_batch_bytes;             /* largest batch one call accepts (1..KMCB200_SPLIT_MAX_BATCH) */
} kmcb200_estimator_params;
/* KMCB200_ERR_INVALID for a bad parameter, KMCB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback).  The counters start at 0. */
int kmcb200_estimator_create(const kmcb200_estimator_params* params, kmcb200_estimator** out);
void kmcb200_estimator_destroy(kmcb200_estimator* h);
/* message of the last failure on this handle (or of the last failed create when h == NULL) */
const char* kmcb200_estimator_last_error(const kmcb200_estimator* h);
/* Number of kernels this handle has launched so far. */
uint64_t kmcb200_estimator_kernel_launches(const kmcb200_estimator* h);
/* Host batch: copied in, hashed; returns when the batch buffer may be reused.  A batch over max_batch_bytes: KMCB200_ERR_INVALID. */
int kmcb200_estimator_add(kmcb200_estimator* h, const uint8_t* seq, uint64_t bytes);
/* Device twin: d_seq in HBM, queued on `stream` (a cudaStream_t; NULL = the legacy default stream) after the handle's earlier work. */
int kmcb200_dev_estimator_add(kmcb200_estimator* h, const uint8_t* d_seq, uint64_t bytes, void* stream);
/* kmcb200_estimator_add of a raw FASTQ / FASTA chunk parsed on the GPU straight into the handle's batch buffer (see kmcb200_fastx_parse for
 * is_final and *consumed; *seq_bytes and *n_records, which may be NULL, receive the batch's length and the records parsed).  bytes + 1 >
 * max_batch_bytes: KMCB200_ERR_INVALID.  Errors are reported on the estimator. */
int kmcb200_estimator_add_fastx(kmcb200_estimator* h, kmcb200_fastx* p, const uint8_t* raw, uint64_t bytes, int is_final, uint64_t* consumed,
	uint64_t* seq_bytes, uint64_t* n_records);
/* counters[2 * 2^27] (host): table 0, then table 1, after every call queued so far, device twin included. */
int kmcb200_estimator_read(kmcb200_estimator* h, uint32_t* counters);
/* *n = max_occ + 1 and hist[0, *n) the estimate of the current counters.  capacity < *n: KMCB200_ERR_CAPACITY, *n set, hist not written. */
int kmcb200_estimator_histogram(kmcb200_estimator* h, uint64_t* hist, uint64_t capacity, uint64_t* n);
int kmcb200_estimator_reset(kmcb200_estimator* h);

/* ---- gzip input: BGZF members inflated on the GPU (RFC 1951 / 1952; what `bgzip` and `samtools` write) ------------------------------
 * A BGZF file is a series of independent gzip members: ID1 ID2 = 1f 8b, CM = 8, FLG = FEXTRA alone, an extra field with a 'BC' subfield
 * (SLEN 2) that holds BSIZE (the member's bytes - 1), the deflate data, then CRC32 and ISIZE (its text bytes, at most 64 KiB).  Every member
 * is inflated by one warp on its own (kmc_b200/csrc/inflate.cuh), so a call that holds thousands of members keeps the GPU busy.  Any
 * other gzip stream (plain `gzip`, `pigz`) is one serial stream: kmc_b200.reads inflates those with zlib on its reader thread.
 * The text is zlib's byte for byte.  A malformed member (invalid codes or code sets, a distance before the member's start, more or less
 * output than ISIZE, a CRC32 mismatch, a truncated stream, ...) makes the call KMCB200_ERR_INVALID with the member's offset in the
 * message, and no text of that call is handed on.  No zlib is linked. */
typedef struct {
	uint64_t in_off;                      /* the member's first byte in the compressed buffer */
	uint64_t out_off;                     /* its first text byte: the exclusive sum of the ISIZEs before it */
	uint32_t in_bytes;                    /* BSIZE + 1 */
	uint32_t isize;                       /* its text bytes (the trailer's ISIZE) */
} kmcb200_bgzf_member;
/* The member walk, host only (no device needed): takes whole BGZF members from raw[0] on while their ISIZE sum fits text_capacity (and, when
 * members is not NULL, while fewer than members_capacity are taken), and stops before a partial member, a non-BGZF member or one whose ISIZE
 * is over 64 KiB.  *consumed: the compressed bytes of the members taken, *text_bytes: their text bytes, *n_members: how many; members[0, n)
 * their table.  KMCB200_ERR_INVALID (message in kmcb200_gunzip_last_error(NULL)) when the first member is not BGZF. */
int kmcb200_bgzf_scan(const uint8_t* raw, uint64_t bytes, uint64_t text_capacity, kmcb200_bgzf_member* members, uint64_t members_capacity,
	uint64_t* consumed, uint64_t* text_bytes, uint64_t* n_members);
typedef struct kmcb200_gunzip kmcb200_gunzip;
typedef struct {
	int32_t device;                       /* CUDA ordinal */
	uint32_t reserved;                    /* 0 */
	uint64_t max_in_bytes;                /* largest compressed buffer one call accepts (1..KMCB200_SPLIT_MAX_BATCH) */
	uint64_t max_out_bytes;               /* largest text one call makes (1..KMCB200_SPLIT_MAX_BATCH) */
} kmcb200_gunzip_params;
/* KMCB200_ERR_INVALID for a bad parameter, KMCB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback).  Workspace: max_in_bytes +
 * max_out_bytes in HBM, and a member table of 24 B per 28 B of max_in_bytes in HBM and in pinned host memory. */
int kmcb200_gunzip_create(const kmcb200_gunzip_params* params, kmcb200_gunzip** out);
void kmcb200_gunzip_destroy(kmcb200_gunzip* p);
/* message of the last failure on this inflater (or of the last failed create or kmcb200_bgzf_scan when p == NULL) */
const char* kmcb200_gunzip_last_error(const kmcb200_gunzip* p);
/* Number of kernels this inflater has launched so far (one per call that holds a member). */
uint64_t kmcb200_gunzip_kernel_launches(const kmcb200_gunzip* p);
/* Host buffers: the members kmcb200_bgzf_scan takes from raw[0, bytes) with min(text_capacity, max_out_bytes) are copied in, inflated on the
 * inflater's own stream, and their text copied to text[0, *text_bytes); *consumed: their compressed bytes (0 and 0: not one whole member
 * fits).  bytes > max_in_bytes or a first member that is not BGZF: KMCB200_ERR_INVALID.  A malformed member: KMCB200_ERR_INVALID, *consumed
 * = *text_bytes = 0 and text is not written. */
int kmcb200_gunzip_inflate(kmcb200_gunzip* p, const uint8_t* raw, uint64_t bytes, uint8_t* text, uint64_t text_capacity, uint64_t* consumed,
	uint64_t* text_bytes);
/* Device twin: d_members[0, n_members) (a kmcb200_bgzf_scan table, copied to HBM), d_raw[0, raw_bytes) and d_text[0, text_capacity) in
 * HBM, queued on `stream` (a cudaStream_t; NULL = the legacy default stream) with no host synchronisation.  *d_error (HBM) receives ~0 when
 * every member is good, else min over the bad members of (member index << 8 | error code); the table is checked against raw_bytes and
 * text_capacity in the kernel. */
int kmcb200_dev_gunzip_inflate(kmcb200_gunzip* p, const kmcb200_bgzf_member* d_members, uint64_t n_members, const uint8_t* d_raw, uint64_t raw_bytes,
	uint8_t* d_text, uint64_t text_capacity, uint64_t* d_error, void* stream);

/* ---- KMC database input (`kmc -fkmc`): .kmc_suf records decoded on the GPU into k-mer reads ----------------------------------------
 * What the reference reads from a KMC database (CBinaryFilesReader::ProcessKMC through CKMCFile::ReadNextKmer, kmc_api/kmc_file.cpp:427-499):
 * every record whose counter passes the database's cutoffs becomes one read, its k-mer.  A chunk is n_records whole records of .kmc_suf
 * (after the "KMCS" marker), (k - lut_prefix_len) / 4 suffix bytes, most significant symbol first, then counter_size bytes, little-endian;
 * first_record is the index of its first record in the file.  The batch is, per kept record in file order, its k symbols in ACGT and one
 * '\n': the batch format of the splitter, the small-k counter and the estimator.
 *   prefix    record g's lut_prefix_len leading symbols are #{ j >= 1 : lut[j] <= g } & (4^lut_prefix_len - 1) (the reference's listing
 *             reader, CPrefixFileBufferForListingMode::GetPrefix).  `lut` is the LUT as that reader sees it: for a KMC2 database all its
 *             n_bins * 4^lut_prefix_len + 1 stored words, for a KMC1 database its 4^lut_prefix_len stored words followed by total_kmers
 *             (kmc_file.h:57-58).  It stays in HBM for the handle's lifetime and must be non-decreasing.
 *   filter    counter_size 0: every record is kept.  Otherwise the counter, accumulated into a uint32, must lie in [min_count, max_count]
 *             (the header's cutoffs; for KMC1 max_count is the 64-bit value of the header's two words).
 * Work per call: 5 kernel launches whatever the size (count, a 3-launch scan, decode), no host synchronisation inside the device form.
 * Workspace: the LUT, plus max_records * (record bytes + k + 1) bytes for the host-buffer form's chunk and output. */
typedef struct kmcb200_kmcdb kmcb200_kmcdb;
typedef struct {
	int32_t device;                       /* CUDA ordinal */
	uint32_t kmer_len;                    /* the database's k, 1..256 */
	uint32_t lut_prefix_len;              /* 0..16, at most k, with (k - lut_prefix_len) % 4 == 0 */
	uint32_t counter_size;                /* 0..4 (5..8 is KMCB200_ERR_INVALID: the reference's uint32 accumulation is undefined there) */
	uint64_t min_count, max_count;        /* the header's cutoffs */
	uint64_t total_kmers;                 /* records in .kmc_suf */
	uint64_t max_records;                 /* largest chunk one call takes (1..KMCB200_SPLIT_MAX_BATCH / (k + 1)): sizes the workspace */
} kmcb200_kmcdb_params;
/* lut[0, lut_entries) as described above is copied to HBM.  KMCB200_ERR_INVALID for a bad parameter, KMCB200_ERR_NO_DEVICE without an
 * sm_90 device (no CPU fallback). */
int kmcb200_kmcdb_create(const kmcb200_kmcdb_params* params, const uint64_t* lut, uint64_t lut_entries, kmcb200_kmcdb** out);
void kmcb200_kmcdb_destroy(kmcb200_kmcdb* d);
const char* kmcb200_kmcdb_last_error(const kmcb200_kmcdb* d);
/* Number of kernels this decoder has launched so far (the _kmcdb entry points below count theirs here too). */
uint64_t kmcb200_kmcdb_kernel_launches(const kmcb200_kmcdb* d);
/* Host buffers: copies the records in, returns when seq[0, *seq_bytes) holds the batch and *kept (optional) the records kept.  n_records
 * above max_records or first_record + n_records above total_kmers: KMCB200_ERR_INVALID.  A batch longer than capacity:
 * KMCB200_ERR_CAPACITY, *seq_bytes / *kept are set and seq is not written. */
int kmcb200_kmcdb_decode(kmcb200_kmcdb* d, const uint8_t* suffix, uint64_t n_records, uint64_t first_record, uint8_t* seq, uint64_t capacity,
	uint64_t* seq_bytes, uint64_t* kept);
/* Device twin: d_suffix / d_seq / d_result in HBM, queued on `stream` (a cudaStream_t; NULL = the legacy default stream).  d_result receives
 * 2 x uint64: [0] sequence bytes, [1] kept records; when [0] exceeds capacity d_seq is not written. */
int kmcb200_dev_kmcdb_decode(kmcb200_kmcdb* d, const uint8_t* d_suffix, uint64_t n_records, uint64_t first_record, uint8_t* d_seq,
	uint64_t capacity, uint64_t* d_result, void* stream);
/* The records decoded straight into the handle's batch buffer, then what kmcb200_split / kmcb200_smallk_add / kmcb200_estimator_add do with
 * a batch (homopolymer compression included, when it is on).  KMCB200_ERR_INVALID when n_records * (k + 1) exceeds the handle's
 * max_batch_bytes, or for the chunk checks of kmcb200_kmcdb_decode.  *seq_bytes and *kept (optional) receive the batch's length and the
 * records kept.  There is no signature-statistics form: the reference takes the signature map from the first input database. */
int kmcb200_split_kmcdb(kmcb200_splitter* sp, kmcb200_kmcdb* d, const uint8_t* suffix, uint64_t n_records, uint64_t first_record,
	uint8_t* out, uint64_t out_capacity, uint64_t* out_bytes, uint64_t* pack_bytes, uint64_t pack_capacity, uint64_t* n_packs,
	kmcb200_bin_fragment* frags, uint64_t* seq_bytes, uint64_t* kept);
int kmcb200_smallk_add_kmcdb(kmcb200_smallk* h, kmcb200_kmcdb* d, const uint8_t* suffix, uint64_t n_records, uint64_t first_record,
	uint64_t* seq_bytes, uint64_t* kept);
int kmcb200_estimator_add_kmcdb(kmcb200_estimator* h, kmcb200_kmcdb* d, const uint8_t* suffix, uint64_t n_records, uint64_t first_record,
	uint64_t* seq_bytes, uint64_t* kept);

/* ---- seam #1: sort host records ------------------------------------------------------------------
 * Contract of SortFunction (raduls.h:19-20, kb_sorter.h:775-779): n records of rec_bytes (multiple of 8,
 * CKmer<SIZE> images) sorted ascending on bytes key_bytes-1..0; the result is left in `tmp` when key_bytes
 * is odd and in `recs` when it is even.  Returns 1 / 0 for tmp / recs, negative on error. */
int kmcb200_sort_records(kmcb200_ctx* ctx, void* recs, void* tmp, uint64_t n, uint32_t rec_bytes, uint32_t key_bytes);

/* ---- device-level entry points (pointers are DEVICE pointers, `stream` is a cudaStream_t or NULL) ---
 * All work is enqueued on `stream` (NULL = the context's compute stream) and is asynchronous with respect to the host. */

/* Expand + sort + count one bin that already lives in HBM.  d_superkmers must be 8-byte aligned and READABLE FOR 32 BYTES PAST
 * `size` (the walk and the staging use 16-byte vector loads on the absolute 16-byte grid); likewise the record buffers given to
 * kmcb200_dev_sort / kmcb200_dev_count must be readable for one record past n (the TMA tile loads round an odd count up to an
 * even one).  The values read there are never used.  pack_bytes is a HOST array.  d_result receives 8 x uint64:
 * [0..3] stats, [4] emitted records, [5] capacity error flag, [6] bin-format error bits,
 * [7] 1 when the hybrid MSD / leaf-count path gave up (skew) and the LSD fallback produced the (identical) result. */
int kmcb200_dev_process_bin(kmcb200_ctx* ctx, uint32_t slot,
	const uint8_t* d_superkmers, uint64_t size, uint64_t n_rec,
	const uint64_t* pack_bytes, uint32_t n_packs,
	uint8_t* d_out, uint64_t out_capacity, uint64_t* d_lut, uint64_t* d_result, void* stream);

/* Individual stages, for per-kernel measurement.  d_recs/d_tmp hold n records of 8*ceil(k/32) bytes.
 * kmcb200_dev_expand also leaves the first partition level's work items and digit counts in the slot's workspace, which
 * kmcb200_dev_sort(..., hist_ready=1) consumes; with hist_ready=0 the sort counts the first digit itself.
 * kmcb200_dev_sort returns 1 when the sorted records are in d_tmp, 0 when they are in d_recs. */
int kmcb200_dev_expand(kmcb200_ctx* ctx, uint32_t slot, const uint8_t* d_superkmers, uint64_t size, uint64_t n_rec,
	const uint64_t* pack_bytes, uint32_t n_packs, void* d_recs, uint64_t* d_result, void* stream);
int kmcb200_dev_sort(kmcb200_ctx* ctx, uint32_t slot, void* d_recs, void* d_tmp, uint64_t n, uint32_t key_bytes,
	int hist_ready, void* stream);
int kmcb200_dev_count(kmcb200_ctx* ctx, uint32_t slot, const void* d_sorted, uint64_t n,
	uint8_t* d_out, uint64_t out_capacity, uint64_t* d_lut, uint64_t* d_result, void* stream);

/* Number of kernels this library has launched on the context so far (bench.py reports the delta). */
uint64_t kmcb200_kernel_launches(const kmcb200_ctx* ctx);
/* Duration in ms of the last-run stages of a slot, measured with CUDA events on the launching stream:
 * ms[0] index+expand, ms[1] sort (all of it), ms[2] count/emit, ms[3..3+n) the n timed intervals of the sort (hybrid MSD:
 * level-1 partition, level-2 count, level-2 partition, leaves, LSD fallback; or the plain LSD passes).
 * Blocks until the slot's work has finished.  Returns n, negative on error. */
int kmcb200_stage_times(kmcb200_ctx* ctx, uint32_t slot, float* ms, uint32_t capacity);
/* Comma-separated names of the timed sort intervals ms[3..] of kmcb200_stage_times ("msd_partition_L1,msd_count_L2,...").
 * Returns their number. */
int kmcb200_stage_names(kmcb200_ctx* ctx, uint32_t slot, char* buf, uint32_t capacity);
/* How the last bin of a slot counted its leaves: out[0] = the bits of the second partition level, out[1] = the leaf kernel
 * (KMCB200_LEAF_*; KMCB200_LEAF_NONE when the bin's leaves were sorted, e.g. a bin too small for the MSD path).  Returns 0, negative on error. */
enum { KMCB200_LEAF_NONE = 0, KMCB200_LEAF_HASH = 1, KMCB200_LEAF_HASH_CTA = 2, KMCB200_LEAF_HASH_WIDE = 3 };
int kmcb200_leaf_plan(kmcb200_ctx* ctx, uint32_t slot, uint32_t* out);

#ifdef __cplusplus
}
#endif
#endif
