// kmc_b200 — host side of the C ABI (include/kmc_b200.h): context, HBM workspace, launch sequences.
// The per-bin sequence mirrors CKmerBinSorter<SIZE>::ProcessBins (kmc_core/kb_sorter.h:210-237):
//   Expand (index + expand kernels) -> Sort (two MSD partition levels) + Compact fused in the leaf kernels (leaf_hash_cta.cuh, leaf_hash.cuh,
//   leaf_hash_wide.cuh; one-word leaves with a dominant k-mer: leaf_warp.cuh);
//   behind a device flag: Sort (one cooperative lsd_sort_kernel over all key bytes) -> Compact (count_emit_kernel).
#include "../../include/kmc_b200.h"
#include "common.cuh"
#include "expand.cuh"
#include "radix_sort.cuh"
#include "count.cuh"
#include "msd_sort.cuh"
#include "leaf_warp.cuh"
#include "leaf_hash.cuh"
#include "leaf_hash_cta.cuh"
#include "leaf_hash_wide.cuh"
#include "split.cuh"
#include "fastx.cuh"
#include "small_k.cuh"

#include <cmath>
#include <cstddef>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>
#include <list>
#include <thread>

using namespace kmcb;

namespace {

constexpr int kMaxPasses = 4 * 8;                 // key bytes of a 4-word record
constexpr int kHistRows = kMaxPasses + 1;
constexpr int kCounterSlots = kMaxPasses + 8;     // tile counters: one per pass + [kMaxPasses] for count_emit
constexpr uint32_t kEpochLimit = (1u << 22) - 2;
constexpr int kStageRing = 4;
constexpr size_t kMaxLeaves = 256 * 1024;          // level 1: 8 bits, level 2: up to 10 bits
constexpr uint32_t kHeavyListCap = 2048;           // leaves of more than kLwHeavy records a bin may have before it takes the LSD fallback

thread_local std::string g_create_error;

// what the expand stage left for level 1: nothing / cells per expand tile (expand.cuh) / the 256 digit totals of the pack walk, and the
// records are not written yet: the level-1 partition expands the bin (expand_kernel<kExpandPartition>) with the arguments kept in Slot::expand_args
enum { kHistNone = 0, kHistTiles = 1, kHistTotals = 2 };

struct ZeroBlock {                                // zeroed with one memset at the start of every bin
	uint64_t hist[kHistRows][256];
	uint32_t counters[kCounterSlots];
	uint32_t status[2];                           // expand: [0] error bits, [1] total tiles
	uint32_t msd_flags[4];                        // [0] kMsdFlagFallback (leaves too large -> LSD passes), [1] always 0
	uint32_t msd_n_items[2];                      // work items of the level-1 / level-2 segmentation
	uint32_t msd_counters[4];                     // tickets: level-1 partition, level-2 partition, leaves, leaf-count
	uint32_t heavy_count[2];                      // [0] large leaves noted by the leaf kernel, [1] ticket of the second (HEAVY) launch
	uint32_t heavy_list[kHeavyListCap];           // their leaf ids
	uint32_t leaf_group_sum[kMaxLeaves / 1024];   // emitted records per group of 1024 leaves
	uint32_t l1_total[256];                       // kHistTotals: k-mers of every level-1 digit, counted by the pack walk
	uint32_t l1_cursor[256];                      // kHistTotals: next free record of every level-1 bucket (expand_kernel<kExpandPartition>)
};

static_assert(sizeof(ZeroBlock) % 4 == 0, "zeroed word by word");

struct Slot {
	cudaStream_t stream = nullptr;
	// records
	uint8_t* recs_a = nullptr; size_t recs_a_cap = 0;
	uint8_t* recs_b = nullptr; size_t recs_b_cap = 0;
	uint8_t* recs_x = nullptr; size_t recs_x_cap = 0;        // kmcb200_process_bin_multi: this GPU's key range, gathered from all GPUs
	// bin + index
	uint8_t* d_bin = nullptr; size_t bin_cap = 0;
	uint64_t* d_pack_start = nullptr; size_t packs_cap = 0;
	uint64_t* h_pack_start[kStageRing] = {}; cudaEvent_t ev_pack[kStageRing] = {}; int ring = 0;   // pinned staging of the pack offsets
	uint32_t* pack_nsk = nullptr; uint32_t* pack_nk = nullptr; uint32_t* pack_tbase = nullptr; uint64_t* pack_kbase = nullptr;
	uint32_t* pack_done = nullptr;
	uint32_t* sk_off = nullptr; size_t sk_off_cap = 0;
	uint32_t* sk_kpre = nullptr; size_t sk_kpre_cap = 0;
	uint32_t* tile_first = nullptr; size_t tile_first_cap = 0;
	uint32_t* tile_pack = nullptr; size_t tile_pack_cap = 0;
	uint4* tile_desc = nullptr; size_t tile_desc_cap = 0;
	ZeroBlock* zero = nullptr;
	uint64_t* desc = nullptr; size_t desc_cap = 0;          // radix look-back descriptors
	// hybrid MSD sort: bucket boundaries and work-item tables
	uint64_t* msd_seg1 = nullptr;                           // [2]      {0, n}
	uint64_t* msd_start2 = nullptr;                         // [257]    level-1 buckets
	uint64_t* msd_start3 = nullptr;                         // [kMaxLeaves + 1]  level-2 buckets
	uint32_t* msd_item_base1 = nullptr;                     // [2]
	uint32_t* msd_item_base2 = nullptr;                     // [257]
	uint32_t* msd_item_seg2 = nullptr; size_t msd_item_seg2_cap = 0;
	uint64_t* msd_item_lo1 = nullptr; size_t msd_item_lo1_cap = 0;      // level-1 items = expand tiles
	uint16_t* msd_item_cnt1 = nullptr; size_t msd_item_cnt1_cap = 0;
	uint16_t* msd_cells = nullptr; size_t msd_cells_cap = 0;            // counts[segment][digit][item] (level 1, then reused by level 2)
	uint32_t* msd_cell_scan = nullptr; size_t msd_cell_scan_cap = 0;    // their exclusive scan
	uint32_t* msd_block_sums = nullptr; size_t msd_block_sums_cap = 0;
	// leaf-count path
	uint8_t* leaf_tmp = nullptr; size_t leaf_tmp_cap = 0;
	uint32_t* leaf_emit = nullptr; uint64_t* leaf_off = nullptr;          // [kMaxLeaves]
	const char* pass_names[kMaxPasses + 8] = {};
	uint32_t last_n_packs = 1;
	uint64_t* cdesc = nullptr; size_t cdesc_cap = 0;        // count look-back descriptors
	int hist_mode = 0;                                      // what the last expansion left for the sort: kHistNone / kHistTiles / kHistTotals
	ExpandArgs expand_args{};                               // kHistTotals: the index's arguments, for the level-1 partition expansion
	// outputs of the host-buffer path
	uint8_t* d_out = nullptr; size_t out_cap = 0;
	uint64_t* d_lut = nullptr;
	uint64_t* d_result = nullptr; uint64_t* h_result = nullptr; uint64_t* h_result_dev = nullptr;
	// events
	cudaEvent_t ev_begin = nullptr, ev_expand = nullptr, ev_sort = nullptr, ev_count = nullptr, ev_result = nullptr;
	cudaEvent_t ev_h2d = nullptr, ev_done = nullptr, ev_walk = nullptr;           // copy stream <-> compute stream hand-over
	cudaEvent_t ev_pass[kMaxPasses + 8] = {};
	int n_passes_run = 0;                                   // number of timed sort intervals (ev_pass[i] .. ev_pass[i+1])
	bool ran_expand = false, ran_sort = false, ran_count = false;
	// oversized bins
	uint64_t* d_hist12 = nullptr; unsigned long long* d_out_counter = nullptr; size_t out_counter_cap = 0;
	uint16_t* d_blk_of_prefix = nullptr; uint64_t* d_region_start = nullptr; size_t region_cap = 0; bool last_scatter = false;      // key blocks, scatter flow
	uint64_t* tot_lut = nullptr; uint64_t* tot_res = nullptr; uint32_t last_blocks = 0;      // totals over the key blocks
	bool scan_lut = false; uint64_t scan_base = 0;                                            // kmcb200_wait_bin_scanned
	uint8_t* d_extras = nullptr; size_t extras_cap = 0; uint64_t* d_pack_rec = nullptr; size_t pack_rec_cap = 0;      // kmcb200_submit_bin_indexed (N4)
	uint64_t* h_pack_rec = nullptr; size_t h_pack_rec_cap = 0; bool have_extras = false;
	bool sync_done = false; uint64_t sync_out_bytes = 0; uint64_t sync_stats[4] = {};
	// pending host-buffer bin
	bool busy = false;
	uint8_t* host_out = nullptr; uint64_t host_out_cap = 0; uint64_t* host_lut = nullptr; uint64_t pending_n_rec = 0;
};

}  // namespace

struct kmcb200_ctx {
	kmcb200_params prm{};
	int words = 1;
	uint32_t key_bytes = 0, suffix_bytes = 0, counter_bytes = 0;
	uint64_t lut_entries = 0;
	int sm_count = 0;
	int occ_radix = 1, occ_expand = 1, occ_expand_part = 1, occ_msd_part = 1, occ_msd_part_wide = 1, occ_msd_local = 1;
	uint32_t force_b2 = 0;                                  // KMCB200_L2_BITS: bits of the second partition level (0: chosen from the bin size)
	bool use_msd = true;                                    // KMCB200_SORT=lsd forces the plain 8-bit LSD passes
	bool scatter_blocks = true;                             // KMCB200_KEY_BLOCKS=filter: key blocks always re-expand the bin with a filter (what happens anyway when the records do not fit in HBM once)
	uint64_t key_block_records = 1ull << 28;                // KMCB200_KEY_BLOCK_RECORDS: preferred size of a key block when the bin is scattered once (leaves of ~1-2 K records)
	bool overlap_walk = true;                               // KMCB200_OVERLAP_WALK=0: the index kernels of a submitted bin on the compute stream instead of its copy stream
	bool use_leaf = true;                                   // KMCB200_LEAF=sort sorts the leaves + count_emit instead of counting them
	int occ_leaf_hash = 1;
	int leaf_cta = 2;                                       // one-word records by leaf_hash_cta_kernel (one table per CTA): 2 = in bins of mean leaves > kLeafCtaMinMean,
	                                                        // 1 = always (KMCB200_LEAF_KERNEL=cta), 0 = never (KMCB200_LEAF_KERNEL=hash: leaf_hash_kernel)
	int leaf_cta_slot_bits = 12;                            // KMCB200_LEAF_CTA = 4:B, the 2^B slots of leaf_hash_cta_kernel's table (4 warps per CTA)
	int occ_leaf_cta = 1;
	uint32_t leaf_max_b2 = 8;                               // KMCB200_LEAF_MAX_B2 (8: on the H100 the 512 / 1024-digit level 2 costs more than it saves, DESIGN 3.1)
	uint32_t leaf_target = 1024;                            // KMCB200_LEAF_TARGET: mean leaf size the second partition level of a large bin aims at (leaf_hash_kernel)
	uint32_t leaf_fill_pct = 62;                            // KMCB200_LEAF_FILL_PCT: leaf_hash_kernel plans a table round for this load
	uint32_t leaf_ratio0_q8 = 90;                           // KMCB200_LEAF_RATIO0: first guess of distinct k-mers per record, x 256 (30x coverage, 1 % errors: ~0.3)
	uint64_t max_block_records = 1ull << 28;                // a bin with more k-mers is counted key block by key block: from the free HBM at create (KMCB200_MAX_BLOCK_RECORDS overrides)
	uint64_t max_chunk_bytes = 1ull << 30;                  // KMCB200_MAX_CHUNK_BYTES: ... and expanded chunk by chunk
	int leaf_slot_bits = 10;                                // KMCB200_LEAF_SLOT_BITS = 8 | 9 | 10: slots of a warp's leaf table
	uint32_t epoch = 1;
	uint64_t launches = 0;
	// All kernels of a context run on ONE stream: the persistent radix passes size their grids to fill the GPU and two of
	// them side by side only steal SMs from each other.  The slots' own streams carry the
	// host<->device copies, so the copies of one bin overlap the kernels of another.
	cudaStream_t compute = nullptr;
	std::vector<Slot> slots;
	std::string err;
};

namespace {

int fail(kmcb200_ctx* c, int code, const char* fmt, ...)
{
	char buf[512];
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(buf, sizeof buf, fmt, ap);
	va_end(ap);
	if (c) c->err = buf;
	else g_create_error = buf;
	return code;
}

#define CU(call)                                                                                             \
	do {                                                                                                     \
		cudaError_t e_ = (call);                                                                             \
		if (e_ != cudaSuccess) return fail(ctx, KMCB200_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
	} while (0)

// Zeroing on the compute stream is done by a kernel, not by cudaMemsetAsync: a memset may be carried out by a copy engine, and
// the copy engines are busy with the next bin's 66 MB host-to-device transfer - the kernels behind the memset would wait for it.
__global__ void zero_words_kernel(uint32_t* p, size_t n_words)
{
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += (size_t)gridDim.x * blockDim.x) p[i] = 0u;
}
int zero_async(kmcb200_ctx* ctx, void* ptr, size_t bytes, cudaStream_t st)
{
	if (bytes == 0) return 0;
	if ((reinterpret_cast<uintptr_t>(ptr) & 3u) || (bytes & 3u) || bytes > (size_t(1) << 28)) { CU(cudaMemsetAsync(ptr, 0, bytes, st)); return 0; }
	const size_t n = bytes / 4;
	zero_words_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, 1184), 256, 0, st>>>(reinterpret_cast<uint32_t*>(ptr), n);
	ctx->launches++;
	CU(cudaGetLastError());
	return 0;
}

// start of a bin: the slot's ZeroBlock, and (when given) the LUT and the 8 result words, in ONE launch
__global__ void bin_init_kernel(uint32_t* zero_block, uint32_t zero_words, uint32_t* lut, size_t lut_words, uint32_t* result)
{
	const size_t stride = (size_t)gridDim.x * blockDim.x, i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	for (size_t i = i0; i < zero_words; i += stride) zero_block[i] = 0u;
	if (lut) for (size_t i = i0; i < lut_words; i += stride) lut[i] = 0u;
	if (result && i0 < 16) result[i0] = 0u;
}

uint32_t byte_log(uint64_t x) { return x < (1u << 8) ? 1 : x < (1u << 16) ? 2 : x < (1u << 24) ? 3 : 4; }   // defs.h:121

template <typename T>
int ensure(kmcb200_ctx* ctx, T*& p, size_t& cap, size_t need_elems, bool zero = false)
{
	if (need_elems <= cap && p) return 0;
	size_t n = std::max<size_t>(need_elems + need_elems / 8, 1024);
	if (p) CU(cudaFree(p));
	p = nullptr; cap = 0;
	CU(cudaMalloc(reinterpret_cast<void**>(&p), n * sizeof(T) + 256));
	if (zero) { CU(cudaMemset(p, 0, n * sizeof(T) + 256)); CU(cudaDeviceSynchronize()); }   // the slot streams are non-blocking
	cap = n;
	return 0;
}

// `count` consecutive epochs for the look-back descriptors of the next launches
int next_epoch(kmcb200_ctx* ctx, uint32_t* out, uint32_t count = 1)
{
	if (ctx->epoch + count >= kEpochLimit) {   // wrap: forget every descriptor ever written - but only once nothing is spinning on them any more
		CU(cudaDeviceSynchronize());
		for (auto& s : ctx->slots) {
			if (s.desc) CU(cudaMemset(s.desc, 0, s.desc_cap * sizeof(uint64_t)));
			if (s.cdesc) CU(cudaMemset(s.cdesc, 0, s.cdesc_cap * sizeof(uint64_t)));
		}
		CU(cudaDeviceSynchronize());
		ctx->epoch = 1;
	}
	*out = ctx->epoch;
	ctx->epoch += count;
	return 0;
}

// --------------------------------------------------------------------------------------------- per-WORDS launchers
template <int WORDS>
int setup_kernels(kmcb200_ctx* ctx)
{
	CU(cudaFuncSetAttribute(radix_pass_kernel<WORDS>, cudaFuncAttributeMaxDynamicSharedMemorySize, SortSmem<WORDS>::kBytes));
	CU(cudaFuncSetAttribute(lsd_sort_kernel<WORDS>, cudaFuncAttributeMaxDynamicSharedMemorySize, SortSmem<WORDS>::kBytes));
	CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_radix, lsd_sort_kernel<WORDS>, SortCfg<WORDS>::kThreads, SortSmem<WORDS>::kBytes));
	CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_expand, expand_kernel<WORDS>, ExpandCfg<WORDS>::kThreads, 0));
	if constexpr (expand_partition_supported<WORDS>())
		CU((cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_expand_part, expand_kernel<WORDS, kExpandPartition>, ExpandCfg<WORDS>::kThreads, 0)));
	const size_t cs = count_smem_bytes<WORDS>(ctx->suffix_bytes + ctx->counter_bytes);
	CU(cudaFuncSetAttribute(count_emit_kernel<WORDS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs));
	CU(cudaFuncSetAttribute(msd_partition_kernel<WORDS>, cudaFuncAttributeMaxDynamicSharedMemorySize, MsdSmem<WORDS>::kBytes));
	CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_msd_part, msd_partition_kernel<WORDS>, MsdCfg<WORDS>::kThreads + 32, MsdSmem<WORDS>::kBytes));
	CU(cudaFuncSetAttribute(msd_partition_kernel<WORDS, 1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, MsdSmem<WORDS, 1024>::kBytes));
	CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_msd_part_wide, msd_partition_kernel<WORDS, 1024>, MsdCfg<WORDS>::kThreads + 32, MsdSmem<WORDS, 1024>::kBytes));
	if (ctx->occ_msd_part_wide < 1) ctx->occ_msd_part_wide = 1;
	const int local_smem = msd_local_cap<WORDS>() * 8 * WORDS + (MsdLocalCfg<WORDS>::kThreads / 32) * 1024;
	CU(cudaFuncSetAttribute(msd_local_sort_kernel<WORDS>, cudaFuncAttributeMaxDynamicSharedMemorySize, local_smem));
	CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_msd_local, msd_local_sort_kernel<WORDS>, MsdLocalCfg<WORDS>::kThreads, local_smem));
	if (ctx->occ_radix < 1) ctx->occ_radix = 1;
	if (ctx->occ_expand < 1) ctx->occ_expand = 1;
	if (ctx->occ_msd_part < 1) ctx->occ_msd_part = 1;
	if (ctx->occ_msd_local < 1) ctx->occ_msd_local = 1;
	return 0;
}

template <int WORDS>
int launch_expand(kmcb200_ctx* ctx, const ExpandArgs& a, cudaStream_t st)
{
	const uint64_t n_bound = a.n_rec == kExpandUnknownRecs ? a.size * 4 : a.n_rec;
	const uint32_t max_tiles = (uint32_t)(n_bound / ExpandCfg<WORDS>::kTile) + a.n_packs + 1;
	const uint32_t grid = std::min<uint32_t>(max_tiles, (uint32_t)(ctx->sm_count * (a.mode == kExpandPartition ? std::max(ctx->occ_expand_part, 1) : ctx->occ_expand)));
	switch (a.mode) {
	case kExpandAll: expand_kernel<WORDS, kExpandAll><<<grid, ExpandCfg<WORDS>::kThreads, 0, st>>>(a); break;
	case kExpandPartition:
		if constexpr (expand_partition_supported<WORDS>()) {
			expand_kernel<WORDS, kExpandPartition><<<grid, ExpandCfg<WORDS>::kThreads, 0, st>>>(a);
			break;
		} else return fail(ctx, KMCB200_ERR_INVALID, "no level-1 partition expansion for %d-word records", WORDS);
	case kExpandCount12: expand_kernel<WORDS, kExpandCount12><<<grid, ExpandCfg<WORDS>::kThreads, 0, st>>>(a); break;
	case kExpandScatter: expand_kernel<WORDS, kExpandScatter><<<grid, ExpandCfg<WORDS>::kThreads, 0, st>>>(a); break;
	default: expand_kernel<WORDS, kExpandFilter><<<grid, ExpandCfg<WORDS>::kThreads, 0, st>>>(a); break;
	}
	ctx->launches++;
	CU(cudaGetLastError());
	return 0;
}

__global__ void msd_setup_kernel(uint64_t* seg1, uint32_t* item_base1, uint32_t* n_items1, uint64_t n, uint32_t tile)
{
	seg1[0] = 0; seg1[1] = n;
	const uint32_t nt = (uint32_t)((n + tile - 1) / tile);
	item_base1[0] = 0; item_base1[1] = nt;
	*n_items1 = nt;
}

// bits of the second partition level.  Counted leaves (the bin path) are streamed by one warp and may be any size: a leaf beyond one
// table round only costs extra rounds, while the 512 / 1024-digit partition kernels are slower per record than the 256-digit one.
// So: leaves of ~1 K records while that takes <= 8 bits, then (one-word records) leaves of leaf_target records in at most leaf_max_b2 bits.
// Sorted leaves (seam #1) must fit on chip, and canonical k-mers crowd into the low prefixes (largest leaf ~4.4x the mean): aim at a
// fifth of the capacity, 8 bits at most.
template <int WORDS>
uint32_t choose_b2(const kmcb200_ctx* ctx, uint64_t n, bool counted_leaves)
{
	auto bits_for = [&](uint64_t target) { uint32_t lg = 0; while ((1ull << lg) < (n + target - 1) / target) ++lg; return lg > 8 ? lg - 8 : 0u; };
	uint32_t b2;
	if (counted_leaves) {
		b2 = std::min(bits_for(1024), 10u);
		// leaf_hash_kernel: a leaf of up to ~2100 records of a 30x bin is ONE table round, and the leaves of a bin spread over 0 .. 2x their mean
		// (measured over the bin sizes of the target workload with scripts/l2_bits_sweep.py, DESIGN 3.1).  One-word records only: the leaves
		// of wider records verify every hit against a record in HBM and lose more from a second table round than the wide scatter costs.
		if (WORDS == 1 && b2 > 8) b2 = std::max(8u, std::min(bits_for(ctx->leaf_target), ctx->leaf_max_b2));
		if (ctx->force_b2) b2 = ctx->force_b2;          // (tests: the wide second level on small bins)
	} else
		b2 = std::min(bits_for(std::max<uint64_t>(msd_local_cap<WORDS>() / 5, 64)), 8u);
	return b2;
}
template <int WORDS> uint32_t choose_nd2(const kmcb200_ctx* ctx, uint64_t n, bool counted_leaves) { return 1u << choose_b2<WORDS>(ctx, n, counted_leaves); }

// upper bound of the level-1 work items of a bin
size_t msd_max_items1(uint64_t n_rec, uint32_t n_packs) { return (size_t)(n_rec / kExpandMinTile) + n_packs + 2; }

template <int WORDS>
int ensure_msd(kmcb200_ctx* ctx, Slot& s, uint64_t n, uint32_t n_packs, uint32_t nd2 = 256)
{
	static_assert(msd_tile<WORDS>() >= ExpandCfg<WORDS>::kTile, "a partition tile must hold an expand tile");
	const size_t items1 = std::max(msd_max_items1(n, n_packs), (size_t)(n / msd_tile<WORDS>()) + 2);
	const size_t items2 = (size_t)(n / msd_tile<WORDS>()) + 260;
	const size_t cells = std::max(256 * items1, (size_t)std::max(nd2, 256u) * items2);
	if (int rc = ensure(ctx, s.msd_item_lo1, s.msd_item_lo1_cap, items1)) return rc;
	if (int rc = ensure(ctx, s.msd_item_cnt1, s.msd_item_cnt1_cap, items1)) return rc;
	if (int rc = ensure(ctx, s.msd_item_seg2, s.msd_item_seg2_cap, std::max(items1, items2))) return rc;
	if (int rc = ensure(ctx, s.msd_cells, s.msd_cells_cap, cells)) return rc;
	if (int rc = ensure(ctx, s.msd_cell_scan, s.msd_cell_scan_cap, cells)) return rc;
	if (int rc = ensure(ctx, s.msd_block_sums, s.msd_block_sums_cap, cells / kCellChunk + 2)) return rc;
	return 0;
}

int launch_cell_scan(kmcb200_ctx* ctx, Slot& s, const uint32_t* n_items, uint32_t nd, size_t max_items, const uint32_t* flags, cudaStream_t st)
{
	const uint32_t nb = (uint32_t)(((size_t)nd * max_items + kCellChunk - 1) / kCellChunk);
	cell_reduce_kernel<<<nb, 256, 0, st>>>(s.msd_cells, n_items, nd, s.msd_block_sums, flags);
	cell_scan_sums_kernel<<<1, 1024, 0, st>>>(s.msd_block_sums, n_items, nd, flags);
	cell_scan_kernel<<<nb, 256, 0, st>>>(s.msd_cells, n_items, nd, s.msd_block_sums, s.msd_cell_scan, flags);
	ctx->launches += 3;
	CU(cudaGetLastError());
	return 0;
}

// All key_bytes 8-bit LSD passes from `in` (ping-pong with `out`) in ONE cooperative launch (radix_sort.cuh).  run_flag / run_need:
// the launch returns at once unless (*run_flag & 3) == run_need.  reset_lut != nullptr: the fallback of the leaf-count path first
// forgets what the leaves added to the LUT and the statistics.
template <int WORDS>
int launch_lsd_sort(kmcb200_ctx* ctx, Slot& s, void* in, void* out, uint64_t n, uint32_t key_bytes, const uint32_t* run_flag, uint32_t run_need,
	uint64_t* reset_lut, uint64_t* reset_result, cudaStream_t st)
{
	constexpr int TILE = SortSmem<WORDS>::kTile;
	LsdSortArgs a{};
	a.a = in; a.b = out; a.n = n; a.n_tiles = (uint32_t)((n + TILE - 1) / TILE); a.key_bytes = key_bytes;
	a.hist = &s.zero->hist[0][0]; a.desc = s.desc; a.tile_counters = s.zero->counters;
	if (int rc = next_epoch(ctx, &a.epoch0, key_bytes)) return rc;
	a.run_flag = run_flag; a.run_need = run_need;
	a.reset_lut = reset_lut; a.reset_lut_entries = ctx->lut_entries; a.reset_result = reset_result;
	const uint32_t grid = std::max(1u, std::min<uint32_t>(a.n_tiles, (uint32_t)(ctx->sm_count * ctx->occ_radix)));
	void* params[] = {&a};
	CU(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(lsd_sort_kernel<WORDS>), dim3(grid), dim3(SortCfg<WORDS>::kThreads), params, SortSmem<WORDS>::kBytes, st));
	ctx->launches++;
	return 0;
}

// Filled by launch_sort when the caller wants to count the leaves itself (leaf_count.cuh) instead of sorting them.
struct LeafPlan {
	bool active = false;
	const void* recs = nullptr;      // partitioned records
	const uint64_t* start = nullptr; // leaf boundaries
	uint32_t n_leaves = 0, low_bits = 0;
};

// launch_sort takes the hybrid MSD path (else: the LSD passes alone) for n records with key_bits significant bits
bool msd_path(const kmcb200_ctx* ctx, uint64_t n, uint32_t key_bits) { return ctx->use_msd && key_bits >= 24 && n >= (1u << 16); }

// Sorts n records from `a` (with `b` as the second buffer).  *result_in_b tells where the sorted records end up.
// kHistTiles: the expand stage has zeroed the slot's ZeroBlock and written the level-1 cells / items.
// kHistTotals: it has zeroed the ZeroBlock and counted the level-1 digit totals, and `a` holds no records yet: the level-1 partition
// expands them from the bin into `b` (MSD path only).
template <int WORDS>
int launch_sort(kmcb200_ctx* ctx, Slot& s, void* a, void* b, uint64_t n, uint32_t key_bytes, uint32_t key_bits, int hist_mode, uint32_t n_packs, cudaStream_t st, bool* result_in_b, LeafPlan* plan = nullptr)
{
	constexpr int TILE = SortSmem<WORDS>::kTile;
	constexpr int MTILE = msd_tile<WORDS>();
	const uint64_t n_tiles64 = (n + TILE - 1) / TILE;
	if (n_tiles64 > 0x7fffffffull || n >= (1ull << 32)) return fail(ctx, KMCB200_ERR_INVALID, "bin too large: %llu records", (unsigned long long)n);
	const uint32_t n_tiles = (uint32_t)n_tiles64;
	// key_bits: significant bits of a record.  2k for records we expanded ourselves; all key bytes for foreign records (seam #1)
	const bool msd = msd_path(ctx, n, key_bits);
	if (hist_mode == kHistTotals && !msd) return fail(ctx, KMCB200_ERR_INVALID, "the records of this bin were not expanded");
	const uint32_t top_shift = key_bits - 8;
	if (int rc = ensure(ctx, s.desc, s.desc_cap, (size_t)n_tiles * 256, true)) return rc;
	if (msd) if (int rc = ensure_msd<WORDS>(ctx, s, n, n_packs, choose_nd2<WORDS>(ctx, n, plan != nullptr))) return rc;      // (sized alike by stage_expand: no reallocation here when its cells are in use)

	const bool hist_ready = hist_mode == kHistTiles || hist_mode == kHistTotals;
	if (hist_mode == kHistNone) if (int rc = zero_async(ctx, s.zero, sizeof(ZeroBlock), st)) return rc;
	int iv = 0;      // timed interval index
	CU(cudaEventRecord(s.ev_pass[0], st));
	void* lsd_in = a; void* lsd_out = b;
	const uint32_t* lsd_flag = nullptr;
	if (msd) {
		const uint32_t b2 = choose_b2<WORDS>(ctx, n, plan != nullptr);
		const uint32_t nd2 = 1u << b2;
		// counted leaves are streamed by one warp: only a very loose limit (one-word records: a leaf may be larger still if ONE k-mer dominates it)
		const uint32_t cap = plan ? (WORDS == 1 ? kLwMaxHeavyLeaf : kLwMaxLeaf) : (uint32_t)msd_local_cap<WORDS>();
		const bool final_in_b = (key_bytes % 2) == 0;                 // where the LSD passes (started from b) end; the leaves go to the same place
		void* fin = final_in_b ? b : a;
		uint32_t* flags = s.zero->msd_flags;
		const uint32_t* never = &flags[1];                             // level 1 always runs: the LSD passes start from its output
		const size_t max_items1 = hist_ready ? msd_max_items1(n, n_packs) : (size_t)(n / MTILE) + 2;
		const size_t max_items2 = (size_t)(n / MTILE) + 260;
		const uint32_t pgrid1 = (uint32_t)std::min<size_t>(max_items1, (size_t)ctx->sm_count * ctx->occ_msd_part);
		const uint32_t pgrid2 = (uint32_t)std::min<size_t>(max_items2, (size_t)ctx->sm_count * (nd2 > 256 ? ctx->occ_msd_part_wide : ctx->occ_msd_part));
		const int local_smem = msd_local_cap<WORDS>() * 8 * WORDS + (MsdLocalCfg<WORDS>::kThreads / 32) * 1024;

		MsdItems items1{};
		if (hist_mode == kHistTiles) {          // items and cells were written by expand_kernel<kExpandAll>
			items1.item_lo = s.msd_item_lo1; items1.item_cnt = s.msd_item_cnt1; items1.n_items = &s.zero->status[1];
		} else if (hist_mode == kHistNone) {
			msd_setup_kernel<<<1, 1, 0, st>>>(s.msd_seg1, s.msd_item_base1, &s.zero->msd_n_items[0], n, MTILE);
			items1.seg_start = s.msd_seg1; items1.item_base = s.msd_item_base1; items1.item_seg = s.msd_item_seg2 /* all zero: see below */;
			items1.n_items = &s.zero->msd_n_items[0];
			if (int rc = zero_async(ctx, s.msd_item_seg2, max_items1 * sizeof(uint32_t), st)) return rc;      // single segment: every item belongs to segment 0
			MsdCountArgs c1{a, items1, top_shift, 256, s.msd_cells, never};
			msd_count_kernel<WORDS><<<(uint32_t)std::min<size_t>(max_items1, (size_t)ctx->sm_count * 4), 512, 0, st>>>(c1);
			ctx->launches += 2;
		}
		if (hist_mode != kHistTotals) {
			if (int rc = launch_cell_scan(ctx, s, items1.n_items, 256, max_items1, never, st)) return rc;
			s.pass_names[iv] = "msd_scan_L1"; CU(cudaEventRecord(s.ev_pass[++iv], st));
		}
		MsdBoundsArgs b1{};
		b1.cell_scan = s.msd_cell_scan; b1.items = items1; b1.S = 1; b1.nd = 256; b1.n = n; b1.start = s.msd_start2;
		b1.cap = b2 == 0 ? cap : 0; b1.flags = flags;
		b1.tile = b2 > 0 ? MTILE : 0; b1.item_base = s.msd_item_base2; b1.item_seg = s.msd_item_seg2; b1.n_items = &s.zero->msd_n_items[1];
		if (hist_mode == kHistTotals) {          // the records go from the bin straight into their level-1 buckets in b
			// the buckets (and their cursors) from the walk's digit totals first: the expansion reserves its runs inside them
			b1.l1_total = s.zero->l1_total; b1.l1_cursor = s.zero->l1_cursor; b1.status = s.zero->status;
			msd_bounds_kernel<<<1, 1024, 0, st>>>(b1);
			ctx->launches++;
			ExpandArgs ea = s.expand_args;
			ea.mode = kExpandPartition; ea.recs = b; ea.l1_cursor = s.zero->l1_cursor; ea.l1_start = s.msd_start2;
			if (int rc = launch_expand<WORDS>(ctx, ea, st)) return rc;
			s.pass_names[iv] = "expand_scatter_L1";
			CU(cudaEventRecord(s.ev_pass[++iv], st));
		} else {
			MsdPartArgs p1{};
			p1.in = a; p1.out = b; p1.items = items1; p1.cell_scan = s.msd_cell_scan; p1.shift = top_shift; p1.nd = 256;
			p1.flags = never;
			msd_partition_kernel<WORDS><<<pgrid1, MsdCfg<WORDS>::kThreads + 32, MsdSmem<WORDS>::kBytes, st>>>(p1);
			ctx->launches++;
			s.pass_names[iv] = "msd_partition_L1";
			CU(cudaEventRecord(s.ev_pass[++iv], st));
			// (the item_seg table of the level-2 items shares its buffer with the all-zero level-1 table of kHistNone: partition first, bounds after)
			msd_bounds_kernel<<<1, 1024, 0, st>>>(b1);
			ctx->launches++;
		}
		if (b2 > 0) {
			MsdItems items2{};
			items2.seg_start = s.msd_start2; items2.item_base = s.msd_item_base2; items2.item_seg = s.msd_item_seg2; items2.n_items = &s.zero->msd_n_items[1];
			MsdCountArgs c2{b, items2, top_shift - b2, nd2, s.msd_cells, flags};
			if (nd2 > 512) msd_count_kernel<WORDS, 1024><<<(uint32_t)std::min<size_t>(max_items2, (size_t)ctx->sm_count * 4), 512, 0, st>>>(c2);
			else if (nd2 > 256) msd_count_kernel<WORDS, 512><<<(uint32_t)std::min<size_t>(max_items2, (size_t)ctx->sm_count * 4), 512, 0, st>>>(c2);
			else msd_count_kernel<WORDS><<<(uint32_t)std::min<size_t>(max_items2, (size_t)ctx->sm_count * 4), 512, 0, st>>>(c2);
			ctx->launches++;
			if (int rc = launch_cell_scan(ctx, s, items2.n_items, nd2, max_items2, flags, st)) return rc;
			MsdBoundsArgs bb{};
			bb.cell_scan = s.msd_cell_scan; bb.items = items2; bb.S = 256; bb.nd = nd2; bb.n = n; bb.start = s.msd_start3; bb.cap = cap; bb.flags = flags; bb.tile = 0;
			msd_bounds_flat_kernel<<<(256 * nd2 + 256) / 256 + 1, 256, 0, st>>>(bb);
			ctx->launches++;
			s.pass_names[iv] = "msd_count_L2"; CU(cudaEventRecord(s.ev_pass[++iv], st));
			MsdPartArgs p2{};
			p2.in = b; p2.out = a; p2.items = items2; p2.cell_scan = s.msd_cell_scan; p2.shift = top_shift - b2; p2.nd = nd2;
			p2.flags = flags;
			if (nd2 > 256) msd_partition_kernel<WORDS, 1024><<<pgrid2, MsdCfg<WORDS>::kThreads + 32, MsdSmem<WORDS, 1024>::kBytes, st>>>(p2);      // (a 512-digit instance with a third TMA buffer was slower)
			else msd_partition_kernel<WORDS><<<pgrid2, MsdCfg<WORDS>::kThreads + 32, MsdSmem<WORDS>::kBytes, st>>>(p2);
			ctx->launches++;
			s.pass_names[iv] = "msd_partition_L2"; CU(cudaEventRecord(s.ev_pass[++iv], st));
		}
		if (plan) {          // the caller counts the leaves (no sort of the duplicates)
			plan->active = true;
			plan->recs = b2 > 0 ? a : b; plan->start = b2 > 0 ? s.msd_start3 : s.msd_start2; plan->n_leaves = 256 * nd2; plan->low_bits = top_shift - b2;
		} else {
			MsdLocalArgs lo{};
			lo.in = b2 > 0 ? a : b; lo.out = fin; lo.start = b2 > 0 ? s.msd_start3 : s.msd_start2; lo.n_buckets = 256 * nd2;
			lo.low_bits = top_shift - b2; lo.bucket_counter = &s.zero->msd_counters[2]; lo.flags = flags;
			const uint32_t lgrid = (uint32_t)std::min<size_t>(lo.n_buckets, (size_t)ctx->sm_count * ctx->occ_msd_local);
			msd_local_sort_kernel<WORDS><<<lgrid, MsdLocalCfg<WORDS>::kThreads, local_smem, st>>>(lo);
			ctx->launches++;
			s.pass_names[iv] = "msd_local_sort"; CU(cudaEventRecord(s.ev_pass[++iv], st));
		}
		lsd_in = b; lsd_out = a; lsd_flag = flags;
		*result_in_b = final_in_b;
	} else
		*result_in_b = (key_bytes % 2) == 1;

	if (plan && plan->active) {        // the caller runs the leaves first, then calls launch_lsd_fallback
		CU(cudaGetLastError());
		s.n_passes_run = iv;
		return 0;
	}
	// 8-bit LSD passes (one cooperative launch): the whole sort when the hybrid path is off (unless the bin is malformed: flags[1]),
	// otherwise its fallback (returns at once unless flagged)
	if (int rc = launch_lsd_sort<WORDS>(ctx, s, lsd_in, lsd_out, n, key_bytes, msd ? lsd_flag : &s.zero->msd_flags[1], msd ? kMsdFlagFallback : 0u, nullptr, nullptr, st)) return rc;
	s.pass_names[iv] = msd ? "lsd_fallback(all passes)" : "lsd_sort(all passes)"; CU(cudaEventRecord(s.ev_pass[++iv], st));
	CU(cudaGetLastError());
	s.n_passes_run = iv;
	return 0;
}

template <int WORDS>
int launch_count(kmcb200_ctx* ctx, Slot& s, const void* sorted, uint64_t n, uint8_t* d_out, uint64_t out_capacity,
	uint64_t* d_lut, uint64_t* d_result, const uint32_t* run_flag, uint32_t run_need, cudaStream_t st, const uint64_t* out_base = nullptr)
{
	constexpr int TILE = count_tile<WORDS>();
	const uint32_t n_tiles = (uint32_t)((n + TILE - 1) / TILE);
	if (int rc = ensure(ctx, s.cdesc, s.cdesc_cap, (size_t)n_tiles, true)) return rc;
	CountArgs a;
	a.recs = sorted; a.n = n; a.n_tiles = n_tiles; a.k = ctx->prm.kmer_len; a.lut_prefix_len = ctx->prm.lut_prefix_len;
	a.cutoff_min = ctx->prm.cutoff_min; a.cutoff_max = ctx->prm.cutoff_max; a.counter_max = ctx->prm.counter_max;
	a.counter_bytes = ctx->counter_bytes; a.suffix_bytes = ctx->suffix_bytes;
	a.out = d_out; a.out_capacity = out_capacity; a.lut = d_lut; a.result = d_result;
	a.desc = s.cdesc; a.tile_counter = &s.zero->counters[kMaxPasses];
	if (int rc = next_epoch(ctx, &a.epoch)) return rc;
	a.run_flag = run_flag; a.run_need = run_need; a.out_base = out_base;
	const size_t smem = count_smem_bytes<WORDS>(ctx->suffix_bytes + ctx->counter_bytes);
	count_emit_kernel<WORDS><<<std::min<uint32_t>(n_tiles, (uint32_t)ctx->sm_count * 6), CountCfg<WORDS>::kThreads, smem, st>>>(a);
	ctx->launches++;
	CU(cudaGetLastError());
	return 0;
}

#define DISPATCH_WORDS(ctx, fn, ...)                                   \
	((ctx)->words == 1 ? fn<1>(__VA_ARGS__) : (ctx)->words == 2 ? fn<2>(__VA_ARGS__) \
	 : (ctx)->words == 3 ? fn<3>(__VA_ARGS__) : fn<4>(__VA_ARGS__))

// --------------------------------------------------------------------------------------------- stages
int set_device(kmcb200_ctx* ctx) { CU(cudaSetDevice(ctx->prm.device)); return 0; }

int check_slot(kmcb200_ctx* ctx, uint32_t slot)
{
	if (!ctx) return KMCB200_ERR_INVALID;
	if (slot >= ctx->slots.size()) return fail(ctx, KMCB200_ERR_INVALID, "slot %u out of range (n_slots=%zu)", slot, ctx->slots.size());
	return 0;
}

// index + expand; pack_bytes is a host array (may be null / empty: the whole bin is one pack)
struct ExpandMode {            // oversized bins: count the top 12 bits / keep one key block (expand.cuh)
	uint32_t mode = kExpandAll, fshift = 0, fprefix = 0, fmask = 0xFFFu;
	uint64_t* hist12 = nullptr;
	unsigned long long* out_counter = nullptr;
	const uint16_t* blk_of_prefix = nullptr; const uint64_t* region_start = nullptr; uint32_t n_blocks = 0;      // kExpandScatter
};

// Host prefix sum of the expander-pack sizes -> pinned staging -> device, on `st`.  The host-buffer path enqueues this on the slot's
// COPY stream, next to the bin itself: on the compute stream the 8 KB copy would queue up behind the next bin's 66 MB H2D transfer on
// the same DMA engine and stall the kernels.
int upload_packs(kmcb200_ctx* ctx, Slot& s, uint64_t size, const uint64_t* pack_bytes, uint32_t n_packs, cudaStream_t st)
{
	const uint32_t np = (n_packs && pack_bytes) ? n_packs : 1;
	if (np + 1 > s.packs_cap) {
		const size_t cap = np + np / 4 + 64;
		CU(cudaDeviceSynchronize());
		for (int i = 0; i < kStageRing; ++i) {
			if (s.h_pack_start[i]) CU(cudaFreeHost(s.h_pack_start[i]));
			s.h_pack_start[i] = nullptr;
		}
		for (void* p : {(void*)s.d_pack_start, (void*)s.pack_nsk, (void*)s.pack_nk, (void*)s.pack_tbase, (void*)s.pack_kbase})
			if (p) CU(cudaFree(p));
		s.packs_cap = 0;
		for (int i = 0; i < kStageRing; ++i) CU(cudaHostAlloc(reinterpret_cast<void**>(&s.h_pack_start[i]), cap * 8, cudaHostAllocDefault));
		CU(cudaMalloc(reinterpret_cast<void**>(&s.d_pack_start), cap * 8));
		CU(cudaMalloc(reinterpret_cast<void**>(&s.pack_nsk), cap * 4));
		CU(cudaMalloc(reinterpret_cast<void**>(&s.pack_nk), cap * 4));
		CU(cudaMalloc(reinterpret_cast<void**>(&s.pack_tbase), cap * 4));
		CU(cudaMalloc(reinterpret_cast<void**>(&s.pack_kbase), cap * 8));
		if (s.pack_done) CU(cudaFree(s.pack_done));
		CU(cudaMalloc(reinterpret_cast<void**>(&s.pack_done), cap * 4));
		s.packs_cap = cap;
	}
	// (ring: the copy of an earlier bin may still be queued)
	s.ring = (s.ring + 1) % kStageRing;
	CU(cudaEventSynchronize(s.ev_pack[s.ring]));
	uint64_t* hps = s.h_pack_start[s.ring];
	uint64_t acc = 0;
	if (n_packs && pack_bytes) {
		for (uint32_t i = 0; i < np; ++i) { hps[i] = acc; acc += pack_bytes[i]; }
	}
	else acc = size;
	hps[0] = 0;
	hps[np] = acc;
	if (acc != size) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "expander packs cover %llu bytes but the bin has %llu", (unsigned long long)acc, (unsigned long long)size);
	CU(cudaMemcpyAsync(s.d_pack_start, hps, (np + 1) * 8, cudaMemcpyHostToDevice, st));
	CU(cudaEventRecord(s.ev_pack[s.ring], st));
	return 0;
}

int stage_expand(kmcb200_ctx* ctx, Slot& s, const uint8_t* d_bin, uint64_t size, uint64_t n_rec,
	const uint64_t* pack_bytes, uint32_t n_packs, void* d_recs, cudaStream_t st, const ExpandMode& em = ExpandMode(), bool packs_uploaded = false,
	uint64_t* zero_lut = nullptr, uint64_t* zero_result = nullptr, cudaStream_t st_walk = nullptr)
{
	// st_walk: the slot's copy stream (host-buffer path).  The index of a bin (init + walk + pack scan, slot-private
	// buffers only) then runs right behind the bin's H2D copy and overlaps the sort / leaves of the bins before it on the compute stream.
	cudaStream_t st_expand = st;
	if (st_walk) st = st_walk;
	if (size >= (1ull << 32)) return fail(ctx, KMCB200_ERR_INVALID, "bin of %llu bytes: bins of 4 GiB or more are not supported", (unsigned long long)size);
	const uint32_t k = ctx->prm.kmer_len;
	const uint32_t min_rec = 1 + (k + 3) / 4;
	const uint32_t np = (n_packs && pack_bytes) ? n_packs : 1;
	if (!packs_uploaded) if (int rc = upload_packs(ctx, s, size, pack_bytes, n_packs, st)) return rc;

	bool big_pack = !(n_packs && pack_bytes) && size > (uint64_t)kWalkChunk;
	if (n_packs && pack_bytes) for (uint32_t i = 0; i < n_packs && !big_pack; ++i) big_pack = pack_bytes[i] > (uint64_t)kWalkChunk;
	s.last_n_packs = np;
	const uint32_t mode = em.mode;          // (kExpandPartition: the index kernels count the level-1 digits, and no expansion runs here)
	const bool msd_items = mode == kExpandAll || mode == kExpandPartition;          // level 1 of the sort follows: its buffers are sized here
	s.hist_mode = mode == kExpandAll ? kHistTiles : mode == kExpandPartition ? kHistTotals : kHistNone;

	if (int rc = ensure(ctx, s.sk_off, s.sk_off_cap, size / min_rec + 2)) return rc;
	if (int rc = ensure(ctx, s.sk_kpre, s.sk_kpre_cap, size / min_rec + 2)) return rc;
	if (int rc = ensure(ctx, s.tile_first, s.tile_first_cap, size * 4 / kExpandMinTile + np + 2)) return rc;
	const uint64_t n_bound = n_rec == kExpandUnknownRecs ? size * 4 : n_rec;        // a record of 1 + ceil((k+a)/4) bytes holds a+1 k-mers: < 4 per byte
	if (int rc = ensure(ctx, s.tile_pack, s.tile_pack_cap, n_bound / kExpandMinTile + np + 2)) return rc;
	if (int rc = ensure(ctx, s.tile_desc, s.tile_desc_cap, 2 * (n_bound / kExpandMinTile + np + 2))) return rc;

	ExpandArgs a;
	a.bin = d_bin; a.size = size; a.pack_start = s.d_pack_start; a.n_packs = np; a.k = k; a.min_rec_bytes = min_rec;
	a.both_strands = ctx->prm.both_strands; a.n_rec = n_rec;
	a.tile = ctx->words == 1 ? ExpandCfg<1>::kTile : ExpandCfg<2>::kTile;
	a.sk_off = s.sk_off; a.sk_kpre = s.sk_kpre; a.tile_first = s.tile_first; a.pack_nsk = s.pack_nsk; a.pack_nk = s.pack_nk;
	a.pack_kbase = s.pack_kbase; a.pack_tbase = s.pack_tbase; a.tile_pack = s.tile_pack; a.tile_pack_cap = n_bound / kExpandMinTile + np + 2;
	a.tile_desc = s.tile_desc;
	a.status = s.zero->status; a.flags = s.zero->msd_flags;
	a.recs = d_recs;
	a.mode = mode; a.fshift = em.fshift; a.fprefix = em.fprefix; a.fmask = em.fmask; a.hist12 = em.hist12; a.out_counter = em.out_counter;
	a.blk_of_prefix = em.blk_of_prefix; a.region_start = em.region_start; a.n_blocks = em.n_blocks;
	if (msd_items)
		if (int rc = DISPATCH_WORDS(ctx, ensure_msd, ctx, s, n_rec, np, DISPATCH_WORDS(ctx, choose_nd2, ctx, n_rec, ctx->use_leaf))) return rc;
	if (mode == kExpandAll) { a.cells1 = s.msd_cells; a.item_lo1 = s.msd_item_lo1; a.item_cnt1 = s.msd_item_cnt1; }
	else { a.cells1 = nullptr; a.item_lo1 = nullptr; a.item_cnt1 = nullptr; }
	a.top_shift = std::max(2u * k, 8u) - 8u;
	a.l1_total = mode == kExpandPartition ? s.zero->l1_total : nullptr;
	a.l1_cursor = nullptr; a.l1_start = nullptr;
	if (mode == kExpandPartition) s.expand_args = a;

	bin_init_kernel<<<64, 256, 0, st>>>(reinterpret_cast<uint32_t*>(s.zero), (uint32_t)(sizeof(ZeroBlock) / 4), reinterpret_cast<uint32_t*>(zero_lut),
		(size_t)ctx->lut_entries * 2, reinterpret_cast<uint32_t*>(zero_result));
	if (s.have_extras && msd_items) {          // N4: stage 1 handed over the length bytes: two prefix sums per pack instead of the walk
		index_from_extras_kernel<<<np, 1024, 0, st>>>(a, s.d_extras, s.d_pack_rec);
		ctx->launches += 2;
		big_pack = false;
	} else {
		walk_packs_parallel_kernel<<<np, kWalkSegs, kWalkChunk + 32, st>>>(a, s.pack_done);
		ctx->launches += 2;
	}
	// a pack of more than 64 KiB (not a collector flush: a caller-made pack, or the whole bin as one pack) is left to the exact warp-per-pack walker
	if (big_pack) {
		walk_packs_kernel<<<(np + kWalkWarpsPerBlock - 1) / kWalkWarpsPerBlock, 32 * kWalkWarpsPerBlock, 0, st>>>(a, s.pack_done);
		ctx->launches++;
	}
	scan_packs_kernel<<<1, 1024, 0, st>>>(a);
	tile_desc_kernel<<<(uint32_t)((a.tile_pack_cap + 255) / 256), 256, 0, st>>>(a);
	ctx->launches += 2;
	CU(cudaGetLastError());
	if (st_expand != st) {
		CU(cudaEventRecord(s.ev_walk, st));
		CU(cudaStreamWaitEvent(st_expand, s.ev_walk, 0));
	}
	if (mode == kExpandPartition) return 0;          // the bin is expanded by level 1 of the sort, once its buckets are known
	return DISPATCH_WORDS(ctx, launch_expand, ctx, a, st_expand);
}

// outputs_zeroed: the bin's init kernel has already cleared the LUT, the result words and the ZeroBlock (run_bin);
// guarded: skip when the bin was found malformed (flags[1], set by scan_packs_kernel)
int stage_count(kmcb200_ctx* ctx, Slot& s, const void* sorted, uint64_t n, uint8_t* d_out, uint64_t out_capacity,
	uint64_t* d_lut, uint64_t* d_result, cudaStream_t st, bool outputs_zeroed = false, bool guarded = false, const uint64_t* out_base = nullptr)
{
	if (!outputs_zeroed) {
		bin_init_kernel<<<64, 256, 0, st>>>(&s.zero->counters[kMaxPasses], 1u, reinterpret_cast<uint32_t*>(d_lut), (size_t)ctx->lut_entries * 2, reinterpret_cast<uint32_t*>(d_result));
		ctx->launches++;
		CU(cudaGetLastError());
	}
	if (n == 0) return 0;
	return DISPATCH_WORDS(ctx, launch_count, ctx, s, sorted, n, d_out, out_capacity, d_lut, d_result, guarded ? &s.zero->msd_flags[1] : nullptr, 0u, st, out_base);
}

// the 8 result words -> pinned host memory, written by the GPU itself (zero-copy): the host-buffer path then needs no copy-engine
// operation that WAITS for the kernels - such a pending wait can hold up the copies of other bins queued behind it on the engine
__global__ void finish_result_kernel(uint64_t* result, uint64_t n_rec, const uint32_t* status, const uint32_t* msd_flags, volatile uint64_t* host_result)
{
	if (threadIdx.x == 0) {
		result[3] = n_rec;              // n_total = n_rec (kb_sorter.h:1166)
		result[6] = status ? status[0] : 0;
		result[7] = msd_flags ? (msd_flags[0] & 1u) : 0;       // 1: the hybrid MSD / leaf-count path gave up and the LSD fallback produced the result
	}
	__syncwarp();
	if (host_result) {
		if (threadIdx.x < 8) host_result[threadIdx.x] = result[threadIdx.x];
		__threadfence_system();
	}
}

// leaf_hash_cta_kernel: one instance per setting of KMCB200_LEAF_CTA (warps per CTA : log2 of the table's slots)
template <int NWARPS, int SLOT_BITS>
int launch_leaf_cta(kmcb200_ctx* ctx, const LeafArgs& la, bool simple, cudaStream_t st)
{
	const size_t smem = sizeof(LcSmem<NWARPS, SLOT_BITS>);
	const uint32_t grid = std::min<uint32_t>(la.n_leaves, (uint32_t)(ctx->sm_count * ctx->occ_leaf_cta));
	if (simple) leaf_hash_cta_kernel<NWARPS, SLOT_BITS, true><<<grid, 32 * NWARPS, smem, st>>>(la);
	else leaf_hash_cta_kernel<NWARPS, SLOT_BITS, false><<<grid, 32 * NWARPS, smem, st>>>(la);
	return 0;
}

template <int NWARPS, int SLOT_BITS>
int setup_leaf_cta(kmcb200_ctx* ctx)
{
	const int smem = (int)sizeof(LcSmem<NWARPS, SLOT_BITS>);
	int occ_t = 1, occ_f = 1;
	CU((cudaFuncSetAttribute(leaf_hash_cta_kernel<NWARPS, SLOT_BITS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)));
	CU((cudaFuncSetAttribute(leaf_hash_cta_kernel<NWARPS, SLOT_BITS, true>, cudaFuncAttributePreferredSharedMemoryCarveout, 100)));
	CU((cudaFuncSetAttribute(leaf_hash_cta_kernel<NWARPS, SLOT_BITS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)));
	CU((cudaFuncSetAttribute(leaf_hash_cta_kernel<NWARPS, SLOT_BITS, false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100)));
	CU((cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_t, leaf_hash_cta_kernel<NWARPS, SLOT_BITS, true>, 32 * NWARPS, smem)));
	CU((cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_f, leaf_hash_cta_kernel<NWARPS, SLOT_BITS, false>, 32 * NWARPS, smem)));
	ctx->occ_leaf_cta = std::max(1, std::min(occ_t, occ_f));
	return 0;
}

// leaf_hash_cta_kernel takes the bins whose mean leaf (records / leaves) is larger than this.  Its gain is that a leaf of up to ~8 K records
// of a 30x bin is one table round where a warp's table needs 2 .. 4 (leaves spread over 0 .. 2x their mean; a warp's round holds ~1800
// records); for leaves that already fit one warp round, the warp kernel's independent warps are faster (DESIGN 3.2: 0.58 against
// 0.77 ms for a 2^26-k-mer bin, mean leaf 1024, on an H100).
constexpr uint64_t kLeafCtaMinMean = 1280;

#define DISPATCH_CTA(ctx, fn, ...) ((ctx)->leaf_cta_slot_bits == 10 ? fn<4, 10>(__VA_ARGS__) : fn<4, 12>(__VA_ARGS__))

template <int WORDS, int SLOT_BITS>
int launch_leaves(kmcb200_ctx* ctx, const LeafArgs& la, uint64_t n_rec, cudaStream_t st)
{
	const size_t hsmem = sizeof(LhSmem<SLOT_BITS>) * kLwWarps;
	const uint32_t hgrid = std::min<uint32_t>((la.n_leaves + kLwWarps - 1) / kLwWarps, (uint32_t)(ctx->sm_count * ctx->occ_leaf_hash));
	// (the usual cutoffs - cutoff_min >= 2, a cutoff_max no count of a leaf reaches - get the instance without the rarely needed transitions)
	const uint32_t max_count = WORDS == 1 ? kLwHeavy : kLwMaxLeaf;
	const bool simple = la.cutoff_min >= 2u && la.cutoff_max >= la.cutoff_min && (la.cutoff_max + 1u == 0u || la.cutoff_max + 1u > max_count + 1u);
	if constexpr (WORDS == 1) {
		if (ctx->leaf_cta == 1 || (ctx->leaf_cta == 2 && n_rec > kLeafCtaMinMean * la.n_leaves)) DISPATCH_CTA(ctx, launch_leaf_cta, ctx, la, simple, st);
		else if (simple) leaf_hash_kernel<SLOT_BITS, true><<<hgrid, 32 * kLwWarps, hsmem, st>>>(la);
		else leaf_hash_kernel<SLOT_BITS, false><<<hgrid, 32 * kLwWarps, hsmem, st>>>(la);
	} else {
		if (simple) leaf_hash_wide_kernel<WORDS, SLOT_BITS, true><<<hgrid, 32 * kLwWarps, hsmem, st>>>(la);
		else leaf_hash_wide_kernel<WORDS, SLOT_BITS, false><<<hgrid, 32 * kLwWarps, hsmem, st>>>(la);
	}
	ctx->launches++;
	CU(cudaGetLastError());
	return 0;
}

// the leaves of one-word records that the leaf kernel only noted (beyond kLwHeavy records: a dominant k-mer)
template <int WORDS, int SLOT_BITS>
int launch_heavy_leaves(kmcb200_ctx* ctx, const LeafArgs& la, cudaStream_t st)
{
	static_assert(WORDS == 1, "only one-word leaves are noted for the heavy launch");
	const size_t smem = sizeof(LwSmem<SLOT_BITS>) * kLwWarps;
	leaf_warp_kernel<SLOT_BITS><<<(uint32_t)ctx->sm_count, 32 * kLwWarps, smem, st>>>(la);
	ctx->launches++;
	CU(cudaGetLastError());
	return 0;
}

template <int WORDS, int SLOT_BITS>
int setup_leaves(kmcb200_ctx* ctx)
{
	const int hsmem = (int)(sizeof(LhSmem<SLOT_BITS>) * kLwWarps);
	int occ_t = 1, occ_f = 1;
	if constexpr (WORDS == 1) {
		CU((cudaFuncSetAttribute(leaf_warp_kernel<SLOT_BITS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(LwSmem<SLOT_BITS>) * kLwWarps))));
		CU((cudaFuncSetAttribute(leaf_hash_kernel<SLOT_BITS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, hsmem)));
		CU((cudaFuncSetAttribute(leaf_hash_kernel<SLOT_BITS, true>, cudaFuncAttributePreferredSharedMemoryCarveout, 100)));
		CU((cudaFuncSetAttribute(leaf_hash_kernel<SLOT_BITS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, hsmem)));
		CU((cudaFuncSetAttribute(leaf_hash_kernel<SLOT_BITS, false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100)));
		CU((cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_t, leaf_hash_kernel<SLOT_BITS, true>, 32 * kLwWarps, hsmem)));
		CU((cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_f, leaf_hash_kernel<SLOT_BITS, false>, 32 * kLwWarps, hsmem)));
		if (ctx->leaf_cta)
			if (int rc = DISPATCH_CTA(ctx, setup_leaf_cta, ctx)) return rc;
	} else {
		CU((cudaFuncSetAttribute(leaf_hash_wide_kernel<WORDS, SLOT_BITS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, hsmem)));
		CU((cudaFuncSetAttribute(leaf_hash_wide_kernel<WORDS, SLOT_BITS, true>, cudaFuncAttributePreferredSharedMemoryCarveout, 100)));
		CU((cudaFuncSetAttribute(leaf_hash_wide_kernel<WORDS, SLOT_BITS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, hsmem)));
		CU((cudaFuncSetAttribute(leaf_hash_wide_kernel<WORDS, SLOT_BITS, false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100)));
		CU((cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_t, leaf_hash_wide_kernel<WORDS, SLOT_BITS, true>, 32 * kLwWarps, hsmem)));
		CU((cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_f, leaf_hash_wide_kernel<WORDS, SLOT_BITS, false>, 32 * kLwWarps, hsmem)));
	}
	ctx->occ_leaf_hash = std::max(1, std::min(occ_t, occ_f));
	return 0;
}

#define DISPATCH_SLOTS(ctx, fn, W, ...) ((ctx)->leaf_slot_bits == 8 ? fn<W, 8>(__VA_ARGS__) : (ctx)->leaf_slot_bits == 10 ? fn<W, 10>(__VA_ARGS__) : fn<W, 9>(__VA_ARGS__))

template <int WORDS> int setup_leaves_w(kmcb200_ctx* ctx) { return DISPATCH_SLOTS(ctx, setup_leaves, WORDS, ctx); }

// Partition (two MSD levels), then COUNT the leaves (leaf_hash_cta.cuh / leaf_hash.cuh / leaf_hash_wide.cuh, leaf_warp.cuh for a dominant k-mer) instead of sorting them; the LSD passes + count_emit_kernel
// stand behind as the device-flagged fallback (they return at once unless a leaf could not be counted).
template <int WORDS>
int run_sort_count_leaves(kmcb200_ctx* ctx, Slot& s, uint64_t n_rec, uint32_t np_eff, uint8_t* d_out, uint64_t out_capacity, uint64_t* d_lut, uint64_t* d_result, cudaStream_t st,
	bool from_blocks = false, uint32_t block_bits = 0, uint32_t block_prefix = 0, bool outputs_zeroed = false, const uint64_t* out_base = nullptr,
	void* ra = nullptr, void* rb = nullptr)
{
	if (!ra) ra = s.recs_a;          // (a key block of a scattered bin sorts its own region of the bin-wide record buffer in place, with rb as scratch)
	if (!rb) rb = s.recs_b;
	// block_bits > 0: the records are one key block of an oversized bin (all share their top block_bits bits = block_prefix):
	// the sort starts below those bits, and nobody has counted the first digit yet
	bool in_b = false;
	LeafPlan plan;
	if (int rc = launch_sort<WORDS>(ctx, s, ra, rb, n_rec, ctx->key_bytes, 2u * ctx->prm.kmer_len - block_bits, from_blocks ? (int)kHistNone : s.hist_mode, np_eff, st, &in_b, &plan)) return rc;
	if (!plan.active) {          // small bin: plain LSD passes, classic count
		CU(cudaEventRecord(s.ev_sort, st));
		s.ran_sort = true;
		const void* sorted = in_b ? rb : ra;
		return stage_count(ctx, s, sorted, n_rec, d_out, out_capacity, d_lut, d_result, st, outputs_zeroed, true, out_base);
	}
	const uint32_t ob = ctx->suffix_bytes + ctx->counter_bytes;
	const size_t pad = (size_t)((ob + 7) / 8) * 8;
	if (int rc = ensure(ctx, s.leaf_tmp, s.leaf_tmp_cap, (size_t)n_rec * pad + 64)) return rc;
	if (!outputs_zeroed) {
		bin_init_kernel<<<64, 256, 0, st>>>(nullptr, 0u, reinterpret_cast<uint32_t*>(d_lut), (size_t)ctx->lut_entries * 2, reinterpret_cast<uint32_t*>(d_result));
		ctx->launches++;
	}
	uint32_t* flags = s.zero->msd_flags;
	LeafArgs la{};
	la.recs = plan.recs; la.start = plan.start; la.n_leaves = plan.n_leaves; la.low_bits = plan.low_bits;
	la.fill_pct = ctx->leaf_fill_pct; la.ratio0_q8 = ctx->leaf_ratio0_q8;
	la.leaf_prefix = block_bits ? block_prefix * plan.n_leaves : 0u;          // n_leaves is a power of two
	la.k = ctx->prm.kmer_len; la.lut_prefix_len = ctx->prm.lut_prefix_len; la.cutoff_min = ctx->prm.cutoff_min; la.cutoff_max = ctx->prm.cutoff_max;
	la.counter_max = ctx->prm.counter_max; la.counter_bytes = ctx->counter_bytes; la.suffix_bytes = ctx->suffix_bytes;
	la.heavy_list = s.zero->heavy_list; la.heavy_count = &s.zero->heavy_count[0]; la.heavy_ticket = &s.zero->heavy_count[1]; la.heavy_cap = kHeavyListCap;
	la.tmp = s.leaf_tmp; la.leaf_emit = s.leaf_emit; la.group_sum = s.zero->leaf_group_sum; la.lut = d_lut; la.result = d_result; la.ticket = &s.zero->msd_counters[3]; la.flags = flags;
	if (int rc = DISPATCH_SLOTS(ctx, launch_leaves, WORDS, ctx, la, n_rec, st)) return rc;
	if constexpr (WORDS == 1) {          // the large leaves the main launch only noted (none in a typical bin: the launch returns at once)
		if (int rc = DISPATCH_SLOTS(ctx, launch_heavy_leaves, WORDS, ctx, la, st)) return rc;
	}
	leaf_scan_kernel<<<(plan.n_leaves + 1023) / 1024, 1024, 0, st>>>(s.leaf_emit, s.zero->leaf_group_sum, plan.n_leaves, s.leaf_off, d_result, out_capacity, ob, flags, out_base);
	leaf_gather_kernel<<<(plan.n_leaves + 7) / 8, 256, 0, st>>>(s.leaf_tmp, plan.start, s.leaf_emit, s.leaf_off, plan.n_leaves, ob, d_out, d_result, flags, out_base);
	ctx->launches += 2;
	int iv = s.n_passes_run;
	s.pass_names[iv] = "leaf_count"; CU(cudaEventRecord(s.ev_pass[++iv], st));
	// fallback (two launches that return at once unless a leaf could not be counted): all LSD passes from the level-1 output in one
	// cooperative kernel (which first forgets what the leaves added to the LUT / statistics), then the classic count
	if (int rc = launch_lsd_sort<WORDS>(ctx, s, rb, ra, n_rec, ctx->key_bytes, flags, kMsdFlagFallback, d_lut, d_result, st)) return rc;
	s.pass_names[iv] = "lsd_fallback(all passes)"; CU(cudaEventRecord(s.ev_pass[++iv], st));
	s.n_passes_run = iv;
	CU(cudaEventRecord(s.ev_sort, st));
	s.ran_sort = true;
	const void* sorted = (ctx->key_bytes % 2 == 0) ? rb : ra;
	return launch_count<WORDS>(ctx, s, sorted, n_rec, d_out, out_capacity, d_lut, d_result, flags, kMsdFlagFallback, st, out_base);
}

// Expand -> Sort -> Compact on device buffers; records live in the slot workspace
int run_bin(kmcb200_ctx* ctx, Slot& s, const uint8_t* d_bin, uint64_t size, uint64_t n_rec, const uint64_t* pack_bytes, uint32_t n_packs,
	uint8_t* d_out, uint64_t out_capacity, uint64_t* d_lut, uint64_t* d_result, cudaStream_t st, bool packs_uploaded = false, uint64_t* host_result = nullptr,
	cudaStream_t st_walk = nullptr)
{
	const size_t rec_bytes = (size_t)ctx->words * 8;
	s.ran_expand = s.ran_sort = s.ran_count = false;
	CU(cudaEventRecord(s.ev_begin, st));
	if (n_rec == 0 || size == 0) {
		if (n_rec != 0 || size != 0) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "bin with size=%llu but n_rec=%llu", (unsigned long long)size, (unsigned long long)n_rec);
		if (int rc = stage_count(ctx, s, nullptr, 0, d_out, out_capacity, d_lut, d_result, st)) return rc;
		if (host_result) { finish_result_kernel<<<1, 32, 0, st>>>(d_result, 0, nullptr, nullptr, host_result); ctx->launches++; }
		CU(cudaEventRecord(s.ev_expand, st)); CU(cudaEventRecord(s.ev_sort, st)); CU(cudaEventRecord(s.ev_count, st));
		s.n_passes_run = 0;
		return 0;
	}
	if (int rc = ensure(ctx, s.recs_a, s.recs_a_cap, n_rec * rec_bytes)) return rc;
	if (int rc = ensure(ctx, s.recs_b, s.recs_b_cap, n_rec * rec_bytes)) return rc;
	// a bin of one-word records that takes the MSD path is expanded once, straight into its level-1 buckets, whose sizes the pack walk
	// counts (expand.cuh, kExpandPartition): its records are never written in tile order and read back by a separate partition pass
	ExpandMode em;
	if (expand_partition_supported<1>() && ctx->words == 1 && n_rec < (1ull << 32) && msd_path(ctx, n_rec, 2u * ctx->prm.kmer_len)) em.mode = kExpandPartition;
	if (int rc = stage_expand(ctx, s, d_bin, size, n_rec, pack_bytes, n_packs, s.recs_a, st, em, packs_uploaded, d_lut, d_result, st_walk)) return rc;
	CU(cudaEventRecord(s.ev_expand, st));
	s.ran_expand = true;
	bool in_b = false;
	const uint32_t np_eff = (n_packs && pack_bytes) ? n_packs : 1u;
	if (ctx->use_leaf) {
		if (int rc = DISPATCH_WORDS(ctx, run_sort_count_leaves, ctx, s, n_rec, np_eff, d_out, out_capacity, d_lut, d_result, st, false, 0u, 0u, true)) return rc;
	} else {
		if (int rc = DISPATCH_WORDS(ctx, launch_sort, ctx, s, s.recs_a, s.recs_b, n_rec, ctx->key_bytes, 2u * ctx->prm.kmer_len, s.hist_mode, np_eff, st, &in_b)) return rc;
		CU(cudaEventRecord(s.ev_sort, st));
		s.ran_sort = true;
		const void* sorted = in_b ? s.recs_b : s.recs_a;
		if (int rc = stage_count(ctx, s, sorted, n_rec, d_out, out_capacity, d_lut, d_result, st, true, true)) return rc;
	}
	finish_result_kernel<<<1, 32, 0, st>>>(d_result, n_rec, s.zero->status, s.zero->msd_flags, host_result);
	ctx->launches++;
	CU(cudaEventRecord(s.ev_count, st));
	s.ran_count = true;
	return 0;
}

// ---------------------------------------------------------------------------------------------
// Oversized bins (SURVEY section 8f N1; the reference's answer is strict-memory mode, bkb_sorter.h / bkb_merger.h): more k-mers than
// one sort can take (max_block_records: sized from the free HBM when the context is created - the records, two buffers plus the
// leaves' temporary one, are what does not fit, 24-96 bytes per k-mer against ~1.1 for the bin bytes), or 4 GiB and more of bin bytes.
//   * the bin bytes are uploaded once, cut at pack boundaries into chunks of < 2 GiB (32-bit offsets inside a chunk);
//   * a bin that is only too LONG (>= 4 GiB of bytes, k-mers within the limit) is one key block: no counting pass at all;
//   * otherwise ONE counting expansion histograms the top 12 bits, the host bisects the histogram into aligned prefixes ("key blocks")
//     of at most max_block_records k-mers, and every block is expanded with a filter, sorted and counted on its own.  Blocks are
//     disjoint ranges of the sorted order, so their outputs simply follow each other and the LUTs add up: bit-identical to one shot;
//   * the whole block loop is ASYNCHRONOUS: a block appends its records behind the earlier ones at a device-side offset (out_base),
//     LUT and statistics are accumulated on the device (accumulate_block_kernel), and the host synchronises once at the end.
struct BinChunk { uint32_t pack0, npacks; uint64_t byte0, bytes, dev_off; };
struct KeyBlock { uint32_t prefix, bits; uint64_t n; };

__global__ void accumulate_block_kernel(uint64_t* tot_lut, const uint64_t* blk_lut, uint64_t lut_entries, uint64_t* tot_res, const uint64_t* blk_res,
	const unsigned long long* appended, uint64_t expected)
{
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < lut_entries; i += (uint64_t)gridDim.x * blockDim.x) tot_lut[i] += blk_lut[i];
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		tot_res[0] += blk_res[0]; tot_res[1] += blk_res[1]; tot_res[2] += blk_res[2];
		tot_res[5] |= blk_res[5]; tot_res[7] |= blk_res[7];
		if (appended && *appended != expected) tot_res[6] |= kErrRecCount;          // the filter took another number of k-mers than the counting pass (or n_rec) said
		tot_res[4] += blk_res[4];                                         // = out_base of the next block
	}
}

int plan_chunks(kmcb200_ctx* ctx, uint64_t size, const uint64_t* pack_bytes, uint32_t n_packs, std::vector<BinChunk>& chunks, uint64_t* dev_bytes)
{
	if (!pack_bytes || n_packs == 0) return fail(ctx, KMCB200_ERR_INVALID, "an oversized bin (%llu bytes) needs its expander packs", (unsigned long long)size);
	BinChunk c{0, 0, 0, 0, 0};
	uint64_t pos = 0, dev = 0;
	for (uint32_t i = 0; i < n_packs; ++i) {
		if (pack_bytes[i] >= ctx->max_chunk_bytes) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "expander pack %u has %llu bytes", i, (unsigned long long)pack_bytes[i]);
		if (c.npacks && c.bytes + pack_bytes[i] > ctx->max_chunk_bytes) { c.dev_off = dev; dev += (c.bytes + 64 + 15) & ~15ull; chunks.push_back(c); c = BinChunk{i, 0, pos, 0, 0}; }
		c.npacks++; c.bytes += pack_bytes[i]; pos += pack_bytes[i];
	}
	if (c.npacks) { c.dev_off = dev; dev += (c.bytes + 64 + 15) & ~15ull; chunks.push_back(c); }
	if (pos != size) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "expander packs cover %llu bytes but the bin has %llu", (unsigned long long)pos, (unsigned long long)size);
	*dev_bytes = dev;
	return 0;
}

// counting expansion of the device-resident chunks: where do the k-mers fall (top 12 bits)?  Also checks the packs.  Synchronises.
int count_top12(kmcb200_ctx* ctx, Slot& s, const std::vector<BinChunk>& chunks, const uint64_t* pack_bytes, std::vector<uint64_t>& hist, cudaStream_t st)
{
	const uint32_t k = ctx->prm.kmer_len;
	if (!s.d_hist12) { CU(cudaMalloc(reinterpret_cast<void**>(&s.d_hist12), 4096 * 8)); }
	if (int rc = zero_async(ctx, s.d_hist12, 4096 * 8, st)) return rc;
	ExpandMode em;
	em.mode = kExpandCount12; em.fshift = 2 * k - 12; em.hist12 = s.d_hist12;
	for (const BinChunk& c : chunks) {
		if (int rc = stage_expand(ctx, s, s.d_bin + c.dev_off, c.bytes, kExpandUnknownRecs, pack_bytes + c.pack0, c.npacks, nullptr, st, em)) return rc;
		uint32_t status = 0;
		CU(cudaMemcpyAsync(&status, s.zero->status, 4, cudaMemcpyDeviceToHost, st));
		CU(cudaStreamSynchronize(st));
		if (status & kErrPackWalk) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "bin format error: an expander pack does not end on a record boundary");
	}
	hist.assign(4096, 0);
	CU(cudaMemcpyAsync(hist.data(), s.d_hist12, 4096 * 8, cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));
	return 0;
}

// aligned prefixes of <= 12 bits inside [lo, hi) of the 4096-entry histogram, each with at most max_records k-mers (bisection; ascending)
int bisect_blocks(kmcb200_ctx* ctx, const std::vector<uint64_t>& hist, uint32_t lo, uint32_t hi, uint64_t max_records, std::vector<KeyBlock>& blocks)
{
	struct Range { uint32_t lo, len; };
	std::vector<Range> todo;
	// cover [lo, hi) with maximal aligned ranges, largest first from the right so that the stack pops them in ascending order
	std::vector<Range> cover;
	for (uint32_t p = lo; p < hi;) {
		uint32_t len = 1;
		while (len < 4096 && (p % (2 * len)) == 0 && p + 2 * len <= hi) len *= 2;
		cover.push_back(Range{p, len});
		p += len;
	}
	for (size_t q = cover.size(); q-- > 0;) todo.push_back(cover[q]);
	while (!todo.empty()) {
		const Range r = todo.back(); todo.pop_back();
		uint64_t cnt = 0;
		for (uint32_t q = r.lo; q < r.lo + r.len; ++q) cnt += hist[q];
		if (cnt == 0) continue;
		if (cnt <= max_records || r.len == 1) {
			if (cnt >= (1ull << 32)) return fail(ctx, KMCB200_ERR_INVALID, "bin too skewed: %llu k-mers share their first 6 symbols", (unsigned long long)cnt);
			uint32_t lg = 0; while ((1u << lg) < r.len) ++lg;
			blocks.push_back(KeyBlock{r.lo >> lg, 12 - lg, cnt});
		} else { todo.push_back(Range{r.lo + r.len / 2, r.len / 2}); todo.push_back(Range{r.lo, r.len / 2}); }      // (the lower half is popped first)
	}
	return 0;
}

// one key block whose records already lie in `region` (n records, 16-byte aligned): sort in place with rb as scratch, count, accumulate
int sort_count_block(kmcb200_ctx* ctx, Slot& s, void* region, void* rb, const KeyBlock& b, uint8_t* d_out, uint64_t out_capacity,
	uint64_t* tot_lut, uint64_t* tot_res, const unsigned long long* appended, cudaStream_t st)
{
	const uint32_t k = ctx->prm.kmer_len;
	if (ctx->use_leaf) {
		if (int rc = DISPATCH_WORDS(ctx, run_sort_count_leaves, ctx, s, b.n, 1u, d_out, out_capacity, s.d_lut, s.d_result, st, true, b.bits, b.prefix, false, tot_res + 4, region, rb)) return rc;
	} else {
		bool in_b = false;
		if (int rc = DISPATCH_WORDS(ctx, launch_sort, ctx, s, region, rb, b.n, ctx->key_bytes, 2u * k - b.bits, (int)kHistNone, 1u, st, &in_b)) return rc;
		CU(cudaEventRecord(s.ev_sort, st));
		if (int rc = stage_count(ctx, s, in_b ? rb : region, b.n, d_out, out_capacity, s.d_lut, s.d_result, st, false, false, tot_res + 4)) return rc;
	}
	accumulate_block_kernel<<<64, 256, 0, st>>>(tot_lut, s.d_lut, ctx->lut_entries, tot_res, s.d_result, appended, b.n);
	ctx->launches++;
	CU(cudaGetLastError());
	return 0;
}

// uploads the tables of a scattering expansion (block of every 12-bit prefix, first record of every block's region) and zeroes the counters
int setup_scatter(kmcb200_ctx* ctx, Slot& s, const std::vector<KeyBlock>& blocks, const std::vector<uint64_t>& region_start, cudaStream_t st)
{
	if (!s.d_out_counter || s.out_counter_cap < blocks.size() + 1) {
		if (s.d_out_counter) CU(cudaFree(s.d_out_counter));
		s.d_out_counter = nullptr;
		s.out_counter_cap = std::max<size_t>(blocks.size() + 1, 64);
		CU(cudaMalloc(reinterpret_cast<void**>(&s.d_out_counter), s.out_counter_cap * 8));
	}
	std::vector<uint16_t> h_blk(4096, (uint16_t)0xFFFF);          // prefixes outside these blocks: skipped
	for (size_t i = 0; i < blocks.size(); ++i) {
		const uint32_t lo = blocks[i].prefix << (12 - blocks[i].bits), len = 1u << (12 - blocks[i].bits);
		for (uint32_t q = lo; q < lo + len; ++q) h_blk[q] = (uint16_t)i;
	}
	if (!s.d_blk_of_prefix) CU(cudaMalloc(reinterpret_cast<void**>(&s.d_blk_of_prefix), 4096 * 2));
	if (!s.d_region_start || s.region_cap < blocks.size()) {
		if (s.d_region_start) CU(cudaFree(s.d_region_start));
		s.d_region_start = nullptr;
		s.region_cap = std::max<size_t>(blocks.size(), 64);
		CU(cudaMalloc(reinterpret_cast<void**>(&s.d_region_start), s.region_cap * 8));
	}
	CU(cudaMemcpyAsync(s.d_blk_of_prefix, h_blk.data(), 4096 * 2, cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(s.d_region_start, region_start.data(), blocks.size() * 8, cudaMemcpyHostToDevice, st));
	CU(cudaStreamSynchronize(st));          // (h_blk goes out of scope)
	return zero_async(ctx, s.d_out_counter, blocks.size() * 8, st);
}

int scatter_chunks(kmcb200_ctx* ctx, Slot& s, const std::vector<BinChunk>& chunks, const uint64_t* pack_bytes, uint32_t n_blocks, void* dst, cudaStream_t st)
{
	ExpandMode es;
	es.mode = kExpandScatter; es.fshift = 2 * ctx->prm.kmer_len - 12; es.out_counter = s.d_out_counter;
	es.blk_of_prefix = s.d_blk_of_prefix; es.region_start = s.d_region_start; es.n_blocks = n_blocks;
	for (const BinChunk& c : chunks)
		if (int rc = stage_expand(ctx, s, s.d_bin + c.dev_off, c.bytes, kExpandUnknownRecs, pack_bytes + c.pack0, c.npacks, dst, st, es)) return rc;
	s.ran_expand = false;
	CU(cudaEventRecord(s.ev_expand, st));
	return 0;
}

// Expands, sorts and counts the given key blocks of the device-resident chunks, one after the other, WITHOUT synchronising: records go to
// d_out behind tot_res[4] records, LUT / statistics are added to tot_lut / tot_res.  The caller zeroes the totals.
//   scatter (the records of all the blocks fit in HBM once, next to one block's scratch): ONE expansion writes every k-mer into the region
//           of its block inside a bin-wide record buffer, and every block is sorted in place there;
//   filter  (the records do not fit, or KMCB200_KEY_BLOCKS=filter): every block expands the whole bin again and keeps its own k-mers.
int run_key_blocks(kmcb200_ctx* ctx, Slot& s, const std::vector<BinChunk>& chunks, const uint64_t* pack_bytes, const std::vector<KeyBlock>& blocks,
	uint8_t* d_out, uint64_t out_capacity, uint64_t* tot_lut, uint64_t* tot_res, cudaStream_t st)
{
	const uint32_t k = ctx->prm.kmer_len;
	const size_t rec_bytes = (size_t)ctx->words * 8;
	uint64_t max_n = 0, sum_n = 0;
	for (const KeyBlock& b : blocks) { max_n = std::max(max_n, b.n); sum_n += b.n; }
	bool scatter = ctx->scatter_blocks && blocks.size() > 1 && blocks.size() <= kExpandMaxBlocks && 2 * k >= 24;
	if (scatter) {          // does the bin-wide buffer fit next to what a block needs (scratch records, padded leaf output, tables)?
		size_t free_b = 0, total_b = 0;
		CU(cudaMemGetInfo(&free_b, &total_b));
		const uint64_t have = (uint64_t)free_b + s.recs_a_cap + s.recs_b_cap + s.leaf_tmp_cap;          // (the slot's own buffers are re-sized below)
		const uint64_t need = sum_n * rec_bytes + max_n * (rec_bytes + 8 * ((ctx->suffix_bytes + ctx->counter_bytes + 7) / 8) + 4) + (256ull << 20);
		scatter = need <= (uint64_t)(0.9 * (double)have);
	}
	s.last_scatter = scatter;
	if (scatter) {
		if (int rc = ensure(ctx, s.recs_a, s.recs_a_cap, (sum_n + blocks.size() + 2) * rec_bytes)) return rc;          // the bin-wide record buffer (+ the regions' alignment gaps)
		if (int rc = ensure(ctx, s.recs_b, s.recs_b_cap, max_n * rec_bytes)) return rc;          // one block's scratch
		std::vector<uint64_t> h_reg(blocks.size());
		uint64_t acc = 0;
		for (size_t i = 0; i < blocks.size(); ++i) {
			acc = (acc + 1) & ~1ull;          // regions start on even records = 16 bytes: the partition kernel's TMA tile loads need it
			h_reg[i] = acc; acc += blocks[i].n;
		}
		if (int rc = setup_scatter(ctx, s, blocks, h_reg, st)) return rc;
		if (int rc = scatter_chunks(ctx, s, chunks, pack_bytes, (uint32_t)blocks.size(), s.recs_a, st)) return rc;
		for (size_t i = 0; i < blocks.size(); ++i)
			if (int rc = sort_count_block(ctx, s, s.recs_a + h_reg[i] * rec_bytes, s.recs_b, blocks[i], d_out, out_capacity, tot_lut, tot_res, s.d_out_counter + i, st)) return rc;
		return 0;
	}
	if (!s.d_out_counter) { s.out_counter_cap = 64; CU(cudaMalloc(reinterpret_cast<void**>(&s.d_out_counter), s.out_counter_cap * 8)); }
	if (int rc = ensure(ctx, s.recs_a, s.recs_a_cap, max_n * rec_bytes)) return rc;          // (sized once: no reallocation, no device synchronisation inside the loop)
	if (int rc = ensure(ctx, s.recs_b, s.recs_b_cap, max_n * rec_bytes)) return rc;
	for (const KeyBlock& b : blocks) {
		if (int rc = zero_async(ctx, s.d_out_counter, 8, st)) return rc;
		ExpandMode ef;
		ef.mode = kExpandFilter; ef.fshift = 2 * k - b.bits; ef.fprefix = b.prefix; ef.out_counter = s.d_out_counter;
		ef.fmask = b.bits ? ((1u << b.bits) - 1u) : 0u;
		if (b.bits == 0) { ef.fshift = 0; ef.fprefix = 0; }          // one block = the whole bin (oversized only by its bytes): keep everything
		for (const BinChunk& c : chunks)
			if (int rc = stage_expand(ctx, s, s.d_bin + c.dev_off, c.bytes, kExpandUnknownRecs, pack_bytes + c.pack0, c.npacks, s.recs_a, st, ef)) return rc;
		s.ran_expand = false;
		CU(cudaEventRecord(s.ev_expand, st));
		if (ctx->use_leaf) {
			if (int rc = DISPATCH_WORDS(ctx, run_sort_count_leaves, ctx, s, b.n, 1u, d_out, out_capacity, s.d_lut, s.d_result, st, true, b.bits, b.prefix, false, tot_res + 4)) return rc;
		} else {
			bool in_b = false;
			if (int rc = DISPATCH_WORDS(ctx, launch_sort, ctx, s, s.recs_a, s.recs_b, b.n, ctx->key_bytes, 2u * k - b.bits, (int)kHistNone, 1u, st, &in_b)) return rc;
			CU(cudaEventRecord(s.ev_sort, st));
			if (int rc = stage_count(ctx, s, in_b ? s.recs_b : s.recs_a, b.n, d_out, out_capacity, s.d_lut, s.d_result, st, false, false, tot_res + 4)) return rc;
		}
		accumulate_block_kernel<<<64, 256, 0, st>>>(tot_lut, s.d_lut, ctx->lut_entries, tot_res, s.d_result, s.d_out_counter, b.n);
		ctx->launches++;
		CU(cudaGetLastError());
	}
	return 0;
}

int ensure_totals(kmcb200_ctx* ctx, Slot& s, cudaStream_t st)
{
	if (!s.tot_lut) {
		CU(cudaMalloc(reinterpret_cast<void**>(&s.tot_lut), ctx->lut_entries * 8));
		CU(cudaMalloc(reinterpret_cast<void**>(&s.tot_res), 64));
	}
	if (int rc = zero_async(ctx, s.tot_lut, ctx->lut_entries * 8, st)) return rc;
	return zero_async(ctx, s.tot_res, 64, st);
}

int run_oversized_bin(kmcb200_ctx* ctx, Slot& s, const uint8_t* h_bin, uint64_t size, uint64_t n_rec, const uint64_t* pack_bytes, uint32_t n_packs,
	uint8_t* h_out, uint64_t out_capacity, uint64_t* h_lut, uint64_t* out_bytes, uint64_t stats[4])
{
	cudaStream_t st = ctx->compute;
	const uint32_t k = ctx->prm.kmer_len;
	std::vector<BinChunk> chunks;
	uint64_t dev_bytes = 0;
	if (int rc = plan_chunks(ctx, size, pack_bytes, n_packs, chunks, &dev_bytes)) return rc;
	if (int rc = ensure(ctx, s.d_bin, s.bin_cap, dev_bytes + 64)) return rc;
	for (const BinChunk& c : chunks) CU(cudaMemcpyAsync(s.d_bin + c.dev_off, h_bin + c.byte0, c.bytes, cudaMemcpyHostToDevice, st));
	std::vector<KeyBlock> blocks;
	if (n_rec <= ctx->max_block_records) blocks.push_back(KeyBlock{0, 0, n_rec});          // only too long: one block, the appended count checks n_rec
	else {
		if (2 * k < 24) return fail(ctx, KMCB200_ERR_INVALID, "a bin of %llu k-mers with k = %u: key blocks need k >= 12", (unsigned long long)n_rec, k);
		std::vector<uint64_t> hist;
		if (int rc = count_top12(ctx, s, chunks, pack_bytes, hist, st)) return rc;
		uint64_t total = 0;
		for (uint64_t v : hist) total += v;
		if (total != n_rec) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "bin format error: the bin holds %llu k-mers, not n_rec = %llu", (unsigned long long)total, (unsigned long long)n_rec);
		// key blocks of the preferred size (leaves of 1-2 K records: the leaf kernel's best case) when ONE scattering expansion can serve them
		// all - i.e. the records fit in HBM once; otherwise as large as one sort can take, because then every block costs an expansion
		size_t free_b = 0, total_b = 0;
		CU(cudaMemGetInfo(&free_b, &total_b));
		const uint64_t rec_b = (uint64_t)ctx->words * 8;
		const bool fits_once = ctx->scatter_blocks && (double)n_rec * rec_b + (double)ctx->key_block_records * (rec_b + 12) * 1.5 < 0.85 * (double)(free_b + s.recs_a_cap + s.recs_b_cap + s.leaf_tmp_cap);
		const uint64_t limit = fits_once ? std::min(ctx->max_block_records, ctx->key_block_records) : ctx->max_block_records;
		if (int rc = bisect_blocks(ctx, hist, 0, 4096, limit, blocks)) return rc;
		if (blocks.size() > kExpandMaxBlocks) { blocks.clear(); if (int rc = bisect_blocks(ctx, hist, 0, 4096, ctx->max_block_records, blocks)) return rc; }
	}
	const uint32_t ob = ctx->suffix_bytes + ctx->counter_bytes;
	if (int rc = ensure(ctx, s.d_out, s.out_cap, out_capacity + 64)) return rc;
	if (int rc = ensure_totals(ctx, s, st)) return rc;
	if (int rc = run_key_blocks(ctx, s, chunks, pack_bytes, blocks, s.d_out, out_capacity, s.tot_lut, s.tot_res, st)) return rc;
	uint64_t r[8];
	CU(cudaMemcpyAsync(r, s.tot_res, 64, cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));          // the only synchronisation of the block loop
	if (r[6]) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "bin format error: the bin does not hold n_rec = %llu k-mers / a pack does not end on a record boundary", (unsigned long long)n_rec);
	const uint64_t bytes = r[4] * (uint64_t)ob;
	if (r[5] || bytes > out_capacity) return fail(ctx, KMCB200_ERR_CAPACITY, "out_capacity %llu too small", (unsigned long long)out_capacity);
	if (bytes) CU(cudaMemcpyAsync(h_out, s.d_out, bytes, cudaMemcpyDeviceToHost, st));
	CU(cudaMemcpyAsync(h_lut, s.tot_lut, ctx->lut_entries * 8, cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));
	s.last_blocks = (uint32_t)blocks.size();
	if (out_bytes) *out_bytes = bytes;
	if (stats) { stats[0] = r[0]; stats[1] = r[1]; stats[2] = r[2]; stats[3] = n_rec; }      // n_total = n_rec (kb_sorter.h:1166)
	return 0;
}

}  // namespace

namespace { __global__ void lut_scan_kernel(uint64_t* lut, uint64_t n, uint64_t base); }

// ================================================================================================= C ABI
extern "C" {

int kmcb200_create(const kmcb200_params* prm, kmcb200_ctx** out_ctx)
{
	kmcb200_ctx* ctx = nullptr;     // fail() then records into the thread-local create error
	if (!prm || !out_ctx) return fail(ctx, KMCB200_ERR_INVALID, "null argument");
	*out_ctx = nullptr;
	if (prm->kmer_len < 1 || prm->kmer_len > KMCB200_MAX_KMER_LEN)
		return fail(ctx, KMCB200_ERR_INVALID, "kmer_len %u outside 1..%d", prm->kmer_len, KMCB200_MAX_KMER_LEN);
	if (prm->lut_prefix_len < 1 || prm->lut_prefix_len >= prm->kmer_len || prm->lut_prefix_len > 15 || (prm->kmer_len - prm->lut_prefix_len) % 4 != 0)
		return fail(ctx, KMCB200_ERR_INVALID, "lut_prefix_len %u illegal for k=%u: need 1 <= p <= 15, p < k, (k-p) %% 4 == 0 (kmc.h:1434-1469)", prm->lut_prefix_len, prm->kmer_len);
	if (prm->n_slots < 1 || prm->n_slots > KMCB200_MAX_SLOTS) return fail(ctx, KMCB200_ERR_INVALID, "n_slots %u outside 1..%d", prm->n_slots, KMCB200_MAX_SLOTS);
	int n_dev = 0;
	if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0)
		return fail(ctx, KMCB200_ERR_NO_DEVICE, "no CUDA device visible: kmc_b200 has no CPU fallback");
	if (prm->device < 0 || prm->device >= n_dev) return fail(ctx, KMCB200_ERR_NO_DEVICE, "device %d not present (%d visible)", prm->device, n_dev);
	cudaDeviceProp dp;
	if (cudaGetDeviceProperties(&dp, prm->device) != cudaSuccess) return fail(ctx, KMCB200_ERR_CUDA, "cudaGetDeviceProperties failed");
	if (dp.major != 9 || dp.minor != 0) return fail(ctx, KMCB200_ERR_NO_DEVICE, "device %d is sm_%d%d; kmc_b200 is built for sm_90a (H100) only", prm->device, dp.major, dp.minor);

	ctx = new kmcb200_ctx();
	ctx->prm = *prm;
	ctx->words = (int)((prm->kmer_len + 31) / 32);
	ctx->key_bytes = (prm->kmer_len + 3) / 4;                                  // rec_len, kb_sorter.h:769
	ctx->suffix_bytes = (prm->kmer_len - prm->lut_prefix_len) / 4;             // kb_sorter.h:1132-1133
	ctx->counter_bytes = prm->counter_max == 1 ? 0 : std::min(byte_log(prm->cutoff_max), byte_log(prm->counter_max));   // defs.h:154-159
	ctx->lut_entries = 1ull << (2 * prm->lut_prefix_len);
	ctx->sm_count = dp.multiProcessorCount;
	if (const char* e = getenv("KMCB200_SORT")) ctx->use_msd = std::string(e) != "lsd";
	if (const char* e = getenv("KMCB200_LEAF")) ctx->use_leaf = std::string(e) != "sort";
	if (const char* e = getenv("KMCB200_KEY_BLOCKS")) ctx->scatter_blocks = std::string(e) != "filter";
	if (const char* e = getenv("KMCB200_KEY_BLOCK_RECORDS")) { const long long v = atoll(e); if (v >= 1024) ctx->key_block_records = (uint64_t)v; }
	if (const char* e = getenv("KMCB200_OVERLAP_WALK")) ctx->overlap_walk = atoi(e) != 0;
	{	// one sort needs two record buffers + the leaves' temporary records (8-byte padded) + ~2 bytes per record of tables: what 60 % of the
		// free HBM (shared by the context's slots) can hold, below 2^32 records (32-bit record indices inside the kernels)
		size_t free_b = 0, total_b = 0;
		if (cudaSetDevice(prm->device) == cudaSuccess && cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && free_b) {
			const uint64_t per_rec = 2ull * 8 * ctx->words + ((ctx->suffix_bytes + ctx->counter_bytes + 7) / 8) * 8 + 2;
			const uint64_t fit = (uint64_t)(0.6 * (double)free_b) / per_rec / std::max<uint64_t>(prm->n_slots, 1);
			ctx->max_block_records = std::max<uint64_t>(1ull << 24, std::min<uint64_t>(fit, (1ull << 32) - (1ull << 24)));
		}
	}
	if (const char* e = getenv("KMCB200_MAX_BLOCK_RECORDS")) { const long long v = atoll(e); if (v >= 1024) ctx->max_block_records = (uint64_t)v; }
	if (const char* e = getenv("KMCB200_MAX_CHUNK_BYTES")) { const long long v = atoll(e); if (v >= (1 << 17) && v < (1ll << 31)) ctx->max_chunk_bytes = (uint64_t)v; }
	if (const char* e = getenv("KMCB200_L2_BITS")) { const int v = atoi(e); if (v >= 1 && v <= 10) ctx->force_b2 = (uint32_t)v; }
	if (const char* e = getenv("KMCB200_LEAF_KERNEL")) { const std::string v(e); ctx->leaf_cta = v == "cta" ? 1 : v == "hash" ? 0 : 2; }
	if (const char* e = getenv("KMCB200_LEAF_CTA")) {
		const std::string v(e);
		if (v == "4:10" || v == "4:12") ctx->leaf_cta_slot_bits = atoi(v.c_str() + 2);
	}
	if (const char* e = getenv("KMCB200_LEAF_MAX_B2")) { const int v = atoi(e); if (v >= 8 && v <= 10) ctx->leaf_max_b2 = (uint32_t)v; }
	if (const char* e = getenv("KMCB200_LEAF_TARGET")) { const int v = atoi(e); if (v >= 128 && v <= 8192) ctx->leaf_target = (uint32_t)v; }
	if (const char* e = getenv("KMCB200_LEAF_FILL_PCT")) { const int v = atoi(e); if (v >= 10 && v <= 85) ctx->leaf_fill_pct = (uint32_t)v; }
	if (const char* e = getenv("KMCB200_LEAF_RATIO0")) { const int v = atoi(e); if (v >= 8 && v <= 256) ctx->leaf_ratio0_q8 = (uint32_t)v; }
	if (const char* e = getenv("KMCB200_LEAF_SLOT_BITS")) { const int b = atoi(e); if (b == 8 || b == 9 || b == 10) ctx->leaf_slot_bits = b; }
	ctx->slots.resize(prm->n_slots);
	auto bail = [&](int rc) { std::string e = ctx->err; kmcb200_destroy(ctx); g_create_error = e; return rc; };
	if (cudaSetDevice(prm->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return bail(KMCB200_ERR_CUDA); }
	if (int rc = DISPATCH_WORDS(ctx, setup_kernels, ctx)) return bail(rc);
	if (int rc = DISPATCH_WORDS(ctx, setup_leaves_w, ctx)) return bail(rc);
	if (cudaFuncSetAttribute(walk_packs_parallel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWalkChunk + 32) != cudaSuccess) {
		ctx->err = "walk_packs_parallel_kernel setup failed"; return bail(KMCB200_ERR_CUDA);
	}
	if (cudaStreamCreateWithFlags(&ctx->compute, cudaStreamNonBlocking) != cudaSuccess) { ctx->err = "cudaStreamCreate failed"; return bail(KMCB200_ERR_CUDA); }
	for (auto& s : ctx->slots) {
		bool ok = cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) == cudaSuccess;
		for (cudaEvent_t* e : {&s.ev_h2d, &s.ev_done, &s.ev_walk}) ok = ok && cudaEventCreateWithFlags(e, cudaEventDisableTiming) == cudaSuccess;
		ok = ok && cudaMalloc(reinterpret_cast<void**>(&s.zero), sizeof(ZeroBlock)) == cudaSuccess;
		ok = ok && cudaMemset(s.zero, 0, sizeof(ZeroBlock)) == cudaSuccess;
		ok = ok && cudaMalloc(reinterpret_cast<void**>(&s.d_lut), ctx->lut_entries * 8) == cudaSuccess;
		ok = ok && cudaMalloc(reinterpret_cast<void**>(&s.msd_seg1), 2 * 8) == cudaSuccess;
		ok = ok && cudaMalloc(reinterpret_cast<void**>(&s.leaf_emit), kMaxLeaves * 4) == cudaSuccess;
		ok = ok && cudaMalloc(reinterpret_cast<void**>(&s.leaf_off), kMaxLeaves * 8) == cudaSuccess;
		ok = ok && cudaMalloc(reinterpret_cast<void**>(&s.msd_start2), 257 * 8) == cudaSuccess;
		ok = ok && cudaMalloc(reinterpret_cast<void**>(&s.msd_start3), (kMaxLeaves + 1) * 8) == cudaSuccess;
		ok = ok && cudaMalloc(reinterpret_cast<void**>(&s.msd_item_base1), 2 * 4) == cudaSuccess;
		ok = ok && cudaMalloc(reinterpret_cast<void**>(&s.msd_item_base2), 257 * 4) == cudaSuccess;
		ok = ok && cudaMalloc(reinterpret_cast<void**>(&s.d_result), 64) == cudaSuccess;
		ok = ok && cudaHostAlloc(reinterpret_cast<void**>(&s.h_result), 64, cudaHostAllocMapped) == cudaSuccess;
		ok = ok && cudaHostGetDevicePointer(reinterpret_cast<void**>(&s.h_result_dev), s.h_result, 0) == cudaSuccess;
		for (cudaEvent_t* e : {&s.ev_begin, &s.ev_expand, &s.ev_sort, &s.ev_count, &s.ev_result}) ok = ok && cudaEventCreate(e) == cudaSuccess;
		for (auto& e : s.ev_pass) ok = ok && cudaEventCreate(&e) == cudaSuccess;
		for (auto& e : s.ev_pack) ok = ok && cudaEventCreateWithFlags(&e, cudaEventDisableTiming) == cudaSuccess;
		if (!ok) { ctx->err = std::string("slot allocation failed: ") + cudaGetErrorString(cudaGetLastError()); return bail(KMCB200_ERR_CUDA); }
	}
	*out_ctx = ctx;
	return KMCB200_OK;
}

void kmcb200_destroy(kmcb200_ctx* ctx)
{
	if (!ctx) return;
	cudaSetDevice(ctx->prm.device);
	cudaDeviceSynchronize();
	for (auto& s : ctx->slots) {
		for (void* p : {(void*)s.recs_a, (void*)s.recs_b, (void*)s.recs_x, (void*)s.d_bin, (void*)s.d_pack_start, (void*)s.pack_nsk, (void*)s.pack_nk, (void*)s.pack_tbase,
				 (void*)s.pack_kbase, (void*)s.pack_done, (void*)s.sk_off, (void*)s.sk_kpre, (void*)s.tile_first, (void*)s.tile_pack, (void*)s.tile_desc, (void*)s.zero, (void*)s.desc,
				 (void*)s.cdesc, (void*)s.d_out, (void*)s.d_lut, (void*)s.d_result, (void*)s.msd_seg1, (void*)s.msd_start2, (void*)s.msd_start3,
				 (void*)s.msd_item_base1, (void*)s.msd_item_base2, (void*)s.msd_item_seg2, (void*)s.msd_item_lo1, (void*)s.msd_item_cnt1,
				 (void*)s.msd_cells, (void*)s.msd_cell_scan, (void*)s.msd_block_sums, (void*)s.leaf_tmp, (void*)s.leaf_emit, (void*)s.leaf_off, (void*)s.d_hist12, (void*)s.d_out_counter, (void*)s.tot_lut, (void*)s.tot_res, (void*)s.d_extras, (void*)s.d_pack_rec, (void*)s.d_blk_of_prefix, (void*)s.d_region_start})
			if (p) cudaFree(p);
		for (auto p : s.h_pack_start) if (p) cudaFreeHost(p);
		for (auto e : s.ev_pack) if (e) cudaEventDestroy(e);
		if (s.h_result) cudaFreeHost(s.h_result);
		if (s.h_pack_rec) cudaFreeHost(s.h_pack_rec);
		for (cudaEvent_t e : {s.ev_begin, s.ev_expand, s.ev_sort, s.ev_count, s.ev_result, s.ev_h2d, s.ev_done, s.ev_walk}) if (e) cudaEventDestroy(e);
		for (auto e : s.ev_pass) if (e) cudaEventDestroy(e);
		if (s.stream) cudaStreamDestroy(s.stream);
	}
	if (ctx->compute) cudaStreamDestroy(ctx->compute);
	delete ctx;
}

const char* kmcb200_last_error(const kmcb200_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }
uint32_t kmcb200_out_rec_bytes(const kmcb200_ctx* ctx) { return ctx ? ctx->suffix_bytes + ctx->counter_bytes : 0; }
uint64_t kmcb200_out_capacity(const kmcb200_ctx* ctx, uint64_t n_rec)
{
	if (!ctx) return 0;
	return ((n_rec + 1) / std::max(ctx->prm.cutoff_min, 1u)) * (uint64_t)(ctx->suffix_bytes + ctx->counter_bytes);   // kb_reader.h:141-150
}
uint64_t kmcb200_lut_entries(const kmcb200_ctx* ctx) { return ctx ? ctx->lut_entries : 0; }
uint64_t kmcb200_kernel_launches(const kmcb200_ctx* ctx) { return ctx ? ctx->launches : 0; }

int kmcb200_host_alloc(kmcb200_ctx* ctx, uint64_t bytes, void** out_ptr)
{
	if (!ctx || !out_ptr) return KMCB200_ERR_INVALID;
	if (int rc = set_device(ctx)) return rc;
	CU(cudaHostAlloc(out_ptr, bytes ? bytes : 1, cudaHostAllocDefault));
	return 0;
}
int kmcb200_host_free(kmcb200_ctx* ctx, void* ptr)
{
	if (!ctx) return KMCB200_ERR_INVALID;
	if (ptr) CU(cudaFreeHost(ptr));
	return 0;
}

static int submit_bin_impl(kmcb200_ctx* ctx, uint32_t slot, const uint8_t* superkmers, uint64_t size, uint64_t n_rec,
	const uint64_t* pack_bytes, uint32_t n_packs, uint8_t* out_suffix, uint64_t out_capacity, uint64_t* lut,
	const uint8_t* extras, uint64_t n_super_kmers, const uint32_t* pack_superkmers);

int kmcb200_submit_bin(kmcb200_ctx* ctx, uint32_t slot, int32_t bin_id,
	const uint8_t* superkmers, uint64_t size, uint64_t n_rec, uint64_t n_plus_x_recs,
	const uint64_t* pack_bytes, const uint64_t* pack_recs, uint32_t n_packs,
	uint8_t* out_suffix, uint64_t out_capacity, uint64_t* lut)
{
	(void)bin_id; (void)n_plus_x_recs; (void)pack_recs;
	return submit_bin_impl(ctx, slot, superkmers, size, n_rec, pack_bytes, n_packs, out_suffix, out_capacity, lut, nullptr, 0, nullptr);
}

int kmcb200_submit_bin_indexed(kmcb200_ctx* ctx, uint32_t slot, int32_t bin_id,
	const uint8_t* superkmers, uint64_t size, uint64_t n_rec, const uint64_t* pack_bytes, uint32_t n_packs,
	const uint8_t* extras, uint64_t n_super_kmers, const uint32_t* pack_superkmers,
	uint8_t* out_suffix, uint64_t out_capacity, uint64_t* lut)
{
	(void)bin_id;
	if (!ctx) return KMCB200_ERR_INVALID;
	if (size && (!extras || !pack_superkmers || !pack_bytes || n_packs == 0)) return fail(ctx, KMCB200_ERR_INVALID, "the indexed form needs extras, pack_bytes and pack_superkmers");
	return submit_bin_impl(ctx, slot, superkmers, size, n_rec, pack_bytes, n_packs, out_suffix, out_capacity, lut, extras, n_super_kmers, pack_superkmers);
}

static int submit_bin_impl(kmcb200_ctx* ctx, uint32_t slot, const uint8_t* superkmers, uint64_t size, uint64_t n_rec,
	const uint64_t* pack_bytes, uint32_t n_packs, uint8_t* out_suffix, uint64_t out_capacity, uint64_t* lut,
	const uint8_t* extras, uint64_t n_super_kmers, const uint32_t* pack_superkmers)
{
	if (int rc = check_slot(ctx, slot)) return rc;
	Slot& s = ctx->slots[slot];
	if (s.busy) return fail(ctx, KMCB200_ERR_BUSY, "slot %u already holds a submitted bin", slot);
	s.have_extras = false;
	if ((size && !superkmers) || !lut || (!out_suffix && out_capacity)) return fail(ctx, KMCB200_ERR_INVALID, "null buffer");
	if (int rc = set_device(ctx)) return rc;
	if (n_rec > ctx->max_block_records || size >= 4 * ctx->max_chunk_bytes) {        // oversized: counted key block by key block, synchronously
		CU(cudaStreamSynchronize(ctx->compute));
		if (int rc = run_oversized_bin(ctx, s, superkmers, size, n_rec, pack_bytes, n_packs, out_suffix, out_capacity, lut, &s.sync_out_bytes, s.sync_stats)) return rc;
		s.busy = true; s.sync_done = true; s.host_lut = lut;
		return 0;
	}
	cudaStream_t st = s.stream;       // copies
	if (int rc = ensure(ctx, s.d_bin, s.bin_cap, size + 64)) return rc;
	if (int rc = ensure(ctx, s.d_out, s.out_cap, out_capacity + 64)) return rc;
	if (size) CU(cudaMemcpyAsync(s.d_bin, superkmers, size, cudaMemcpyHostToDevice, st));
	s.have_extras = false;
	if (extras && size && n_rec) {          // N4: the length bytes + the first record of every pack travel next to the bin
		if (int rc = ensure(ctx, s.d_extras, s.extras_cap, n_super_kmers + 64)) return rc;
		if (int rc = ensure(ctx, s.d_pack_rec, s.pack_rec_cap, (size_t)n_packs + 2)) return rc;
		if (s.h_pack_rec_cap < (size_t)n_packs + 2) {
			CU(cudaStreamSynchronize(st));
			if (s.h_pack_rec) CU(cudaFreeHost(s.h_pack_rec));
			s.h_pack_rec = nullptr; s.h_pack_rec_cap = 0;
			CU(cudaHostAlloc(reinterpret_cast<void**>(&s.h_pack_rec), ((size_t)n_packs + 2 + n_packs / 4) * 8, cudaHostAllocDefault));
			s.h_pack_rec_cap = (size_t)n_packs + 2 + n_packs / 4;
		} else CU(cudaEventSynchronize(s.ev_h2d));          // (the previous bin's copy out of this staging buffer is done)
		uint64_t acc = 0;
		for (uint32_t i = 0; i < n_packs; ++i) { s.h_pack_rec[i] = acc; acc += pack_superkmers[i]; }
		s.h_pack_rec[n_packs] = acc;
		if (acc != n_super_kmers) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "pack_superkmers add up to %llu records, n_super_kmers is %llu", (unsigned long long)acc, (unsigned long long)n_super_kmers);
		CU(cudaMemcpyAsync(s.d_extras, extras, n_super_kmers, cudaMemcpyHostToDevice, st));
		CU(cudaMemcpyAsync(s.d_pack_rec, s.h_pack_rec, ((size_t)n_packs + 1) * 8, cudaMemcpyHostToDevice, st));
		s.have_extras = true;
	}
	const bool with_packs = size != 0 && n_rec != 0;
	if (with_packs) if (int rc = upload_packs(ctx, s, size, pack_bytes, n_packs, st)) return rc;      // on the copy stream, next to the bin
	CU(cudaEventRecord(s.ev_h2d, st));
	CU(cudaStreamWaitEvent(ctx->compute, s.ev_h2d, 0));
	if (int rc = run_bin(ctx, s, s.d_bin, size, n_rec, pack_bytes, n_packs, s.d_out, out_capacity, s.d_lut, s.d_result, ctx->compute, with_packs, s.h_result_dev,
		ctx->overlap_walk ? st : nullptr)) return rc;
	CU(cudaGetLastError());
	CU(cudaEventRecord(s.ev_result, ctx->compute));
	s.busy = true;
	s.host_out = out_suffix; s.host_out_cap = out_capacity; s.host_lut = lut; s.pending_n_rec = n_rec;
	return 0;
}

int kmcb200_wait_bin(kmcb200_ctx* ctx, uint32_t slot, uint64_t* out_bytes, uint64_t stats[4])
{
	if (int rc = check_slot(ctx, slot)) return rc;
	Slot& s = ctx->slots[slot];
	if (!s.busy) return fail(ctx, KMCB200_ERR_INVALID, "slot %u has no submitted bin", slot);
	if (int rc = set_device(ctx)) return rc;
	s.busy = false;
	const bool scan = s.scan_lut;
	s.scan_lut = false;
	if (s.sync_done) {          // an oversized bin: everything happened inside submit
		s.sync_done = false;
		if (scan) { uint64_t acc = s.scan_base; for (uint64_t i = 0; i < ctx->lut_entries; ++i) { const uint64_t x = s.host_lut[i]; s.host_lut[i] = acc; acc += x; } }
		if (out_bytes) *out_bytes = s.sync_out_bytes;
		if (stats) for (int i = 0; i < 4; ++i) stats[i] = s.sync_stats[i];
		return 0;
	}
	CU(cudaEventSynchronize(s.ev_result));
	const uint64_t* r = s.h_result;
	if (r[6] & (kErrPackWalk | kErrRecCount)) {
		cudaStreamSynchronize(s.stream);
		return fail(ctx, KMCB200_ERR_BIN_FORMAT, "bin format error (bits %llu): %s", (unsigned long long)r[6],
			(r[6] & kErrPackWalk) ? "an expander pack does not end on a record boundary" : "the bin does not hold n_rec k-mers");
	}
	const uint64_t bytes = r[4] * (uint64_t)(ctx->suffix_bytes + ctx->counter_bytes);
	if (r[5] || bytes > s.host_out_cap) {
		cudaStreamSynchronize(s.stream);
		return fail(ctx, KMCB200_ERR_CAPACITY, "out_capacity %llu too small for %llu bytes", (unsigned long long)s.host_out_cap, (unsigned long long)bytes);
	}
	if (scan) {          // the completer's prefix sum (kb_completer.cpp:191-201) on the GPU: the LUT arrives as it goes into .kmc_pre
		lut_scan_kernel<<<1, 1024, 0, s.stream>>>(s.d_lut, ctx->lut_entries, s.scan_base);
		ctx->launches++;
	}
	CU(cudaMemcpyAsync(s.host_lut, s.d_lut, ctx->lut_entries * 8, cudaMemcpyDeviceToHost, s.stream));
	if (bytes) CU(cudaMemcpyAsync(s.host_out, s.d_out, bytes, cudaMemcpyDeviceToHost, s.stream));
	CU(cudaStreamSynchronize(s.stream));
	if (out_bytes) *out_bytes = bytes;
	if (stats) for (int i = 0; i < 4; ++i) stats[i] = r[i];
	return 0;
}

int kmcb200_process_bin(kmcb200_ctx* ctx, int32_t bin_id,
	const uint8_t* superkmers, uint64_t size, uint64_t n_rec, uint64_t n_plus_x_recs,
	const uint64_t* pack_bytes, const uint64_t* pack_recs, uint32_t n_packs,
	uint8_t* out_suffix, uint64_t out_capacity, uint64_t* out_bytes, uint64_t* lut, uint64_t stats[4])
{
	if (int rc = kmcb200_submit_bin(ctx, 0, bin_id, superkmers, size, n_rec, n_plus_x_recs, pack_bytes, pack_recs, n_packs, out_suffix, out_capacity, lut)) return rc;
	return kmcb200_wait_bin(ctx, 0, out_bytes, stats);
}

// ---- one bin over several GPUs (SURVEY section 8f N2; the reference's analogue is the big-bucket team sort, raduls_impl.h:672-745)
// Every GPU gets a contiguous SHARE of the bin's packs straight from the host (its own PCIe link), counts the top 12 bits of its share,
// and - once the host has added the histograms up, cut the key space into one contiguous range per GPU and the ranges into key blocks -
// expands its share ONCE, scattering every k-mer into the region of its key block.  Then the records are exchanged: every GPU pulls, for
// each of its own blocks, that block's region from every GPU with peer copies over NVLink (an all-to-all of 8 B x n_rec x (N-1)/N in
// total, the only inter-GPU traffic of this path), sorts and counts its blocks in place, and the per-GPU outputs follow each other in key
// order - the same bytes as one GPU would produce.  Expansion, H2D and sort all shrink with the number of GPUs.
int kmcb200_process_bin_multi(kmcb200_ctx* const* ctxs, uint32_t n_ctx, int32_t bin_id,
	const uint8_t* superkmers, uint64_t size, uint64_t n_rec, const uint64_t* pack_bytes, uint32_t n_packs,
	uint8_t* out_suffix, uint64_t out_capacity, uint64_t* out_bytes, uint64_t* lut, uint64_t stats[4])
{
	if (!ctxs || n_ctx == 0 || !ctxs[0]) return KMCB200_ERR_INVALID;
	kmcb200_ctx* ctx = ctxs[0];
	if (n_ctx > 64) return fail(ctx, KMCB200_ERR_INVALID, "at most 64 contexts");
	for (uint32_t g = 0; g < n_ctx; ++g) {
		if (!ctxs[g] || ctxs[g]->slots.empty() || ctxs[g]->slots[0].busy) return fail(ctx, KMCB200_ERR_INVALID, "context %u is null or busy", g);
		if (ctxs[g]->words != ctx->words || memcmp(&ctxs[g]->prm, &ctx->prm, offsetof(kmcb200_params, device)) != 0) return fail(ctx, KMCB200_ERR_INVALID, "context %u has other parameters", g);
	}
	if ((size && !superkmers) || !lut || (!out_suffix && out_capacity)) return fail(ctx, KMCB200_ERR_INVALID, "null buffer");
	const uint32_t k = ctx->prm.kmer_len;
	if (n_rec == 0 || size == 0 || n_ctx == 1 || 2 * k < 24 || n_rec < 4096ull * n_ctx || !pack_bytes || n_packs < n_ctx)          // nothing to split
		return kmcb200_process_bin(ctx, bin_id, superkmers, size, n_rec, n_rec, pack_bytes, nullptr, n_packs, out_suffix, out_capacity, out_bytes, lut, stats);
	const size_t rec_bytes = (size_t)ctx->words * 8;
	const uint32_t ob = ctx->suffix_bytes + ctx->counter_bytes;

	struct Part {
		uint32_t pack0 = 0, npacks = 0; uint64_t byte0 = 0, bytes = 0;          // the share of the bin this GPU expands
		std::vector<BinChunk> chunks;
		std::vector<uint64_t> hist;                                               // top 12 bits of the share's k-mers
		std::vector<uint64_t> src_off;                                            // [blocks] first record of every block's region in the share's scatter buffer
		std::vector<uint32_t> own;                                                // blocks (global indices) of this GPU's key range, ascending
		std::vector<uint64_t> dst_off;                                            // [own] first record of the block in the GPU's range buffer
		uint64_t n_share = 0, n_range = 0, cap = 0, bytes_out = 0;
		uint64_t r[8] = {};
		std::vector<uint64_t> lut;
		int rc = 0;
		cudaEvent_t ev_scatter = nullptr;
	};
	std::vector<Part> parts(n_ctx);
	{	// contiguous shares of ~size / n_ctx bytes, cut at pack boundaries
		uint64_t pos = 0;
		uint32_t g = 0;
		parts[0].pack0 = 0; parts[0].byte0 = 0;
		for (uint32_t i = 0; i < n_packs; ++i) {
			if (g + 1 < n_ctx && parts[g].npacks > 0 && pos >= (uint64_t)(g + 1) * size / n_ctx && n_packs - i >= n_ctx - g - 1) { ++g; parts[g].pack0 = i; parts[g].byte0 = pos; }
			parts[g].npacks++; parts[g].bytes += pack_bytes[i]; pos += pack_bytes[i];
		}
		if (pos != size) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "expander packs cover %llu bytes but the bin has %llu", (unsigned long long)pos, (unsigned long long)size);
	}
	auto run_all = [&](auto&& fn) {          // one host thread per GPU
		std::vector<std::thread> threads;
		for (uint32_t g = 1; g < n_ctx; ++g) threads.emplace_back([&, g] { parts[g].rc = fn(g); });
		parts[0].rc = fn(0);
		for (auto& t : threads) t.join();
		for (uint32_t g = 0; g < n_ctx; ++g) if (parts[g].rc) { if (g) ctx->err = ctxs[g]->err; return parts[g].rc; }
		return 0;
	};
	// ---- phase A: own share host -> device, counting expansion
	if (int rc = run_all([&](uint32_t g) -> int {
		kmcb200_ctx* ctx = ctxs[g];
		Slot& s = ctx->slots[0];
		Part& P = parts[g];
		if (int rc = set_device(ctx)) return rc;
		if (P.npacks == 0) { P.hist.assign(4096, 0); return 0; }
		uint64_t dev_bytes = 0;
		if (int rc = plan_chunks(ctx, P.bytes, pack_bytes + P.pack0, P.npacks, P.chunks, &dev_bytes)) return rc;
		if (int rc = ensure(ctx, s.d_bin, s.bin_cap, dev_bytes + 64)) return rc;
		for (const BinChunk& c : P.chunks) CU(cudaMemcpyAsync(s.d_bin + c.dev_off, superkmers + P.byte0 + c.byte0, c.bytes, cudaMemcpyHostToDevice, ctx->compute));
		return count_top12(ctx, s, P.chunks, pack_bytes + P.pack0, P.hist, ctx->compute);
	})) return rc;
	std::vector<uint64_t> hist(4096, 0);
	uint64_t total = 0;
	for (uint32_t g = 0; g < n_ctx; ++g) for (uint32_t q = 0; q < 4096; ++q) { hist[q] += parts[g].hist[q]; parts[g].n_share += parts[g].hist[q]; }
	for (uint64_t v : hist) total += v;
	if (total != n_rec) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "bin format error: the bin holds %llu k-mers, not n_rec = %llu", (unsigned long long)total, (unsigned long long)n_rec);
	// ---- key ranges (~n_rec / n_ctx k-mers each) and their key blocks
	std::vector<uint32_t> cut(n_ctx + 1, 4096);
	cut[0] = 0;
	{
		uint64_t acc = 0;
		uint32_t g = 1;
		for (uint32_t q = 0; q < 4096 && g < n_ctx; ++q) {
			acc += hist[q];
			while (g < n_ctx && acc * n_ctx >= (uint64_t)g * n_rec) cut[g++] = q + 1;
		}
	}
	std::vector<KeyBlock> blocks;          // all GPUs' blocks, ascending
	std::vector<uint32_t> owner;
	uint64_t limit = std::min(ctx->max_block_records, ctx->key_block_records);
	for (int attempt = 0; attempt < 8; ++attempt) {
		blocks.clear(); owner.clear();
		for (uint32_t g = 0; g < n_ctx; ++g) {
			const size_t before = blocks.size();
			if (int rc = bisect_blocks(ctx, hist, cut[g], cut[g + 1], limit, blocks)) return rc;
			owner.resize(blocks.size(), g);
			(void)before;
		}
		if (blocks.size() <= kExpandMaxBlocks) break;
		limit *= 2;                          // too many blocks for one scattering expansion: larger ones
	}
	if (blocks.size() > kExpandMaxBlocks) return fail(ctx, KMCB200_ERR_INVALID, "bin too skewed for %u GPUs: %zu key blocks", n_ctx, blocks.size());
	for (uint32_t g = 0; g < n_ctx; ++g) {
		Part& P = parts[g];
		P.src_off.resize(blocks.size());
		uint64_t acc = 0;
		for (size_t b = 0; b < blocks.size(); ++b) {
			uint64_t c = 0;
			const uint32_t lo = blocks[b].prefix << (12 - blocks[b].bits), len = 1u << (12 - blocks[b].bits);
			for (uint32_t q = lo; q < lo + len; ++q) c += P.hist[q];
			P.src_off[b] = acc; acc += c;          // (source regions need no alignment: they are only ever copied from)
		}
		acc = 0;
		for (size_t b = 0; b < blocks.size(); ++b) if (owner[b] == g) {
			acc = (acc + 1) & ~1ull;
			P.own.push_back((uint32_t)b); P.dst_off.push_back(acc);
			acc += blocks[b].n; P.n_range += blocks[b].n;
		}
		P.cap = ((P.n_range + 1) / std::max(ctx->prm.cutoff_min, 1u)) * (uint64_t)ob;
		P.lut.resize(ctx->lut_entries);
	}
	auto share_count = [&](uint32_t g, size_t b) { return (b + 1 < blocks.size() ? parts[g].src_off[b + 1] : parts[g].n_share) - parts[g].src_off[b]; };
	auto drop_events = [&]() {
		for (uint32_t g = 0; g < n_ctx; ++g) if (parts[g].ev_scatter) { cudaSetDevice(ctxs[g]->prm.device); cudaStreamSynchronize(ctxs[g]->compute); cudaEventDestroy(parts[g].ev_scatter); parts[g].ev_scatter = nullptr; }
		cudaSetDevice(ctx->prm.device);
	};
	// ---- phase B: every GPU scatters its share into per-block regions (one expansion); buffers of the exchange are sized
	if (int rc = run_all([&](uint32_t g) -> int {
		kmcb200_ctx* ctx = ctxs[g];
		Slot& s = ctx->slots[0];
		Part& P = parts[g];
		if (int rc = set_device(ctx)) return rc;
		cudaStream_t st = ctx->compute;
		if (!P.ev_scatter) CU(cudaEventCreateWithFlags(&P.ev_scatter, cudaEventDisableTiming));
		uint64_t max_n = 0;
		for (uint32_t b : P.own) max_n = std::max(max_n, blocks[b].n);
		if (int rc = ensure(ctx, s.recs_a, s.recs_a_cap, (P.n_share + 2) * rec_bytes)) return rc;                       // the share, scattered by block
		if (int rc = ensure(ctx, s.recs_x, s.recs_x_cap, (P.n_range + P.own.size() + 2) * rec_bytes)) return rc;       // the range, block after block
		if (int rc = ensure(ctx, s.recs_b, s.recs_b_cap, (max_n + 2) * rec_bytes)) return rc;                         // one block's scratch
		if (int rc = ensure(ctx, s.d_out, s.out_cap, P.cap + 64)) return rc;
		if (int rc = ensure_totals(ctx, s, st)) return rc;
		if (P.npacks) {
			if (int rc = setup_scatter(ctx, s, blocks, P.src_off, st)) return rc;
			if (int rc = scatter_chunks(ctx, s, P.chunks, pack_bytes + P.pack0, (uint32_t)blocks.size(), s.recs_a, st)) return rc;
			// (the share must have delivered what its counting pass announced - otherwise the exchange below would copy garbage)
			std::vector<unsigned long long> got(blocks.size());
			CU(cudaMemcpyAsync(got.data(), s.d_out_counter, blocks.size() * 8, cudaMemcpyDeviceToHost, st));
			CU(cudaStreamSynchronize(st));
			for (size_t b = 0; b < blocks.size(); ++b) if (got[b] != share_count(g, b)) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "bin format error on GPU %u's share", g);
		}
		CU(cudaEventRecord(P.ev_scatter, st));
		return 0;
	})) { drop_events(); return rc; }
	// ---- phase C: the exchange (every GPU pulls its blocks' regions from every GPU), then sort + count block after block, in place
	int rc_c = run_all([&](uint32_t h) -> int {
		kmcb200_ctx* ctx = ctxs[h];
		Slot& s = ctx->slots[0];
		Part& P = parts[h];
		if (int rc = set_device(ctx)) return rc;
		cudaStream_t st = ctx->compute;
		for (uint32_t g = 0; g < n_ctx; ++g) if (g != h && ctxs[g]->prm.device != ctx->prm.device) {
			int can = 0;
			cudaDeviceCanAccessPeer(&can, ctx->prm.device, ctxs[g]->prm.device);
			if (can) { cudaError_t e = cudaDeviceEnablePeerAccess(ctxs[g]->prm.device, 0); if (e != cudaSuccess) cudaGetLastError(); }      // (already enabled is fine)
		}
		for (uint32_t g = 0; g < n_ctx; ++g) CU(cudaStreamWaitEvent(st, parts[g].ev_scatter, 0));
		for (size_t i = 0; i < P.own.size(); ++i) {
			const uint32_t b = P.own[i];
			uint64_t sub = 0;
			for (uint32_t g = 0; g < n_ctx; ++g) {
				const uint64_t c = share_count(g, b);
				if (c) CU(cudaMemcpyPeerAsync(s.recs_x + (P.dst_off[i] + sub) * rec_bytes, ctx->prm.device,
					ctxs[g]->slots[0].recs_a + parts[g].src_off[b] * rec_bytes, ctxs[g]->prm.device, c * rec_bytes, st));
				sub += c;
			}
			if (sub != blocks[b].n) return fail(ctx, KMCB200_ERR_CUDA, "internal error: block %u has %llu records, expected %llu", b, (unsigned long long)sub, (unsigned long long)blocks[b].n);
			if (int rc = sort_count_block(ctx, s, s.recs_x + P.dst_off[i] * rec_bytes, s.recs_b, blocks[b], s.d_out, P.cap, s.tot_lut, s.tot_res, nullptr, st)) return rc;
		}
		CU(cudaMemcpyAsync(P.r, s.tot_res, 64, cudaMemcpyDeviceToHost, st));
		CU(cudaMemcpyAsync(P.lut.data(), s.tot_lut, ctx->lut_entries * 8, cudaMemcpyDeviceToHost, st));
		CU(cudaStreamSynchronize(st));
		return 0;
	});
	drop_events();          // (also waits for every GPU: nobody still copies out of a neighbour's scatter buffer)
	if (rc_c) return rc_c;
	uint64_t pos = 0, acc[3] = {0, 0, 0};
	for (uint32_t g = 0; g < n_ctx; ++g) {
		if (parts[g].r[6]) return fail(ctx, KMCB200_ERR_BIN_FORMAT, "bin format error on GPU %u's key range", g);
		parts[g].bytes_out = parts[g].r[4] * (uint64_t)ob;
		if (parts[g].r[5] || pos + parts[g].bytes_out > out_capacity) return fail(ctx, KMCB200_ERR_CAPACITY, "out_capacity %llu too small", (unsigned long long)out_capacity);
		pos += parts[g].bytes_out;
	}
	// ---- outputs in key order, LUTs and statistics added up
	pos = 0;
	for (uint64_t i = 0; i < ctx->lut_entries; ++i) lut[i] = 0;
	for (uint32_t g = 0; g < n_ctx; ++g) {
		kmcb200_ctx* c = ctxs[g];
		cudaSetDevice(c->prm.device);
		if (parts[g].bytes_out) { cudaError_t e = cudaMemcpyAsync(out_suffix + pos, c->slots[0].d_out, parts[g].bytes_out, cudaMemcpyDeviceToHost, c->compute); if (e != cudaSuccess) return fail(ctx, KMCB200_ERR_CUDA, "D2H of GPU %u's records failed: %s", g, cudaGetErrorString(e)); }
		pos += parts[g].bytes_out;
		for (int i = 0; i < 3; ++i) acc[i] += parts[g].r[i];
		if (parts[g].n_range) for (uint64_t i = 0; i < ctx->lut_entries; ++i) lut[i] += parts[g].lut[i];
	}
	for (uint32_t g = 0; g < n_ctx; ++g) { cudaSetDevice(ctxs[g]->prm.device); cudaStreamSynchronize(ctxs[g]->compute); }
	cudaSetDevice(ctx->prm.device);
	if (out_bytes) *out_bytes = pos;
	if (stats) { stats[0] = acc[0]; stats[1] = acc[1]; stats[2] = acc[2]; stats[3] = n_rec; }
	return 0;
}

int kmcb200_sort_records(kmcb200_ctx* ctx, void* recs, void* tmp, uint64_t n, uint32_t rec_bytes, uint32_t key_bytes)
{
	if (int rc = check_slot(ctx, 0)) return rc;
	if (rec_bytes != (uint32_t)ctx->words * 8) return fail(ctx, KMCB200_ERR_INVALID, "rec_bytes %u does not match the context (k=%u -> %d bytes)", rec_bytes, ctx->prm.kmer_len, ctx->words * 8);
	if (key_bytes < 1 || key_bytes > rec_bytes || !recs || !tmp) return fail(ctx, KMCB200_ERR_INVALID, "bad key_bytes / buffers");
	if (int rc = set_device(ctx)) return rc;
	Slot& s = ctx->slots[0];
	if (s.busy) return fail(ctx, KMCB200_ERR_BUSY, "slot 0 busy");
	const int where = (key_bytes & 1) ? 1 : 0;      // kb_sorter.h:776-779
	if (n == 0) return where;
	cudaStream_t st = ctx->compute;
	if (int rc = ensure(ctx, s.recs_a, s.recs_a_cap, n * rec_bytes)) return rc;
	if (int rc = ensure(ctx, s.recs_b, s.recs_b_cap, n * rec_bytes)) return rc;
	CU(cudaMemcpyAsync(s.recs_a, recs, n * rec_bytes, cudaMemcpyHostToDevice, st));
	bool in_b = false;
	if (int rc = DISPATCH_WORDS(ctx, launch_sort, ctx, s, s.recs_a, s.recs_b, n, key_bytes, 8u * key_bytes, (int)kHistNone, 0u, st, &in_b)) return rc;
	CU(cudaMemcpyAsync(where ? tmp : recs, in_b ? s.recs_b : s.recs_a, n * rec_bytes, cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));
	return where;
}

// ---- device-level entry points
int kmcb200_dev_process_bin(kmcb200_ctx* ctx, uint32_t slot, const uint8_t* d_superkmers, uint64_t size, uint64_t n_rec,
	const uint64_t* pack_bytes, uint32_t n_packs, uint8_t* d_out, uint64_t out_capacity, uint64_t* d_lut, uint64_t* d_result, void* stream)
{
	if (int rc = check_slot(ctx, slot)) return rc;
	if (int rc = set_device(ctx)) return rc;
	Slot& s = ctx->slots[slot];
	s.have_extras = false;          // (a length-byte array of an earlier kmcb200_submit_bin_indexed on this slot does not describe this bin)
	return run_bin(ctx, s, d_superkmers, size, n_rec, pack_bytes, n_packs, d_out, out_capacity, d_lut, d_result, stream ? (cudaStream_t)stream : ctx->compute);
}

int kmcb200_dev_expand(kmcb200_ctx* ctx, uint32_t slot, const uint8_t* d_superkmers, uint64_t size, uint64_t n_rec,
	const uint64_t* pack_bytes, uint32_t n_packs, void* d_recs, uint64_t* d_result, void* stream)
{
	if (int rc = check_slot(ctx, slot)) return rc;
	if (int rc = set_device(ctx)) return rc;
	Slot& s = ctx->slots[slot];
	cudaStream_t st = stream ? (cudaStream_t)stream : ctx->compute;
	if (n_rec == 0) return 0;
	s.have_extras = false;
	CU(cudaEventRecord(s.ev_begin, st));
	if (int rc = stage_expand(ctx, s, d_superkmers, size, n_rec, pack_bytes, n_packs, d_recs, st)) return rc;
	if (d_result) {
		if (int rc = zero_async(ctx, d_result, 64, st)) return rc;
		finish_result_kernel<<<1, 32, 0, st>>>(d_result, n_rec, s.zero->status, nullptr, nullptr);
		ctx->launches++;
	}
	CU(cudaEventRecord(s.ev_expand, st));
	s.ran_expand = true; s.ran_sort = s.ran_count = false;
	return 0;
}

int kmcb200_dev_sort(kmcb200_ctx* ctx, uint32_t slot, void* d_recs, void* d_tmp, uint64_t n, uint32_t key_bytes, int hist_ready, void* stream)
{
	if (int rc = check_slot(ctx, slot)) return rc;
	if (key_bytes < 1 || key_bytes > (uint32_t)ctx->words * 8) return fail(ctx, KMCB200_ERR_INVALID, "key_bytes %u", key_bytes);
	if (int rc = set_device(ctx)) return rc;
	Slot& s = ctx->slots[slot];
	cudaStream_t st = stream ? (cudaStream_t)stream : ctx->compute;
	const int where = (key_bytes & 1) ? 1 : 0;
	if (n == 0) return where;
	if (!hist_ready) CU(cudaEventRecord(s.ev_expand, st));
	bool in_b = false;
	if (int rc = DISPATCH_WORDS(ctx, launch_sort, ctx, s, d_recs, d_tmp, n, key_bytes, hist_ready ? 2u * ctx->prm.kmer_len : 8u * key_bytes, hist_ready ? s.hist_mode : (int)kHistNone, s.last_n_packs, st, &in_b)) return rc;
	CU(cudaEventRecord(s.ev_sort, st));
	s.ran_sort = true; s.ran_count = false;
	if (!hist_ready) s.ran_expand = false;
	return in_b ? 1 : 0;
}

int kmcb200_dev_count(kmcb200_ctx* ctx, uint32_t slot, const void* d_sorted, uint64_t n, uint8_t* d_out, uint64_t out_capacity,
	uint64_t* d_lut, uint64_t* d_result, void* stream)
{
	if (int rc = check_slot(ctx, slot)) return rc;
	if (int rc = set_device(ctx)) return rc;
	Slot& s = ctx->slots[slot];
	cudaStream_t st = stream ? (cudaStream_t)stream : ctx->compute;
	CU(cudaEventRecord(s.ev_sort, st));
	if (int rc = stage_count(ctx, s, d_sorted, n, d_out, out_capacity, d_lut, d_result, st)) return rc;
	finish_result_kernel<<<1, 32, 0, st>>>(d_result, n, nullptr, nullptr, nullptr);
	ctx->launches++;
	CU(cudaEventRecord(s.ev_count, st));
	s.ran_count = true; s.ran_expand = false; s.ran_sort = false;
	return 0;
}

int kmcb200_stage_times(kmcb200_ctx* ctx, uint32_t slot, float* ms, uint32_t capacity)
{
	if (int rc = check_slot(ctx, slot)) return rc;
	if (!ms || capacity < 3) return fail(ctx, KMCB200_ERR_INVALID, "ms capacity");
	if (int rc = set_device(ctx)) return rc;
	Slot& s = ctx->slots[slot];
	for (uint32_t i = 0; i < capacity; ++i) ms[i] = 0.f;
	if (s.ran_count) CU(cudaEventSynchronize(s.ev_count));
	else if (s.ran_sort) CU(cudaEventSynchronize(s.ev_sort));
	else if (s.ran_expand) CU(cudaEventSynchronize(s.ev_expand));
	if (s.ran_expand) CU(cudaEventElapsedTime(&ms[0], s.ev_begin, s.ev_expand));
	if (s.ran_sort) {
		CU(cudaEventElapsedTime(&ms[1], s.ev_expand, s.ev_sort));
		for (int p = 0; p < s.n_passes_run && 3 + p < (int)capacity; ++p) CU(cudaEventElapsedTime(&ms[3 + p], s.ev_pass[p], s.ev_pass[p + 1]));
	}
	if (s.ran_count) CU(cudaEventElapsedTime(&ms[2], s.ev_sort, s.ev_count));
	return s.ran_sort ? s.n_passes_run : 0;
}

int kmcb200_stage_names(kmcb200_ctx* ctx, uint32_t slot, char* buf, uint32_t capacity)
{
	if (int rc = check_slot(ctx, slot)) return rc;
	if (!buf || !capacity) return fail(ctx, KMCB200_ERR_INVALID, "buffer");
	Slot& s = ctx->slots[slot];
	std::string out;
	for (int p = 0; p < s.n_passes_run; ++p) { if (p) out += ","; out += s.pass_names[p] ? s.pass_names[p] : "?"; }
	snprintf(buf, capacity, "%s", out.c_str());
	return s.n_passes_run;
}

}  // extern "C"

#include "db_writer.inl"
#include "splitter.inl"
#include "stage0.inl"
#include "fastx.inl"
#include "small_k.inl"
