/*
 * cg_internal.h -- shared declarations of libcitus_gpu.so (host C++ and CUDA).
 * Not part of the C-ABI (include/citus_gpu.h is).
 */
#ifndef CG_INTERNAL_H
#define CG_INTERNAL_H

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>

#include "citus_gpu.h"

#define CG_BLCKSZ 8192
#define CG_PAGE_HEADER 24
#define CG_BYTES_PER_PAGE (CG_BLCKSZ - CG_PAGE_HEADER)
#define CG_FIRST_LOGICAL_OFFSET (2ull * CG_BYTES_PER_PAGE)

int cg_set_error(int code, const char *fmt, ...);
extern unsigned long long g_cg_launches;   /* kernels launched by this library (every <<<>>> site) */

#define CG_CUDA(call)                                                                        \
	do {                                                                                     \
		cudaError_t e__ = (call);                                                            \
		if (e__ != cudaSuccess)                                                              \
			return cg_set_error(CG_ECUDA, "%s failed: %s (%s:%d)", #call,                     \
								cudaGetErrorString(e__), __FILE__, __LINE__);                 \
	} while (0)

/* stream-ordered scratch that is returned to the pool on every exit path */
struct CgAsyncBuf
{
	void *p = nullptr;
	cudaStream_t stream = nullptr;
	CgAsyncBuf() {}
	CgAsyncBuf(const CgAsyncBuf &) = delete;
	CgAsyncBuf &operator=(const CgAsyncBuf &) = delete;
	~CgAsyncBuf() { if (p) cudaFreeAsync(p, stream); }
	cudaError_t alloc(size_t bytes, cudaStream_t s) { stream = s; return cudaMallocAsync(&p, bytes ? bytes : 8, s); }
	template <typename T> T *as() const { return (T *) p; }
};

struct CgContext
{
	int device = -1;
	int sm_count = 0;
	cudaStream_t compute = nullptr;  /* kernels */
	cudaStream_t copy = nullptr;     /* side stream for H2D staging */
	/* pinned staging ring */
	static const int kPinnedBlocks = 4;
	size_t pinned_block_bytes = 0;
	uint8_t *pinned[kPinnedBlocks] = {nullptr, nullptr, nullptr, nullptr};
	cudaEvent_t pinned_free[kPinnedBlocks] = {nullptr, nullptr, nullptr, nullptr};
	cudaEvent_t ev_a = nullptr, ev_b = nullptr;
	int stage_threads = 16;
	cudaStream_t own_compute = nullptr;
	/* DMA staging: shards in flight */
	static const int kDmaDepth = 3;
	cudaEvent_t dma_done[kDmaDepth] = {nullptr, nullptr, nullptr};
	cudaEvent_t dma_copied = nullptr;
	int dma_slot = 0;
	uint8_t *meta_pinned[kDmaDepth] = {nullptr, nullptr, nullptr};   /* pinned ring for per-scan metadata */
	size_t meta_cap[kDmaDepth] = {0, 0, 0};
	/* device buffers of the shards in flight (grown on demand, reused: no allocator in the scan loop) */
	struct DevBuf { uint8_t *p = nullptr; size_t cap = 0; };
	DevBuf slot_arena[kDmaDepth], slot_raw[kDmaDepth], slot_meta[kDmaDepth];
	/* decode streams: the decompression of consecutive shards rotates over kDmaDepth streams, so that the
	 * decode kernels of all shards in flight (each a latency-bound chain per value stream) can be resident together */
	cudaStream_t decode_stream[kDmaDepth] = {nullptr, nullptr, nullptr};
	unsigned decode_rr = 0;
	cudaEvent_t decoded[kDmaDepth] = {nullptr, nullptr, nullptr};
	uint8_t *zstd_scratch = nullptr;             /* literal buffers of the resident zstd decoders */
	size_t zstd_scratch_bytes = 0;
	unsigned long long *d_stage_err = nullptr;   /* error flags raised by staging kernels of cg_shard_stage */
	/* per-launch profiling */
	bool profiling = false;
	std::vector<cudaEvent_t> prof_events;   /* pairs */
	size_t prof_used = 0;
};
int cg_prof_mark(CgContext *ctx, cudaStream_t stream);   /* records the next event of the pool when profiling */
CgContext *cg_ctx(void);   /* NULL + error set if cg_init has not run */
int cg_ensure_pinned(CgContext *ctx);

/* ------------------------------------------------------------------------------ *
 *  HBM layout of a staged shard.
 *  arena: every (chunk group, staged column) owns
 *     [exists bitmap, padded with zero bits to a multiple of 16 B]
 *     [value stream, padded to a multiple of 16 B]
 *     [rank directory: uint32 per 64 rows = number of non-NULL rows before the block]
 *                                       (only when the chunk has NULLs)
 *  all 16-byte aligned, in chunk-group-major order (so a block of consecutive chunk
 *  groups is one contiguous H2D copy).  A compressed value stream (lz4 / pglz) keeps its
 *  on-disk bytes in that place; its decompressed value slot lives in a second area behind
 *  the chunk-group regions, filled by cg_decompress_kernel, and values_off points there.
 * ------------------------------------------------------------------------------ */
struct DevChunkCol
{
	uint64_t values_off;
	uint64_t exists_off;
	uint64_t rank_off;      /* valid iff value_count != row_count */
	uint32_t value_count;   /* non-NULL rows = decompressed_size / attlen */
	uint32_t row_count;
};

struct CgShard
{
	int natts = 0;
	std::vector<CgColumnDesc> columns;       /* all attributes */
	std::vector<int32_t> staged;             /* staged attribute indexes */
	std::vector<int32_t> slot_of_att;        /* att -> staged slot or -1 */
	uint64_t rows = 0;
	uint64_t nchunkgroups = 0;
	uint8_t *d_arena = nullptr;
	uint64_t arena_bytes = 0;
	DevChunkCol *d_chunkcols = nullptr;      /* [nchunkgroups][nstaged] */
	std::vector<DevChunkCol> h_chunkcols;
	std::vector<uint32_t> h_stream_bytes;    /* uncompressed value-stream bytes per (chunk group, staged column) */
	std::vector<uint32_t> cg_rows;           /* rows per chunk group */
	/* host copy of the metadata needed for chunk-group skipping */
	std::vector<CgStripe> stripes;
	std::vector<CgSkipNode> nodes;
	std::vector<uint64_t> stripe_first_cg;   /* first chunk-group id of each stripe */
	/* chunk groups surviving the last WHERE list (SelectedChunkMask), cached on the device */
	uint32_t *d_selected = nullptr;
	std::vector<uint32_t> h_selected;
	bool sel_valid = false;
	int32_t sel_pushdown = 0, sel_nquals = 0;
	CgQual sel_quals[CG_MAX_QUALS];
	int32_t sel_nqexpr = 0;
	int8_t sel_qexpr[CG_MAX_QEXPR];
	int64_t sel_filtered = 0;
	uint32_t sel_nullmask = 0;               /* plan columns that have NULLs in some chunk group of the second part */
	/* the list is ordered [chunk groups without NULLs in the plan columns | the rest] */
	std::vector<uint8_t> sel_slots;
	uint32_t sel_nfast = 0;
	uint32_t sel_max_cg_rows = 0;
	uint64_t sel_rows_fast = 0, sel_rows_total = 0;   /* rows of the first part / of the whole selection */
	uint64_t algorithmic_bytes_per_cg_col(uint64_t cg, int slot) const
	{
		const DevChunkCol &c = h_chunkcols[cg * staged.size() + slot];
		return (uint64_t) h_stream_bytes[cg * staged.size() + slot] + (c.row_count + 7) / 8;
	}
};

/* ------------------------------------------------------------------------------ *
 *  Kernel plan (passed by value as a __grid_constant__ parameter).
 * ------------------------------------------------------------------------------ */
#define CG_KMAX_COLS 8
#define CG_KMAX_WORDS 32

enum { CG_MODE_GLOBAL = 0, CG_MODE_DENSE = 1, CG_MODE_HASH = 2 };

/* word ops reuse CG_WORD_* from the public header */

struct KAgg
{
	int8_t kind;        /* CG_AGG_* */
	int8_t nfactors;
	int8_t is_float;
	int8_t nlimbs;      /* integer SUM: 1 = whole sum fits int64, 2 = (low32, high) limb words */
	int8_t pcol[3];     /* plan-column index of every factor */
	int8_t word0;       /* first accumulator word (count(x): its NULL-count word) */
	int8_t nullword;    /* word counting NULL inputs among the group's rows:
						 * non-NULL inputs = rows in group (word 0) - this word */
	int8_t ovchk;       /* integer term with no proven bound: every factor and product is checked for int64
						 * overflow (CG_ERRFLAG_TERM_OVERFLOW) */
	int8_t pad[2];
	int64_t a[3];
	int64_t b[3];
	int64_t bound;      /* nlimbs == 1: every |term| must be <= bound */
	int64_t tbound;     /* integer SUM: the caller-proven bound on |term| whatever nlimbs is (0 = unknown) */
};

struct KPlan
{
	const uint8_t *arena;
	const DevChunkCol *chunkcols;
	const uint32_t *selected;     /* chunk-group ids to scan */
	uint32_t nselected;
	int32_t nstaged;

	int32_t ncols;                /* plan columns (deduplicated) */
	uint8_t slot[CG_KMAX_COLS];   /* staged slot */
	uint8_t len[CG_KMAX_COLS];
	uint8_t isfloat[CG_KMAX_COLS];

	int32_t nquals;
	uint8_t qcol[CG_MAX_QUALS];
	uint8_t qop[CG_MAX_QUALS];
	int64_t qk[CG_MAX_QUALS];
	/* integer conjuncts in range form: pass iff ((x >= qlo && x <= qhi) != qneg) */
	int64_t qlo[CG_MAX_QUALS];
	int64_t qhi[CG_MAX_QUALS];
	uint8_t qneg[CG_MAX_QUALS];

	int32_t ngroup;
	uint8_t gcol[CG_MAX_GROUP_COLS];

	int32_t naggs;
	KAgg aggs[CG_MAX_AGGS];

	/* group table */
	int32_t mode;
	int32_t nwords;               /* accumulator words per group; word 0 = rows in group */
	int32_t stride;               /* 64-bit words per entry (hash: key + words, padded) */
	uint64_t *table;              /* accumulator words: dense [capacity+1][stride]; hash [capacity+2][stride] */
	int64_t *hkeys;               /* hash: key of every slot, [capacity+2] */
	uint64_t capacity;            /* hash: power of two */
	int32_t hash_shift;           /* hash: 64 - log2(capacity) */
	int64_t key_min;              /* dense (two group columns: minimum of the first) */
	int64_t key_min1;             /* dense, two group columns: minimum of the second */
	uint64_t range1;              /* ... and its range; slot = (k0 - key_min) * range1 + (k1 - key_min1) */
	uint8_t wordop[CG_KMAX_WORDS];

	unsigned long long *stats;    /* [0] rows scanned [1] rows removed [2] error flags
								   * [3] rows added to packed words [4] rows drained from packed words */
	/* shared-memory kernel (cg_scan_small.cu): accumulator words that get a private cell per lane;
	 * the NULL-input counters and the NULL-key group stay on (rare) global atomics */
	int8_t hot_of_word[CG_KMAX_WORDS];   /* word -> cell index or -1 */
	int32_t nhot;
	/* optimistic packed accumulators (direct-indexed tables): packed[slot] += (term << shift) + 1 */
	uint64_t *packed;
	int32_t pack_shift;
	int32_t pack_word;            /* accumulator word the packed sum belongs to */
	/* WHERE tree in postfix form over the atoms above (0 tokens = AND of all atoms) */
	int32_t nqexpr;
	int8_t qexpr[CG_MAX_QEXPR];
	/* work units: a chunk group is cut into `slices` row ranges of slice_rows rows (the last one shorter) when a launch has
	 * too few chunk groups to fill the GPU (small shards); 1 = one unit per chunk group */
	int32_t slices;
	uint32_t slice_rows;
	uint32_t max_cg_rows;         /* largest chunk group of the launch (host-known; 0 = unknown: no slicing) */
};

/* plan of the specialised kernel (cg_scan_fast.cu): column roles in fixed order
 * [range quals..., group key, summed columns...] */
struct FPlan
{
	const uint8_t *arena;
	const DevChunkCol *chunkcols;
	const uint32_t *selected;
	uint32_t nselected;
	int32_t nstaged;
	int32_t nquals, nsums, mode;
	uint32_t flags;               /* CG_FAST_* */
	uint8_t slot[6];
	uint8_t qneg[2];
	uint8_t slimbs[3];
	uint8_t sword[3];
	int64_t qlo[2], qhi[2];
	int64_t sbound[3];
	uint64_t *table;
	int64_t *hkeys;
	uint64_t capacity;
	int32_t hash_shift;
	int32_t stride;
	int64_t key_min;
	unsigned long long *stats;
	uint64_t *packed;             /* non-NULL: count(*) and sum number pack_sum share one word */
	int32_t pack_shift;
	int32_t pack_sum;
	int32_t slices;               /* see KPlan */
	uint32_t slice_rows;
	uint32_t max_cg_rows;
};
/* how many row ranges a chunk group is cut into so that `nselected` chunk groups give a launch of `grid_full` CTAs at least two
 * units per CTA; step = rows one CTA iteration covers (slice boundaries stay multiples of it) */
static inline void cg_choose_slices(uint32_t nselected, uint32_t grid_full, uint32_t step, uint32_t max_chunk_rows, int32_t *slices, uint32_t *slice_rows)
{
	uint32_t s = nselected ? (2u * grid_full + nselected - 1) / nselected : 1u;
	uint32_t max_s = (max_chunk_rows + step - 1) / step;
	if (s > max_s) s = max_s;
	if (s < 1) s = 1;
	uint32_t rows = ((max_chunk_rows + s - 1) / s + step - 1) / step * step;
	*slices = (int32_t) ((max_chunk_rows + rows - 1) / rows);
	*slice_rows = rows;
}

#define CG_FAST_PAIRED 1u       /* pair lanes so that one reduction instruction covers both words of a group */
#define CG_FAST_NO_HINTS 2u     /* disable the L2 eviction hints (A/B measurements) */

#define CG_HASH_EMPTY ((int64_t) 0x8000000000000000ull)
#define CG_ERRFLAG_TABLE_FULL 1ull
#define CG_ERRFLAG_NULL_MULTIKEY 2ull
#define CG_ERRFLAG_KEY_RANGE 4ull
#define CG_ERRFLAG_SUM_BOUND 8ull
#define CG_ERRFLAG_DECOMPRESS 16ull
#define CG_ERRFLAG_VARLENA 32ull
#define CG_ERRFLAG_TERM_OVERFLOW 64ull   /* an integer aggregate argument left int64 */
#define CG_COMM_TAIL 16           /* words behind an accumulator array that travel with it in a combine (cg_comm.cu) */
#define CG_STAT_PACKED_ADDED 3
#define CG_STAT_PACKED_DRAINED 4

struct CgPartial
{
	CgScanDesc desc;
	std::vector<CgColumnDesc> columns;
	int mode = CG_MODE_GLOBAL;
	int nwords = 1;
	int stride = 1;
	uint64_t capacity = 0;      /* addressable slots (dense: domain size, hash: pow2) */
	uint64_t entries = 0;       /* allocated entries incl. the special ones */
	int64_t key_min = 0, key_max = -1;
	int64_t key_min1 = 0;        /* two group columns, direct-indexed: second column's minimum and range */
	uint64_t range1 = 0;
	int64_t max_rows = 0;
	uint8_t wordop[CG_KMAX_WORDS];
	KAgg aggs[CG_MAX_AGGS];
	uint64_t *d_table = nullptr;
	int64_t *d_hkeys = nullptr;            /* hash mode: separate key array (same allocation as d_table) */
	unsigned long long *d_stats = nullptr;   /* 8 words */
	/* optimistic packing */
	uint64_t *d_packed = nullptr;
	int pack_shift = 0;
	int pack_word = 0;
	bool packing_enabled = false;
	bool packed_dirty = false;
	bool wide_dirty = false;        /* the wide accumulator words hold something (not only the packed words) */
	bool table_initialised = false;
	unsigned long long *h_ret = nullptr;    /* pinned: statistics + row counts read back by export_rows */
	bool read_packed_direct = false; /* result rows were decoded from the packed words since the last drain */
	int launches_since_drain = 0;
	uint64_t rows_since_drain = 0;  /* rows scanned into packed words since the last drain (upper bound) */
	/* scratch for export */
	int64_t *d_out_keys = nullptr;
	uint64_t *d_out_words = nullptr;
	uint8_t *d_out_nulls = nullptr;
	unsigned long long *d_out_count = nullptr;
	uint64_t out_capacity = 0;
	/* pinned host buffer the result rows are fetched through */
	uint8_t *h_out = nullptr;
	size_t h_out_cap = 0;
};

/* cg_scan.cu */
int cg_launch_scan(CgContext *ctx, const KPlan &plan, bool any_nulls, bool all8, cudaStream_t stream);
/* one chunk buffer to move from the raw (page-payload) device buffer to its aligned arena slot */
struct RealignItem
{
	uint64_t src;       /* byte offset in the raw buffer (any alignment) */
	uint64_t dst;       /* arena offset, 16-byte aligned */
	uint32_t len;       /* bytes to copy */
	uint32_t padded;    /* slot size: bytes beyond len are zeroed */
};
void cg_realign_set_tma(int on);
int cg_launch_realign(const uint8_t *raw, uint8_t *arena, const RealignItem *items, uint64_t nitems, cudaStream_t stream);

/* cg_decompress.cu: one compressed value stream (arena offset src, comp_len bytes) to decode into its
 * value slot (arena offset dst, raw_len bytes, zero padding up to `padded`) */
struct DecodeItem
{
	uint64_t src;
	uint64_t dst;
	uint32_t comp_len;
	uint32_t raw_len;
	uint32_t padded;
	uint32_t kind;      /* CG_COMPRESSION_LZ4 / CG_COMPRESSION_PGLZ / CG_COMPRESSION_ZSTD */
};
void cg_decompress_set_lz4_lanes(int on);
void cg_decompress_set_lz4_lane_warps(int n);
int cg_launch_decompress(CgContext *ctx, uint8_t *arena, const DecodeItem *items, const DecodeItem *h_items, uint64_t nitems,
						 unsigned long long *err, unsigned long long flag, cudaStream_t stream);

/* cg_varlena.cu: one varlena value stream (arena offset src, raw_len bytes: the on-disk stream, or its decompressed
 * slot) to decode into a dense fixed-width array of `count` values at arena offset dst */
struct VarlenaItem
{
	uint64_t src;
	uint64_t dst;
	uint32_t raw_len;
	uint32_t count;
	uint32_t kind;      /* CG_TYPE_NUMERIC / CG_TYPE_BPCHAR1 */
	uint32_t scale;
};
int cg_launch_varlena_decode(CgContext *ctx, uint8_t *arena, const VarlenaItem *items, uint64_t nitems, unsigned long long *err,
							 unsigned long long flag, cudaStream_t stream);
/* class and numeric scale of a column; the width the scan kernels see (a varlena column is decoded to a fixed width) */
static inline int cg_type_class(const CgColumnDesc &c) { return c.type_class & 0xff; }
static inline int cg_type_scale(const CgColumnDesc &c) { return c.type_class >> 8; }
static inline bool cg_is_varlena(const CgColumnDesc &c) { return c.attlen < 0; }
static inline int cg_decoded_len(const CgColumnDesc &c) { return c.attlen > 0 ? c.attlen : (cg_type_class(c) == CG_TYPE_NUMERIC ? 8 : 1); }

/* cg_scan_small.cu */
bool cg_small_eligible(const KPlan &plan);
int cg_launch_scan_small(CgContext *ctx, const KPlan &plan, bool all8, cudaStream_t stream);
/* cg_scan_fast.cu */
int cg_launch_scan_fast(CgContext *ctx, const FPlan &plan, cudaStream_t stream);
int cg_launch_drain(CgPartial *p, cudaStream_t stream);
int cg_launch_rank(CgContext *ctx, const uint8_t *arena, const DevChunkCol *chunkcols, uint64_t first,
				   uint64_t count, cudaStream_t stream);
int cg_launch_table_init(CgPartial *p, cudaStream_t stream);
int cg_launch_export(CgPartial *p, uint64_t out_capacity, int64_t *d_keys, uint8_t *d_nulls, uint64_t *d_words,
					 unsigned long long *d_count, cudaStream_t stream);
int cg_launch_export_packed(CgPartial *p, uint64_t out_capacity, int64_t *d_keys, uint8_t *d_nulls, uint64_t *d_words,
							unsigned long long *d_count, cudaStream_t stream);
int cg_launch_merge(CgPartial *p, const int64_t *d_keys, const uint8_t *d_nulls, const uint64_t *d_words,
					int64_t nrows, cudaStream_t stream);

/* cg_jit.cpp: plan-specialised kernels through NVRTC */
int cg_jit_level(void);
void cg_jit_set_level(int level);     /* CG_JIT: 0 = off, 1 = where no specialised ahead-of-time kernel applies (default), 2 = always */
/* nullable: bit c set = plan column c may have NULLs in the chunk groups of this launch (the kernel then reads
 * its exists bitmap + rank directory wherever a chunk's value_count differs from its row count) */
int cg_launch_scan_jit(CgContext *ctx, const KPlan &plan, uint32_t nullable, cudaStream_t stream, bool *launched, bool *used_packed,
					   bool *packed_only = nullptr);

/* cg_partition.cu: the same without host synchronisation (counts stay on the device; d_counts has P + 1 words,
 * the last one counts rows whose hash fell in no interval) */
int cg_partition_index_async(const int64_t *d_keys, const uint8_t *d_nulls, int64_t n, int32_t key_len, int32_t by_hash,
							 const int32_t *mins, const int32_t *maxs, int32_t P, int32_t *d_index, int64_t *d_counts);
int cg_partition_scatter_async(const int32_t *d_index, int64_t n, int32_t P, const int32_t *h_order, const int64_t *const *d_cols,
							   int32_t ncols, int64_t *const *d_out);

/* Scatter straight into the receive buffers of other ranks (peer-mapped memory).  Output positions are
 * destination-major: positions [pos_begin[d], pos_begin[d + 1]) belong to rank d, whose buffer holds column c at
 * base[d] + c * stride[d]; a row the local scatter would place at index i of the send order lands at adj[d] + i. */
#define CG_MAX_RANKS 16
struct CgPeerScatter
{
	int64_t *base[CG_MAX_RANKS];
	int64_t stride[CG_MAX_RANKS];
	int64_t adj[CG_MAX_RANKS];
	int32_t pos_begin[CG_MAX_RANKS + 1];
	int32_t nranks;
};
/* called after routing, the histogram and the offset scan are enqueued and before the scatter is launched: the
 * caller exchanges the counts and says where the rows go */
struct CgScatterHook
{
	int (*fn)(void *arg, CgPeerScatter *out);
	void *arg;
};

int cg_partition_route_scatter_async(const int64_t *d_keys, const uint8_t *d_nulls, int64_t n, int32_t key_len, int32_t by_hash,
									 const int32_t *mins, const int32_t *maxs, int32_t P, const int32_t *h_order,
									 const int64_t *const *d_cols, int32_t ncols, int64_t *const *d_out, int64_t *d_counts,
									 cudaEvent_t after_counts, const CgScatterHook *peer_hook = nullptr);

/* cg_comm.cu */
void cg_comm_set_peer_window(int on);

/* cg_plan.cpp */
int cg_partial_shape(CgPartial *p, const CgScanDesc *desc, const CgColumnDesc *columns, int32_t natts,
					 int64_t key_min, int64_t key_max, int64_t max_rows);
bool cg_build_fast_plan(const CgScanDesc *desc, const KPlan &plan, bool all8, FPlan *fast);
int cg_build_plan(const CgScanDesc *desc, const CgColumnDesc *columns, int natts,
				  const std::vector<int32_t> *slot_of_att, CgPartial *partial, KPlan *plan,
				  bool *all8);

#endif
