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
	/* the library's last enqueue on the compute stream was a scan launch: CG_CHAIN_* (see cg_chain_scan) */
	int scan_chain = 0;
	/* scan profiling: one (start, end) event pair per chain of scan launches */
	bool profiling = false;
	std::vector<cudaEvent_t> prof_events;
	size_t prof_used = 0;
	uint64_t prof_launches = 0;
};
enum { CG_CHAIN_NONE = 0, CG_CHAIN_OPEN = 1, CG_CHAIN_CLOSED = 2 };
/* called by the scan launch helpers right before a scan launch on `stream`; *overlap = true: launch it with programmatic
 * stream serialization (it may overlap the previous scan launch).  chainable = false for the interpretive kernels. */
int cg_chain_scan(CgContext *ctx, cudaStream_t stream, bool chainable, bool *overlap);
/* called before every other enqueue of the library on `stream`: ends the chain of scan launches when `stream` is the
 * compute stream */
int cg_chain_end(CgContext *ctx, cudaStream_t stream);
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

/*
 * Narrow image of an 8-byte integer chunk column (cg_narrow.cu), built at staging next to the plain arena for the
 * ahead-of-time fast kernel: value = base + field in wrapping uint64, field r at bits [r * width, r * width + width) of
 * a bit stream of 64-bit little-endian words.  Rows [64 k, 64 k + 64) take exactly the words [k * width, k * width +
 * width), so a warp's 64 consecutive rows are one contiguous run of at most 256 bytes; the stream holds
 * ceil(rows / 64) * width words, 16-byte aligned.  width = CG_NARROW_NONE: no image (NULLs in the chunk column, or the
 * column has no image in this shard).
 */
#define CG_NARROW_NONE 255u
#define CG_NARROW_MAX_WIDTH 32u
struct DevPackCol
{
	uint64_t off;           /* byte offset of the bit stream in CgShard.d_narrow */
	int64_t base;           /* minimum of the chunk column */
	uint32_t width;         /* bits per row, 0 .. CG_NARROW_MAX_WIDTH, or CG_NARROW_NONE */
	uint32_t pad;
};
/* words of a chunk column's bit stream */
static inline __host__ __device__ uint64_t cg_narrow_words(uint32_t rows, uint32_t width)
{
	return (uint64_t) ((rows + 63u) / 64u) * width;
}

/* the device copy of a plan's IN / NOT IN codes (2 * CG_MAX_IN_VALUES words, allocated by the first scan with a list):
 * written with cudaMemcpyAsync on the compute stream before a launch whose codes differ from the last ones written
 * (last), so that the copy is ordered behind every earlier launch that reads the buffer (cg_set_stream synchronises the
 * old stream before switching).  The copies come from a ring of pinned slots: a slot is rewritten once the copy recorded
 * in its event has run, so the host does not wait behind the stream's earlier kernels.  A partial owns one for its
 * scans, a shard one for its row scans (cg_scan_shard_rows) */
struct CgSetBuf
{
	uint64_t *d_sets = nullptr;
	std::vector<uint64_t> last;
	static const int kSlots = 4;
	uint64_t *h_sets[kSlots] = {nullptr, nullptr, nullptr, nullptr};
	cudaEvent_t copied[kSlots] = {nullptr, nullptr, nullptr, nullptr};
	int slot = 0;
	void release()
	{
		cudaFree(d_sets);
		d_sets = nullptr;
		for (int i = 0; i < kSlots; i++)
		{
			if (copied[i]) { cudaEventSynchronize(copied[i]); cudaEventDestroy(copied[i]); }
			if (h_sets[i]) cudaFreeHost(h_sets[i]);
			copied[i] = nullptr; h_sets[i] = nullptr;
		}
		last.clear();
	}
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
	std::vector<int64_t> sel_lists;          /* the IN lists the WHERE atoms of that list read (cg_where_lists) */
	int64_t sel_filtered = 0;
	uint32_t sel_nullmask = 0;               /* plan columns that have NULLs in some chunk group of the second part */
	/* the list is ordered [chunk groups without NULLs in the plan columns | the rest] */
	std::vector<uint8_t> sel_slots;
	uint32_t sel_nfast = 0;
	uint32_t sel_max_cg_rows = 0;
	uint64_t sel_rows_fast = 0, sel_rows_total = 0;   /* rows of the first part / of the whole selection */
	/* narrow images (cg_narrow.cu): a staged column has them in every NULL-free chunk group or in none */
	uint8_t *d_narrow = nullptr;
	uint64_t narrow_bytes = 0;
	DevPackCol *d_packcols = nullptr;        /* [nchunkgroups][nstaged] */
	std::vector<DevPackCol> h_packcols;
	std::vector<uint8_t> slot_narrow;        /* per staged slot: 1 = the column has images */
	/* the IN-list codes of the row scans (cg_scan_shard_rows); they never touch the selection cache above */
	CgSetBuf row_sets;
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
#define CG_KMAX_WORDS CG_MAX_WORDS

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
	int8_t filt;        /* the aggregate has a FILTER: nullword counts the rows that gave no input (NULL input or
						 * filter not TRUE); count(*) then gets a nullword of its own (count = rows - it) */
	int8_t barg;        /* bool_and / bool_or: the argument is the predicate tree argexpr[a] over the filter pool;
						 * nullword counts the rows that gave no input (argument UNKNOWN, or FILTER not TRUE) */
	/* CG_AGG_VARIANCE: word0 (and nlimbs, bound) hold sum(x) as a sum's words do; sum(x^2) is qlimbs words from qword on:
	 * 1 = the whole sum, 2 = (x^2 low 32 bits, x^2 >> 32), 4 = the four 32-bit limbs of the unsigned 128-bit x^2.  0 for
	 * the other kinds.  These two bytes sit in what was padding before a[], so no offset moves (the generated kernels of
	 * plans without the kind restate the struct without them, cg_jit.cpp) */
	int8_t qlimbs;
	int8_t qword;
	int64_t a[3];
	int64_t b[3];
	int64_t bound;      /* nlimbs == 1 (and CG_AGG_VARIANCE with a term bound): every |term| must be <= bound */
	int64_t tbound;     /* integer SUM: the caller-proven bound on |term| whatever nlimbs is (0 = unknown) */
};

/* the list of one IN / NOT IN atom: codes sets[off .. off + len), len = 0 for a list of NULLs only; steps = ceil(log2(len)),
 * the fixed length of its binary search; nnull = the list has a NULL element */
struct KSet
{
	uint16_t off;
	uint16_t len;
	uint8_t steps;
	uint8_t nnull;
	uint8_t pad[2];
};

/* the code of a value in its column's comparison order, as unsigned: an integer with its sign bit flipped; a float8 (bits)
 * through f8_ordered after -0.0 -> +0.0 (every NaN already maps to one code) */
static inline __host__ __device__ uint64_t cg_set_code(int64_t v, bool isfloat)
{
	if (!isfloat) return (uint64_t) v ^ 0x8000000000000000ull;
	uint64_t u = (uint64_t) v;
	if (u == 0x8000000000000000ull) u = 0;
	if ((u & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return ~0ull;
	return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

/* the other side of a column atom "x <op> y" (x = the atom's plan column): y is plan column col2.  Integer-like sides
 * compare x * mul with y (right = 0) or x with y * mul (right = 1), exactly in 128 bits; mul = 10^(scale difference), 1
 * for equal scales, char(1) and float sides (float sides compare their cg_set_code) */
struct KCmp
{
	int64_t mul;
	uint8_t col2;
	uint8_t right;
	uint8_t pad[6];
};

/* one CASE arm (CgCaseArm) with its columns as plan columns: WHEN tree when[0 .. nwhen) over the filter atoms (0 tokens =
 * ELSE); result form CG_CASE_*: the constant a[0], or the product over nfactors of (a[f] + b[f] * v[pcol[f]]) */
struct KArm
{
	int64_t a[3];
	int64_t b[3];
	int8_t nwhen;
	int8_t form;
	int8_t nfactors;
	int8_t pcol[3];
	int8_t when[CG_MAX_QEXPR];
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
	/* aggregate FILTER atoms in the form of the WHERE atoms (0 when no aggregate has a filter), and per aggregate
	 * its postfix tree over them (0 tokens = no filter) */
	int32_t nfquals;
	uint8_t fcol[CG_MAX_FILTER_QUALS];
	uint8_t fop[CG_MAX_FILTER_QUALS];
	int64_t fk[CG_MAX_FILTER_QUALS];
	int64_t flo[CG_MAX_FILTER_QUALS];
	int64_t fhi[CG_MAX_FILTER_QUALS];
	uint8_t fneg[CG_MAX_FILTER_QUALS];
	int32_t nfexpr[CG_MAX_AGGS];
	int8_t fexpr[CG_MAX_AGGS][CG_MAX_QEXPR];
	/* bool_and / bool_or: per aggregate its predicate argument, a postfix tree over the same atoms (0 tokens = none).
	 * These two fields and the composite key's stay behind fexpr: the generated kernels of plans with neither restate the
	 * struct up to fexpr only (cg_jit.cpp) */
	int32_t nargexpr[CG_MAX_AGGS];
	int8_t argexpr[CG_MAX_AGGS][CG_MAX_QEXPR];
	/* composite key (CgScanDesc.composite_key): the key is the mixed-radix code over gcol[0..ngroup) (cg_plan.cpp), then
	 * a one-column key with key_min 0 and no NULL group.  Column g's digit is 0 for NULL, v - kmin[g] + 1 otherwise, and
	 * a value with v - kmin[g] >= kradix[g] - 1 is out of range.  Last, so that the generated kernels of other plans
	 * restate the struct without them (cg_jit.cpp) */
	int32_t composite;
	int64_t kmin[CG_MAX_GROUP_COLS];
	uint64_t kradix[CG_MAX_GROUP_COLS];
	/* IN / NOT IN atoms (qop / fop CG_OP_IN, CG_OP_NOT_IN): sets = every list's sorted, distinct codes (cg_set_code), back to
	 * back in device memory; an atom's list is qset / fset [q].  Behind the composite key, so that the generated kernels of
	 * plans without lists restate the struct without them (cg_jit.cpp) */
	const uint64_t *sets;
	KSet qset[CG_MAX_QUALS];
	KSet fset[CG_MAX_FILTER_QUALS];
	/* column atoms (qop / fop CG_OP_COL_*): the other side of WHERE / pool atom q is qcc / fcc [q].  Behind the lists, so
	 * that the generated kernels of plans without column atoms restate the struct without them (cg_jit.cpp) */
	KCmp qcc[CG_MAX_QUALS];
	KCmp fcc[CG_MAX_FILTER_QUALS];
	/* CASE arguments (CgScanDesc.case_arms): aggregate a with cnarms[a] > 0 takes its term from arms[cfirst[a] ..
	 * cfirst[a] + cnarms[a]).  Behind the column atoms, so that the generated kernels of plans without CASE restate the
	 * struct without them (cg_jit.cpp) */
	int32_t ncase;                /* arms in use, 0 = no CASE */
	int8_t cfirst[CG_MAX_AGGS];
	int8_t cnarms[CG_MAX_AGGS];
	KArm arms[CG_MAX_CASE_ARMS];
};

static inline __host__ __device__ bool cg_op_is_column(int op) { return op >= CG_OP_COL_LT && op <= CG_OP_COL_NE; }

static inline bool cg_desc_has_filters(const CgScanDesc *d)
{
	for (int a = 0; a < d->naggs && a < CG_MAX_AGGS; a++)
		if (d->nfilter_expr[a] > 0) return true;
	return false;
}

/* some aggregate's argument is a CASE */
static inline bool cg_desc_has_case(const CgScanDesc *d)
{
	for (int a = 0; a < d->naggs && a < CG_MAX_AGGS; a++)
		if (d->case_narms[a] > 0) return true;
	return false;
}

/* the filter atom pool is read by some FILTER, some bool_and / bool_or argument or some CASE arm */
static inline bool cg_desc_uses_pool(const CgScanDesc *d)
{
	for (int a = 0; a < d->naggs && a < CG_MAX_AGGS; a++)
		if (d->nfilter_expr[a] > 0 || d->narg_expr[a] > 0 || d->case_narms[a] > 0) return true;
	return false;
}

static inline bool cg_kind_is_bool(int kind) { return kind == CG_AGG_BOOL_AND || kind == CG_AGG_BOOL_OR; }
static inline bool cg_kind_is_bit(int kind) { return kind == CG_AGG_BIT_AND || kind == CG_AGG_BIT_OR; }
/* an integer aggregate whose sum(x) words follow sum's form (word0, nlimbs, bound) */
static inline __host__ __device__ bool cg_kind_sums(int kind) { return kind == CG_AGG_SUM || kind == CG_AGG_VARIANCE; }
static inline __host__ __device__ bool cg_plan_has_variance(const KAgg *aggs, int naggs)
{
	for (int a = 0; a < naggs; a++)
		if (aggs[a].kind == CG_AGG_VARIANCE) return true;
	return false;
}

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
	/* nonzero: every column the plan reads has narrow images in this shard, and the kernel reads those instead of the
	 * arena (set by cg_scan_shard; the chunk groups the fast kernel takes are NULL-free, so all of them have images) */
	int32_t narrow;
	const uint8_t *narrow_base;
	const DevPackCol *packcols;
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
	/* the codes of the IN / NOT IN lists of the scan in flight */
	CgSetBuf sets;
};

/* cg_scan.cu */
int cg_launch_scan(CgContext *ctx, const KPlan &plan, bool all8, cudaStream_t stream);
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
void cg_decompress_set_zstd_coop(int on);
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
/* char(1) is decoded to a 2-byte slot so that the kernels' signed loads see the byte unsigned (0..255) */
static inline int cg_decoded_len(const CgColumnDesc &c) { return c.attlen > 0 ? c.attlen : (cg_type_class(c) == CG_TYPE_NUMERIC ? 8 : 2); }

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

/* cg_partition.cu: per-partition exclusive scan of per-block counts on ctx->compute, with all SMs.  d_block[b * P + p]
 * becomes the sum of d_block[b' * P + p] over b' < b, d_tot[p] the sum over all nblocks (> 0) blocks; scratch holds the
 * chunk sums until it is returned to the pool in stream order. */
int partition_scan_blocks(CgContext *ctx, unsigned long long *d_block, unsigned long long *d_tot, int64_t nblocks, int P, CgAsyncBuf *scratch);

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

/* cg_join.cu: build the chained join table over sides[0] and run the plan over the joined rows of sides[1] (cg_join_aggregate;
 * a plan column's slot is its joined-row attribute: build columns first, then probe columns), on `stream` */
int cg_launch_join_aggregate(CgContext *ctx, const KPlan &plan, const CgJoinSide *const sides[2], cudaStream_t stream);

/* cg_scan_rows.cu: the row scan (cg_scan_shard_rows).  A tile is CG_ROW_TILE rows of one chunk group starting at row0 (a
 * multiple of it); its selection bits are the bitmap words [word, word + ceil(rows / 64)) */
#define CG_ROW_TILE 2048
#define CG_MAX_ROW_COLS 16
struct RowTile
{
	uint64_t word;
	uint32_t cg;
	uint32_t row0;
};
/* the projected columns of a row scan: staged slot, decoded width and float flag of every output column, and the caller's
 * device arrays (nulls[c] may be NULL when the column has no NULLs in the chunk groups scanned) */
struct KRowOut
{
	const uint8_t *arena;
	const DevChunkCol *chunkcols;
	int32_t nstaged;
	int32_t ncols;
	uint8_t slot[CG_MAX_ROW_COLS];
	uint8_t len[CG_MAX_ROW_COLS];
	uint8_t isfloat[CG_MAX_ROW_COLS];
	int64_t *cols[CG_MAX_ROW_COLS];
	uint8_t *nulls[CG_MAX_ROW_COLS];
};
/* pass 1: the WHERE tree of plan (arena, chunkcols and nstaged set; selected unused) over every tile: bitmap bits and the
 * passing rows of every tile in counts[t] */
int cg_launch_rows_select(CgContext *ctx, const KPlan &plan, const RowTile *tiles, int64_t ntiles, uint64_t *bitmap,
						  unsigned long long *counts, cudaStream_t stream);
/* pass 3: the passing rows of every tile to offsets[t] + their rank in the tile */
int cg_launch_rows_write(CgContext *ctx, const KRowOut &out, const RowTile *tiles, int64_t ntiles, const uint64_t *bitmap,
						 const unsigned long long *offsets, cudaStream_t stream);

/* cg_comm.cu */
void cg_comm_set_peer_window(int on);

/* cg_plan.cpp */
/* the composite key codec (the only place that knows the code): radix[g] of every key column and the domain D; CG_EINVAL
 * for a descriptor that is not composite or has a bad column count, CG_EUNSUPPORTED when D > 2^63 */
int cg_key_codec(const CgScanDesc *desc, uint64_t *radix, unsigned __int128 *domain);
/* identity of the key codec, folded into what ranks agree on before they combine (0 for the other key forms) */
uint64_t cg_key_codec_id(const CgScanDesc *desc);
int cg_partial_shape(CgPartial *p, const CgScanDesc *desc, const CgColumnDesc *columns, int32_t natts,
					 int64_t key_min, int64_t key_max, int64_t max_rows);
bool cg_build_fast_plan(const CgScanDesc *desc, const KPlan &plan, bool all8, FPlan *fast);
/* narrow images of a freshly staged shard (cg_narrow.cu); best effort: when they cannot be built the shard stays as staged */
void cg_shard_build_narrow(CgContext *ctx, CgShard *sh);
/* set_codes (may be NULL): receives the codes plan->qset / fset index (KPlan.sets is left NULL for the caller to point at
 * their device copy) */
int cg_build_plan(const CgScanDesc *desc, const CgColumnDesc *columns, int natts,
				  const std::vector<int32_t> *slot_of_att, CgPartial *partial, KPlan *plan,
				  bool *all8, std::vector<uint64_t> *set_codes = nullptr);
/* the WHERE half of cg_build_plan alone, for a descriptor without aggregates, group columns, FILTER or CASE (the row scan):
 * plan columns, atoms, IN-list codes, column atoms and the tree; no group table */
int cg_build_where_plan(const CgScanDesc *desc, const CgColumnDesc *columns, int natts, const std::vector<int32_t> *slot_of_att,
						KPlan *plan, std::vector<uint64_t> *set_codes);
/* what of the IN lists a WHERE list reads, for comparing two WHERE lists (empty without IN / NOT IN atoms) */
std::vector<int64_t> cg_where_lists(const CgScanDesc *desc);

#endif
