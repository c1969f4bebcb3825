/*
 * citus_gpu.h -- C-ABI of libcitus_gpu.so: the H100 (sm_90a) implementation of Citus's
 * columnar shard-scan / partial-aggregate / combine / hash-repartition hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8(b)).  Plain C, plain pointers and
 * sizes, no CUDA or torch types.  Every entry point returns 0 on success or a CG_E* code;
 * the message is read with cg_last_error() (thread-local).  Nothing here longjmps: the
 * PostgreSQL-side glue turns a non-zero return into ereport(ERROR) (INTEGRATION.md).
 *
 * Reference interfaces each block replaces are cited as file:line under
 * the Citus sources' src/.
 */
#ifndef CITUS_GPU_H
#define CITUS_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CG_OK 0
#define CG_EINVAL 1        /* bad argument / unsupported plan shape */
#define CG_ECUDA 2         /* CUDA runtime error (message has the cudaError string) */
#define CG_ENOMEM 3
#define CG_ECORRUPT 4      /* relation image inconsistent with its metadata */
#define CG_ETABLEFULL 5    /* group table too small: retry with a larger expected_groups */
#define CG_EUNSUPPORTED 6  /* valid SQL, but outside what the GPU path handles: caller falls
                            * back to the reference's row-at-a-time executor */
#define CG_ECOMM 8          /* NCCL / communicator error, or another rank failed the query */
#define CG_ERETRY_UNPACKED 7 /* an optimistic packed accumulator overflowed (see cg_partial_set_packing):
                            * nothing wrong was returned; call cg_partial_set_packing(p, 0),
                            * cg_partial_reset(p) and scan again */

const char *cg_last_error(void);

/* ---------------------------------------------------------------------------------- *
 *  Device context.  One per process (a PostgreSQL backend is one process; CUDA is
 *  initialised lazily in the backend, never in the postmaster -- SURVEY.md 7.3).
 * ---------------------------------------------------------------------------------- */
int cg_init(int device_ordinal);          /* idempotent */
int cg_device_count(int *count);
int cg_synchronize(void);                 /* waits for the library's streams */
/* Run the kernels on a stream owned by the caller (a CUstream / cudaStream_t handle passed as
 * void *; NULL restores the library's own stream; (void *) 1 is CUDA's legacy default stream,
 * cudaStreamLegacy).  Lets a host that already has a stream -- e.g. the one its NCCL
 * collectives are ordered on -- keep everything in one queue. */
int cg_set_stream(void *cuda_stream);
/* Device timing of the fused scan kernels.  Consecutive scan launches on the library's stream --
 * the shards of one query -- form a chain whose launches overlap (programmatic dependent launch of
 * the fast and the generated scan kernels); any other work the library enqueues on that stream
 * ends the chain.  Between begin and collect, a CUDA event is recorded on the stream before the
 * first launch of every chain and one where the chain ends (no event between two launches of a
 * chain, no host synchronisation).  collect ends the open chain, waits for the events and returns
 * the number of scan kernel launches, the summed busy time of the chains and the longest chain
 * (ms); total / launches is the average time per launch. */
int cg_profile_begin(void);
int cg_profile_collect(int32_t *launches, double *total_ms, double *max_ms);
/* number of CUDA kernels this library has launched so far (all kernels, all entry points) */
uint64_t cg_kernel_launches(void);
/* Plan-specialised kernels (cg_jit.cpp): query shapes without an ahead-of-time specialisation are
 * written out as straight-line CUDA and compiled with NVRTC the first time they are seen (CG_JIT=0
 * turns this off; the interpretive kernels then run everything).  Counters, and a GPU-less check that
 * a query shape generates valid sm_90a code: kind = 0 plain aggregate / 1 shared-memory cells /
 * 2 global table; source (may be NULL) receives the generated CUDA. */
uint64_t cg_jit_launches(void);
uint64_t cg_jit_compiles(void);
/* run-time switches (tests and A/B measurements drive every kernel family through the same C-ABI calls):
 *   "jit" 0 | 1 | 2, "force_general" 0 | 1     which kernel family scans
 *   "realign_tma" 0 | 1                         cp.async.bulk or plain-load form of the page realign kernel
 *   "lz4_lanes" 0 | 1 | 2 (< 0 = default = 2)    LZ4 streams: eight lanes per stream | a lane per stream | by launch size
 *   "lz4_lane_warps" n                          (probe) warps per SM the lane-per-stream kernel spreads a launch over
 *   "zstd_coop" 0 | 1 (< 0 = default = 1)       Zstandard frames: one lane decodes a frame | the warp cooperates on it
 *   "peer_window" 0 | 1                         exchange steps over NCCL | over the IPC-mapped peer window; the same
 *                                               value on every rank
 *   "narrow_images" 0 | 1 (default 1)           shards staged from then on get no narrow images | get them where they
 *                                               fit (a shard without them is what a failed image build leaves)
 * An unknown name is CG_EINVAL. */
int cg_set_option(const char *name, int64_t value);
struct CgScanDesc;
struct CgColumnDesc;
int cg_jit_compile_check(const struct CgScanDesc *desc, const struct CgColumnDesc *columns, int32_t natts, int64_t key_min,
						 int64_t key_max, int64_t max_rows, int32_t *kind, char *source, size_t source_len);
/* the same for the kernel form that reads NULL-bearing chunks: bit a of nullable_atts = attribute a may be NULL */
int cg_jit_compile_check_nullable(const struct CgScanDesc *desc, const struct CgColumnDesc *columns, int32_t natts, int64_t key_min,
								  int64_t key_max, int64_t max_rows, uint32_t nullable_atts, int32_t *kind, char *source,
								  size_t source_len);
/* Pin the calling thread (and threads it creates afterwards: the staging threads) to the CPUs
 * of the device's NUMA node, so that host pages it first-touches and the DMA reads of them stay
 * on the socket the GPU hangs off.  *node = the node, or -1 when nothing was changed (single
 * node, sysfs unreadable, cpuset excludes the node).  cg_numa_unbind restores the old mask. */
int cg_numa_bind(int32_t *node);
int cg_numa_unbind(void);
void cg_shutdown(void);

/* ---------------------------------------------------------------------------------- *
 *  Relation metadata: field-for-field what the reference keeps per stripe / chunk, in this header's own
 *  layout (NOT memory-compatible with ColumnChunkSkipNode / StripeMetadata: Datum min / max become int64 or
 *  float8 bits, bool / enum fields become int32); pg_glue/gpu_columnar_agg.c build_relation_image() converts.
 * ---------------------------------------------------------------------------------- */

/* include/columnar/columnar_compression.h:17-27 CompressionType */
enum { CG_COMPRESSION_NONE = 0, CG_COMPRESSION_PGLZ = 1, CG_COMPRESSION_LZ4 = 2, CG_COMPRESSION_ZSTD = 3 };

/* include/columnar/columnar.h:85-111 ColumnChunkSkipNode
 * (catalog columnar.chunk, backend/columnar/sql/citus_columnar--11.1-1.sql:48-64) */
typedef struct CgSkipNode
{
	int32_t has_minmax;
	int32_t compression_type;
	int64_t min_value;          /* by-value Datum: sign-extended integer or float8 bits */
	int64_t max_value;
	uint64_t row_count;
	uint64_t value_offset;      /* valueChunkOffset, relative to the stripe's file_offset */
	uint64_t value_length;
	uint64_t exists_offset;
	uint64_t exists_length;
	uint64_t decompressed_size; /* decompressedValueSize */
	int32_t compression_level;
	int32_t reserved;
} CgSkipNode;

/* include/columnar/columnar_metadata.h:21-42 StripeMetadata (catalog columnar.stripe) */
typedef struct CgStripe
{
	uint64_t id;
	uint64_t file_offset;       /* logical offset of the stripe (page aligned) */
	uint64_t data_length;
	uint64_t row_count;
	uint64_t first_row_number;
	uint32_t column_count;
	uint32_t chunk_row_count;   /* chunk_group_row_limit the stripe was written with */
	uint32_t chunk_count;
	uint32_t skipnode_base;     /* node(col,chunk) = nodes[skipnode_base + col*chunk_count + chunk] */
} CgStripe;

enum { CG_TYPE_INT = 0, CG_TYPE_FLOAT = 1,
	   /* by-reference (varlena) types whose values are scaled integers or one character: attlen = -1.
		* numeric(p, s): type_class = CG_TYPE_NUMERIC | s << 8; the column then behaves like an int8 column holding
		* value * 10^s (aggregate results carry the scale; cg_numeric_out prints them), a value with more fractional
		* digits than s, NaN, +-Infinity or outside [-2^63, 2^63 - 1] fails the scan with CG_EUNSUPPORTED.
		* char(1): CG_TYPE_BPCHAR1, behaves like an integer column holding the character's byte as an UNSIGNED value
		* 0..255: PostgreSQL compares bpchar under the C collation with memcmp, so in a single-byte encoding 0xE9 sorts
		* above 'A'.  Quals, group keys, min / max and the skip nodes' min_value / max_value all use that value; it is
		* not the sign-extended int1 of a 1-byte CG_TYPE_INT column. */
	   CG_TYPE_NUMERIC = 2, CG_TYPE_BPCHAR1 = 3 };
#define CG_TYPE_NUMERIC_SCALE(s) (CG_TYPE_NUMERIC | ((s) << 8))

/* the slice of the TupleDesc the path needs (Form_pg_attribute attlen / attalign / type class) */
typedef struct CgColumnDesc
{
	int32_t attlen;     /* 1, 2, 4, 8: fixed-width by-value types; -1: varlena (CG_TYPE_NUMERIC / CG_TYPE_BPCHAR1 only) */
	int32_t type_class; /* CG_TYPE_* (low byte) | numeric scale << 8 */
} CgColumnDesc;

/* A columnar relation as the reader sees it: the main fork's 8 KB pages (as they sit in
 * shared_buffers / the file: 24-byte page header + 8168-byte payload, metapage in block 0,
 * data from block 2 -- backend/columnar/columnar_storage.c:21-31,117-126) + its visible
 * stripes and their skip lists (backend/columnar/columnar_metadata.c:717 ReadStripeSkipList). */
typedef struct CgRelation
{
	const uint8_t *pages;
	uint64_t nblocks;
	const CgStripe *stripes;
	int32_t nstripes;
	const CgSkipNode *nodes;
	int32_t nnodes;
	const CgColumnDesc *columns;
	int32_t natts;
} CgRelation;

/* ---------------------------------------------------------------------------------- *
 *  Query description: what the worker task's  Agg <- ColumnarScan  subtree computes
 *  (SURVEY.md 3.3).  Replaces ColumnarBeginRead(projectedColumnList, qualConditions)
 *  include/columnar/columnar.h:251-258 + the plan quals applied by ExecScan
 *  backend/columnar/columnar_customscan.c:1907-1913 + the worker half of the aggregate
 *  split planner/multi_logical_optimizer.c:3160-3484.
 * ---------------------------------------------------------------------------------- */
enum { CG_OP_LT = 0, CG_OP_LE = 1, CG_OP_EQ = 2, CG_OP_GE = 3, CG_OP_GT = 4, CG_OP_NE = 5,
	   CG_OP_IN = 6, CG_OP_NOT_IN = 7, CG_OP_IS_NULL = 8, CG_OP_IS_NOT_NULL = 9,
	   CG_OP_COL_LT = 16, CG_OP_COL_LE = 17, CG_OP_COL_EQ = 18, CG_OP_COL_GE = 19, CG_OP_COL_GT = 20, CG_OP_COL_NE = 21 };
/* 10 .. 15 are not operators: a descriptor that uses one is CG_EINVAL, as it was before the column atoms existed */

/* one atom of a predicate tree: "column <op> constant" (btree operators), a list membership test or a NULL test.
 * CG_OP_IN / CG_OP_NOT_IN ([PG] ScalarArrayOpExpr "x = ANY(array)" / "x <> ALL(array)", which is how IN and NOT IN lists
 * are planned): konst is the index of a list in CgScanDesc.in_lists.  CG_OP_IS_NULL / CG_OP_IS_NOT_NULL ([PG] NullTest):
 * konst must be 0.  Any atom may use them, in the WHERE quals and in the filter_quals pool alike.  With x the row's value,
 * S the list's non-NULL elements and nnulls its NULL elements (three-valued, as ExecEvalScalarArrayOp / ExecEvalNullTest):
 *                       x is NULL   x in S   x not in S, nnulls > 0   x not in S, nnulls = 0
 *     x IN (...)        UNKNOWN     TRUE     UNKNOWN                  FALSE
 *     x NOT IN (...)    UNKNOWN     FALSE    UNKNOWN                  TRUE
 *     x IS NULL         TRUE        FALSE    FALSE                    FALSE
 *     x IS NOT NULL     FALSE       TRUE     TRUE                     TRUE
 * so an IS test is never UNKNOWN.  Membership is equality in the column's btree order: a float column compares as float8
 * (every NaN equals every NaN, -0.0 equals +0.0); an integer-like column compares the decoded value, as konst does
 * (int1 / 2 / 4 / 8, date, timestamp, bool 0 / 1, char(1) as an unsigned byte, numeric(p, s) as value * 10^s).
 * Chunk-group skipping follows the reference ([PG] predicate_refuted_by with weak = false over the pushed-down clauses):
 * an IS test is never pushed down and refutes nothing; NOT IN refutes nothing (as <> does); IN refutes a chunk's
 * [min, max] iff its list has at most 100 elements (nvalues + nnulls, duplicates included), no NULL element, and every
 * element lies outside [min, max].
 * CG_OP_COL_LT .. CG_OP_COL_NE ([PG] OpExpr "x <op> y" over two Vars of the scanned relation): "column <op> other", with
 * konst the 0-based attribute index of the other column (it may be the column itself).  Any atom may use them, as above.
 * With y the other column's value of the same row:
 *                       x or y is NULL   otherwise
 *     x <op> y          UNKNOWN          TRUE or FALSE
 * The two columns must be of one comparison class, else the descriptor is CG_EUNSUPPORTED:
 *     integer-like   int1 / 2 / 4 / 8, bool, numeric(p, s) in any pairing: exact on the mathematical values.  The side of
 *                    the smaller scale is multiplied by 10^(scale difference) (an integer column has scale 0), in 128 bits,
 *                    so int8 < numeric(12, 2) compares x * 100 with y as [PG]'s cast to numeric does
 *     char(1)        against char(1) only: the unsigned byte
 *     float          float4 / float8 in any pairing: float4 widened to float8 (exact), float8 btree order (every NaN
 *                    equals every NaN and is above +inf, -0.0 equals +0.0)
 * An integer-like column against a float column is CG_EUNSUPPORTED ([PG] casts it to float8, which rounds int8).  A
 * column atom is never pushed down ([PG] ExtractPushdownClause wants a constant side): it refutes no chunk group and adds
 * no bound. */
typedef struct CgQual
{
	int32_t column;   /* 0-based attribute index */
	int32_t op;       /* CG_OP_* */
	int64_t konst;    /* integer, or float8 bits for float columns; IN / NOT IN: list index; IS [NOT] NULL: 0;
					   * CG_OP_COL_*: the other column's attribute index */
} CgQual;

#define CG_MAX_IN_LISTS 8
#define CG_MAX_IN_VALUES 1024          /* the elements of all lists of a query together */
#define CG_IN_REFUTE_MAX 100           /* [PG] MAX_SAOP_ARRAY_SIZE: a longer list refutes no chunk group */
/* one IN / NOT IN list: the array's elements as written (any order, duplicates allowed); the library sorts, removes
 * duplicates and canonicalises them.  A list has at least one element (nvalues + nnulls > 0). */
typedef struct CgInList
{
	int32_t first;     /* its non-NULL elements are in_values[first .. first + nvalues) */
	int32_t nvalues;
	int32_t nnulls;    /* its NULL elements */
	int32_t reserved;
} CgInList;

enum { CG_AGG_COUNT_STAR = 0, CG_AGG_COUNT = 1, CG_AGG_SUM = 2, CG_AGG_MIN = 3, CG_AGG_MAX = 4,
	   CG_AGG_BIT_AND = 5, CG_AGG_BIT_OR = 6, CG_AGG_BOOL_AND = 7, CG_AGG_BOOL_OR = 8, CG_AGG_VARIANCE = 9 };

/* aggregate argument = product over factors of (a + b * column); covers sum(x),
 * sum(x*y), sum(x*(1-d)), sum(x*(1-d)*(1+t)) on scaled-integer decimals (TPC-H Q1/Q6).
 * bit_and / bit_or (CG_AGG_BIT_*): the argument is one bare integer column (nfactors 1, a 0, b 1, is_float 0); the
 * result is in the column's type, the words hold it sign-extended to 64 bits.  bool_and / bool_or / every
 * (CG_AGG_BOOL_*): nfactors 0, the argument is the predicate tree arg_expr[a] of CgScanDesc.  None of the four takes
 * a term_abs_bound.
 * CG_AGG_VARIANCE: the state of var_pop / var_samp / variance / stddev_pop / stddev_samp / stddev over an integer
 * argument (the term sum takes: int1/2/4/8, numeric(p, s) as value * 10^s), which PostgreSQL keeps as the exact integers
 * N, sum(x) and sum(x^2).  The argument follows sum's rules: the same int64 overflow check, the same optional
 * term_abs_bound (a row over it fails the scan with CG_EINVAL; cg_relation_bounds fills it), FILTER, WHERE and every key
 * form.  A float argument is CG_EUNSUPPORTED (float8_accum's result cannot be matched bit for bit in any order).  All
 * six SQL names share this state: the name only picks the final function, cg_numeric_var_out, on the host.
 * cg_partial_fetch_ex returns N in count, sum(x) in sum_hi:sum_lo and sum(x^2) in sumsq. */
typedef struct CgAggSpec
{
	int32_t kind;        /* CG_AGG_* */
	int32_t nfactors;    /* 0 (count(*)) .. 3 */
	int32_t column[3];
	int32_t is_float;    /* float8 arithmetic (sum is order dependent: tolerance, not bit-exact) */
	int64_t a[3];        /* integers, or float8 bits when is_float */
	int64_t b[3];
	int64_t term_abs_bound; /* integer SUM: caller-proven bound on |argument| (from the skip lists'
							 * min/max), 0 = unknown.  When bound * max_rows < 2^63 the sum is kept in
							 * one 64-bit word instead of two; a row that violates the bound fails the
							 * scan with CG_EINVAL (never a wrong answer).  Without a bound, an integer
							 * sum / min / max argument that leaves int64 (in b*x, a + b*x or a product)
							 * fails the scan with CG_EUNSUPPORTED, like PostgreSQL's "bigint out of range". */
} CgAggSpec;

#define CG_MAX_QUALS 8
#define CG_MAX_AGGS 8
#define CG_MAX_GROUP_COLS 4
/* WHERE as a boolean tree over the atoms quals[0..nquals): postfix tokens, >= 0 = atom index,
 * CG_QX_AND / CG_QX_OR combine the two entries on top of the stack (PostgreSQL's BoolExpr; NOT is
 * folded into the operators).  nqual_expr = 0 means the plain AND of all atoms. */
#define CG_MAX_QEXPR 16
#define CG_QX_AND (-1)
#define CG_QX_OR (-2)
#define CG_MAX_FILTER_QUALS 8

/* Conditional aggregate argument ([PG] CaseExpr inside Aggref.args): sum(CASE WHEN c1 THEN r1 WHEN c2 THEN r2 ELSE r3 END).
 * An arm is a WHEN tree and a result; nwhen = 0 marks the ELSE arm, which must be its aggregate's last arm.  The WHEN tree is
 * the postfix token list when[0..nwhen) over CgScanDesc.filter_quals, in the filter_expr language (every atom kind).
 * The result (form):
 *   CG_CASE_NULL      the NULL constant
 *   CG_CASE_CONST     the constant a[0]: an integer, or float8 bits when the aggregate is_float
 *   CG_CASE_PRODUCT   product over nfactors (1..3) affine factors (a[f] + b[f] * column[f]), exactly as CgAggSpec's argument;
 *                     NULL when a factor column is NULL in the row */
#define CG_MAX_CASE_ARMS 16            /* the arms of all aggregates of a query together */
enum { CG_CASE_NULL = 0, CG_CASE_CONST = 1, CG_CASE_PRODUCT = 2 };
typedef struct CgCaseArm
{
	int32_t nwhen;                     /* 0 = ELSE */
	int8_t when[CG_MAX_QEXPR];
	int32_t form;                      /* CG_CASE_* */
	int32_t nfactors;                  /* CG_CASE_PRODUCT: 1 .. 3 */
	int32_t column[3];
	int64_t a[3];                      /* CG_CASE_CONST: the constant in a[0] */
	int64_t b[3];
} CgCaseArm;

typedef struct CgScanDesc
{
	int32_t nquals;
	CgQual quals[CG_MAX_QUALS];
	int32_t enable_qual_pushdown;   /* columnar.enable_qual_pushdown (columnar_customscan.c:225-236) */
	int32_t ngroup_cols;            /* 0 = plain aggregate */
	int32_t group_cols[CG_MAX_GROUP_COLS];
	int32_t naggs;
	CgAggSpec aggs[CG_MAX_AGGS];
	int64_t expected_groups;        /* planner's group estimate; 0 = let the library size the table */
	/* [PG] ExecQual over AND/OR trees (columnar_customscan.c:1907-1913): a row passes iff the tree is TRUE
	 * under three-valued logic -- an atom on a NULL input is not TRUE.  Chunk-group skipping follows
	 * predicate_refuted_by for the base constraint of ONE column at a time (columnar_reader.c:1132-1187):
	 * an AND node is refuted when any arm is, an OR node when all arms are. */
	int32_t nqual_expr;
	int8_t qual_expr[CG_MAX_QEXPR];
	int32_t reserved;
	/* Aggregate FILTER (WHERE ...) clauses ([PG] Aggref.aggfilter; the worker aggregate keeps the filter,
	 * multi_logical_optimizer.c:3279-3280, 3479).  The atoms filter_quals[0..nfilter_quals) are a pool of their own:
	 * they never take part in WHERE or in chunk-group skipping (SelectedChunkMask sees the scan's quals only), and
	 * cg_relation_bounds ignores them.  Aggregate a's filter is the postfix tree filter_expr[a][0..nfilter_expr[a]) over
	 * that pool, in the qual_expr token language; nfilter_expr[a] = 0 = no filter, so a zero-filled tail is a query
	 * without filters.  A row that passes WHERE joins its group whatever the filters say; it is an input of aggregate
	 * a only when a's tree is TRUE under three-valued logic (an atom on a NULL column is not TRUE), and a rejected
	 * row's argument is not evaluated: it raises neither the int64 overflow nor the term_abs_bound error.  So a group
	 * without accepted rows has count(*) / count(x) = 0 and sum / min / max = NULL (count 0).  A column read only by a
	 * filter is staged and counts toward the query's column limit.
	 * The pool is shared with the predicate arguments of bool_and / bool_or below: at most CG_MAX_FILTER_QUALS atoms
	 * for all FILTERs and arguments of a query together, and an atom they have in common is stored once. */
	int32_t nfilter_quals;
	CgQual filter_quals[CG_MAX_FILTER_QUALS];
	int32_t nfilter_expr[CG_MAX_AGGS];
	int8_t filter_expr[CG_MAX_AGGS][CG_MAX_QEXPR];
	/* Predicate argument of bool_and / bool_or / every (CG_AGG_BOOL_*): aggregate a's argument p is the postfix tree
	 * arg_expr[a][0..narg_expr[a]) over the filter_quals pool, 1..CG_MAX_QEXPR tokens; narg_expr[a] = 0 for every other
	 * kind, so a zero-filled tail is a query without predicate arguments.  p is evaluated under three-valued logic: an
	 * atom on a NULL column is UNKNOWN (a float atom is never UNKNOWN otherwise: NaN compares in btree order), AND is
	 * FALSE if an arm is FALSE, OR is TRUE if an arm is TRUE.  A row whose p is UNKNOWN is no input (like a NULL
	 * argument), and so is a row the aggregate's FILTER rejects (its p is not consulted).  bool_and = every input is
	 * TRUE, bool_or = some input is TRUE; with no input the result is NULL.  cg_partial_fetch returns the value in
	 * minmax (0 / 1) and the number of inputs in count (0 = NULL); chunk-group skipping and cg_relation_bounds ignore
	 * the argument atoms, as they ignore the filter atoms. */
	int32_t narg_expr[CG_MAX_AGGS];
	int8_t arg_expr[CG_MAX_AGGS][CG_MAX_QEXPR];
	/* Composite GROUP BY key.  composite_key = 0: the key forms above -- one column, or two columns of at most 4 bytes
	 * packed into one int64 (low 32 bits: the first), where a NULL in either column fails the scan with CG_EUNSUPPORTED;
	 * ngroup_cols > 2 is CG_EINVAL.  composite_key = 1: ngroup_cols = K in 1..CG_MAX_GROUP_COLS columns of any integer-like
	 * type (int1 / int2 / int4 / int8, bool, char(1), numeric(p, s); float is CG_EUNSUPPORTED), NULLs included, with every
	 * row's key value of column c in [key_col_min[c], key_col_max[c]] (cg_relation_key_bounds; key_col_min > key_col_max
	 * = the column is NULL in every row).  The key is one exact int64 code, a mixed-radix number:
	 *     d_c = 0 if column c is NULL, else v_c - key_col_min[c] + 1;   R_c = key_col_max[c] - key_col_min[c] + 2 (1 if all NULL)
	 *     code = ((d_0 * R_1 + d_1) * R_2 + d_2) * R_3 + d_3,   in [0, D), D = R_0 * ... * R_{K-1}
	 * Codes sort the way the key tuples sort, NULL lowest in each column.  cg_partial_create refuses D > 2^63 with
	 * CG_EUNSUPPORTED and ignores its key_min / key_max; the partial is then a one-column partial over the code, with no
	 * NULL group: direct-indexed when D <= 2^26, else a hash table.  A row whose key value lies outside its column's
	 * bounds joins no group and fails the scan with CG_EINVAL, in every table kind.  cg_partial_fetch,
	 * cg_partial_export_device, cg_partial_merge_rows and cg_partial_merge_values carry codes in their key arrays;
	 * key_nulls is always 0 on export, and a row merged with a non-zero key_nulls entry is refused with CG_EINVAL
	 * (merge_values: at once; merge_rows: by the calls that read the partial).  cg_group_key_decode / cg_group_key_encode
	 * convert.  A scan's descriptor must have the
	 * partial's key columns and bounds (CG_EINVAL otherwise); a zero-filled tail is composite_key = 0. */
	int32_t composite_key;
	int64_t key_col_min[CG_MAX_GROUP_COLS];
	int64_t key_col_max[CG_MAX_GROUP_COLS];
	/* The lists of the CG_OP_IN / CG_OP_NOT_IN atoms (see CgQual), shared by the WHERE quals and the filter_quals pool:
	 * in_lists[0 .. nin_lists), their non-NULL elements in in_values[0 .. nin_values) in konst's convention (decoded integer,
	 * or float8 bits).  They are held in the descriptor, not behind a pointer, so that a copy of it is a whole query.  A
	 * zero-filled tail is a query without lists. */
	int32_t nin_lists;
	CgInList in_lists[CG_MAX_IN_LISTS];
	int32_t nin_values;
	int64_t in_values[CG_MAX_IN_VALUES];
	/* CASE arguments (CgCaseArm).  case_narms[a] > 0: aggregate a's argument is the searched CASE over the arms
	 * case_arms[case_first[a] .. case_first[a] + case_narms[a]); two aggregates may name the same range (avg's sum and count).
	 * case_narms[a] = 0 = no CASE, so a zero-filled tail is a query without CASE.  Per row that passes WHERE:
	 *   - a row aggregate a's FILTER rejects is no input, and its CASE is not consulted;
	 *   - otherwise the WHEN trees are evaluated in order under three-valued logic (UNKNOWN is not TRUE); the value is the
	 *     result of the first arm whose tree is TRUE, else the ELSE arm's, else NULL;
	 *   - only the chosen arm's result is evaluated: an int64 overflow or a term_abs_bound violation in an arm that was not
	 *     chosen raises nothing; in the chosen arm it fails the scan as it does for a plain argument (CG_EUNSUPPORTED /
	 *     CG_EINVAL);
	 *   - a NULL value is no input: it is counted in the aggregate's no-input word, as a NULL argument is.
	 * So sum(CASE WHEN c THEN x ELSE 0 END) gives 0 for a group whose rows all fail c, where sum(x) FILTER (WHERE c) gives
	 * NULL; count(CASE WHEN c THEN 1 END) counts the rows where c is TRUE.
	 * Kinds: CG_AGG_COUNT, CG_AGG_SUM, CG_AGG_MIN, CG_AGG_MAX and CG_AGG_VARIANCE, with nfactors = 0 (the arms carry the terms).
	 * A CASE aggregate has exactly the words of its kind (with the no-input word), so fetch, export, merge and combine are
	 * unchanged, and optimistic packing follows sum's rule.  An integer CASE has integer results at one scale the caller
	 * chose (a, b and the constants pre-scaled; the value comes back exact at that scale, but [PG]'s display scale of a
	 * numeric CASE whose arms differ in scale depends on which arms supplied inputs, which the words do not record); a float
	 * CASE has float8 results.  Columns an arm reads are plan columns (staged, counted toward the column limit) and the
	 * atoms of its WHEN tree share the filter_quals pool.  cg_relation_bounds gives a CASE sum the largest bound over its
	 * arms (a constant counts |k|, a NULL arm 0); WHEN atoms take no part in bounds or chunk-group skipping.
	 * A scan or join into a partial must carry the CASE arguments the partial was created with (the same arms in the same
 * order, wherever they sit in case_arms), else CG_EINVAL.
 * CG_EINVAL: a CASE on another kind, or with nfactors != 0; an arm range outside [0, ncase_arms) or ncase_arms >
	 * CG_MAX_CASE_ARMS; an ELSE arm that is not the last of its range; a malformed WHEN tree or a token outside the pool; a
	 * bad form, a product with nfactors outside 1 .. 3 or a column outside [0, natts).  Column types are checked as for a
	 * plain argument of the kind (integer / float mismatch CG_EINVAL; variance of a float CG_EUNSUPPORTED, of char(1)
	 * CG_EINVAL). */
	int32_t case_first[CG_MAX_AGGS];
	int32_t case_narms[CG_MAX_AGGS];
	int32_t ncase_arms;
	int32_t reserved2;
	CgCaseArm case_arms[CG_MAX_CASE_ARMS];
} CgScanDesc;

/* EXPLAIN ANALYZE counters (columnar_customscan.c:1966-1999 and ExecScan instrumentation) */
typedef struct CgScanStats
{
	int64_t rows_scanned;            /* rows handed to the qual */
	int64_t rows_removed_by_filter;  /* "Rows Removed by Filter" */
	int64_t chunk_groups_filtered;   /* "Columnar Chunk Groups Removed by Filter" */
	int64_t rows_passed;
	int64_t chunk_groups_scanned;
	int64_t bytes_scanned;           /* algorithmic bytes: sum over projected columns of
									  * value bytes + exists bytes of the scanned chunk groups */
	double kernel_ms;                /* device time of the fused kernel(s), CUDA events */
	int64_t h2d_bytes;               /* cg_scan_relation: bytes copied host -> device */
} CgScanStats;

/* ---------------------------------------------------------------------------------- *
 *  Staged shards: the projected column chunks of a relation resident in HBM.
 *  Replaces LoadFilteredStripeBuffers / LoadColumnBuffers / ColumnarStorageRead
 *  (backend/columnar/columnar_reader.c:1007-1124, columnar_storage.c:463-492): each
 *  (column, chunk) exists/value buffer is copied out of the 8 KB pages into pinned
 *  memory at a 16-byte aligned slot and sent with cudaMemcpyAsync on a side stream.
 * ---------------------------------------------------------------------------------- */
typedef struct CgShard CgShard;

/* columns: attribute indexes to stage (NULL/0 = all).  The call returns when the shard
 * is resident.  Compressed value streams (lz4, pglz, zstd) are decoded on the GPU behind the copies. */
int cg_shard_stage(const CgRelation *rel, const int32_t *columns, int32_t ncolumns, CgShard **out);
void cg_shard_free(CgShard *shard);
uint64_t cg_shard_device_bytes(const CgShard *shard);   /* the arena and the narrow images */
uint64_t cg_shard_rows(const CgShard *shard);

/* Narrow images.  Besides the plain arena, cg_shard_stage keeps every staged 8-byte integer column whose NULL-free chunk
 * columns each span at most 2^32 values (max - min < 2^32) in a second, bit-packed form: per chunk column base = min and
 * width = bits(max - min), 0 .. 32, and row r at bits [r * width, r * width + width) of a bit stream.  The ahead-of-time
 * fast kernel reads those images when every column of its plan has them; everything else reads the arena.  The images
 * are best effort: when their memory cannot be had (with a fixed headroom left free) the shard is staged without them.
 * cg_shard_narrow_bytes = bytes of the images (0: none); cg_shard_narrow_column = 1 when attribute att has them. */
uint64_t cg_shard_narrow_bytes(const CgShard *shard);
int32_t cg_shard_narrow_column(const CgShard *shard, int32_t att);
/* One chunk column's image, read back: *base, *width and its bit stream (ceil(rows / 64) * width words, *nbytes bytes) into
 * host_buf, which must hold them; host_buf = NULL only reports them.  *width = 255 and *nbytes = 0 when the chunk column has
 * no image.  CG_EINVAL: chunk group or attribute out of range, the attribute is not staged, or capacity is too small. */
int cg_shard_narrow_image(const CgShard *shard, int64_t cg, int32_t att, int64_t *base, uint32_t *width, void *host_buf,
						  uint64_t capacity, uint64_t *nbytes);

/* The layout cg_shard_stage gives the narrow images of ncg chunk groups x ncols staged columns, arrays [ncg][ncols]:
 * candidate[c] = column c may have images (8-byte integer); rows[g] = rows of chunk group g; nullfree[g][c] = the chunk
 * column has no NULLs; mins / maxs = its exact minimum / maximum (read only where nullfree).  A candidate column gets
 * images (col_narrow[c] = 1) when every NULL-free chunk column of it spans max - min < 2^32.  Out, per chunk column:
 * widths (255 = no image), bases, byte offsets of the 16-byte aligned bit streams (ceil(rows / 64) * width words each);
 * *total_bytes = bytes of all streams. */
int cg_narrow_plan(int64_t ncg, int32_t ncols, const uint8_t *candidate, const uint32_t *rows, const uint8_t *nullfree,
				   const int64_t *mins, const int64_t *maxs, uint8_t *col_narrow, uint8_t *widths, int64_t *bases, uint64_t *offs,
				   uint64_t *total_bytes);

/* ---------------------------------------------------------------------------------- *
 *  Partial aggregate state: the device-resident group table a worker task accumulates
 *  (PostgreSQL nodeAgg's hash table + transition values, and on the coordinator the
 *  combine HashAggregate over sum(sum)/sum(count), multi_logical_optimizer.c:1807-1885,
 *  2231-2275).  One CgPartial may accumulate several shards of the same GPU (legal for
 *  the commutative/associative built-ins) or exactly one (a per-task result).
 * ---------------------------------------------------------------------------------- */
typedef struct CgPartial CgPartial;

/* key_min/key_max: exact bounds of the (packed) group key over the data to be scanned,
 * taken from the skip lists; when the domain is small the table is direct-indexed.
 * Pass key_min > key_max to force the general hash table. */
int cg_partial_create(const CgScanDesc *desc, const CgColumnDesc *columns, int32_t natts,
					  int64_t key_min, int64_t key_max, int64_t max_rows, CgPartial **out);
void cg_partial_free(CgPartial *p);
int cg_partial_reset(CgPartial *p);
/* Optimistic packing (on by default when the plan allows it): for a direct-indexed GROUP BY
 * with count(*) and a bounded integer sum, a row updates ONE 64-bit word
 * (sum << C | count) with one L2 reduction instead of two; packed words are drained into
 * the exact wide accumulators between launches.  A group that receives 2^C or more rows
 * between two drains would overflow its count field: this is detected exactly (the drained
 * counts must add up to the rows added) and reported as CG_ERETRY_UNPACKED by the calls that
 * read the partial -- never as a wrong result. */
int cg_partial_set_packing(CgPartial *p, int32_t enable);

/* Fused decode + filter + partial aggregate of one staged shard into `into`.
 * Chunk-group skipping (SelectedChunkMask, columnar_reader.c:1132-1187) runs on the host
 * from the skip nodes; surviving chunk groups are scanned by one kernel launch.
 * stats may be NULL. The call is asynchronous with respect to the host unless stats is
 * given (counters need the kernel to finish). */
int cg_scan_shard(const CgShard *shard, const CgScanDesc *desc, CgPartial *into, CgScanStats *stats);

/* Row-emitting scan of one staged shard:
 *     SELECT atts[0 .. ncols) FROM shard WHERE <desc's WHERE tree>        in the shard's row order
 * the filter query of a repartition join's map task (worker_partition_query_result,
 * executor/partitioned_intermediate_results.c:115-298), with the rows left in device columns.
 *   WHERE.  desc supplies the WHERE part only: quals, qual_expr, IN lists, IS [NOT] NULL atoms, column atoms and
 *   enable_qual_pushdown, with the rules of cg_scan_shard (a row passes only when the tree is TRUE under three-valued
 *   logic; chunk-group skipping is SelectedChunkMask over the skip nodes).  A desc with aggregates, group columns, FILTER
 *   or predicate-argument trees, CASE arms or a composite key is CG_EINVAL.  The WHERE columns count toward the kernels'
 *   column limit (8) as for a scan (CG_EUNSUPPORTED over it).
 *   Order.  Stripes in order, chunk groups in order, rows in order: the order in which ColumnarScan hands rows to
 *   PartitionedResultDestReceiver, so cg_partition_copy_serialize over these rows writes the reference's files.
 *   Columns.  1 .. 16 output columns (the COPY serializer's limit); an attribute may appear more than once; one that is
 *   out of range or not staged in the shard is CG_EINVAL.  d_cols[c] receives the values of atts[c] in CgJoinSide's form:
 *   integers sign-extended to int64, bool 0 / 1, char(1) as the unsigned byte, numeric(p, s) as value * 10^s, float4 /
 *   float8 as float8 bits; a NULL's value slot holds 0.
 *   NULLs.  d_nulls may be NULL, and so may any d_nulls[c]; a given null array receives one byte per output row, 1 for
 *   NULL and 0 otherwise.  With capacity > 0, d_nulls[c] is required when atts[c] has NULLs in a chunk group that
 *   survives skipping (value_count != row_count in its skip node): a missing one is CG_EINVAL before anything is
 *   launched.
 *   Capacity.  *nrows = the number of passing rows.  capacity = 0 writes nothing (size the arrays, call again); a capacity
 *   below *nrows is CG_EINVAL with *nrows set and no output byte written.  d_cols and every d_cols[c] must be device
 *   pointers when capacity > 0.
 *   Synchronisation.  The call waits once for the host to read the total; the writes are enqueued on the library's
 *   compute stream (cg_set_stream), so the next library call on it -- routing, the exchange, a join -- sees them.  With
 *   stats the call also waits for the writes.  The row scan ends a chain of scan launches like any other enqueue, and
 *   leaves the shard's chunk-group selection for cg_scan_shard as it was.
 *   Stats (may be NULL): rows_scanned (rows of the surviving chunk groups), rows_removed_by_filter, rows_passed,
 *   chunk_groups_filtered, chunk_groups_scanned, bytes_scanned = the algorithmic bytes of the WHERE columns plus those of
 *   the distinct projected columns over the surviving chunk groups, kernel_ms = device time of the row kernels.
 *   A shard without rows, or one whose chunk groups are all skipped, gives *nrows = 0 and CG_OK.
 * Not covered: host pages (cg_scan_relation's transient form; stage first), narrow images, expressions in the
 * projection. */
int cg_scan_shard_rows(const CgShard *shard, const CgScanDesc *desc, const int32_t *atts, int32_t ncols, int64_t capacity,
					   int64_t *const *d_cols, uint8_t *const *d_nulls, int64_t *nrows, CgScanStats *stats);

/* End-to-end call on HOST buffers: stage + scan.  This is what a GpuColumnarAgg CustomScan
 * node calls once per shard task.  Pageable pages (shared_buffers as it is today) are
 * de-framed by host threads into pinned blocks and sent with cudaMemcpyAsync; pages in
 * pinned memory (cg_relation_register, or a shared_buffers segment registered once at
 * startup) are sent by the copy engine itself as runs of whole pages (1-D copies);
 * the GPU drops the page headers and re-aligns the chunk buffers. */
int cg_relation_register(const CgRelation *rel);      /* cudaHostRegister of the page image */
int cg_relation_unregister(const CgRelation *rel);
int cg_scan_relation(const CgRelation *rel, const CgScanDesc *desc, CgPartial *into, CgScanStats *stats);

/* Result rows.  Group order is unspecified (it is a hash aggregate).
 * For aggregate j of group i (index i*naggs + j):
 *   sum_hi/sum_lo  128-bit integer sum (two's complement), or float8 sum in fsum
 *   count          count(*) / count(x) value, or for sum/min/max the number of non-NULL
 *                  inputs (0 => the SQL result is NULL)
 *   minmax         min or max (integer, or float8 bits); bit_and / bit_or (sign-extended); bool_and / bool_or (0 / 1)
 *   count          of bit_* / bool_*: the number of inputs (0 => NULL)
 * Any output pointer may be NULL. */
int cg_partial_ngroups(CgPartial *p, int64_t *ngroups);
int cg_partial_fetch(CgPartial *p, int64_t capacity, int64_t *keys, uint8_t *key_nulls,
					 int64_t *sum_hi, uint64_t *sum_lo, int64_t *count, int64_t *minmax,
					 double *fsum, int64_t *ngroups);
/* cg_partial_fetch plus sumsq [capacity * naggs * 3]: for a CG_AGG_VARIANCE aggregate, sum(x^2) of the group as an
 * unsigned 192-bit little-endian integer in the argument's scaled units (x^2 <= 2^126, at most 2^32 rows per group), in
 * the same group order as the other arrays (0 for the other kinds).  One call, because the order of the groups is not
 * the same from one call to the next.  cg_partial_fetch is this call with sumsq = NULL.  A group of 2^32 rows or more
 * in a partial with a limb-word sum is CG_EUNSUPPORTED. */
int cg_partial_fetch_ex(CgPartial *p, int64_t capacity, int64_t *keys, uint8_t *key_nulls,
						int64_t *sum_hi, uint64_t *sum_lo, int64_t *count, int64_t *minmax,
						double *fsum, uint64_t *sumsq, int64_t *ngroups);

/* The inverse of cg_partial_fetch: partial-aggregate ROWS held on the host (group key + per aggregate the 128-bit
 * sum, count, min / max, float sum; arrays [nrows * naggs] laid out like cg_partial_fetch's) are folded into p by the
 * combine kernel.  What the coordinator does with the per-shard result rows it receives (adaptive_executor.c:3964-4189
 * ReceiveResults -> TupleDestination) in place of a CPU HashAggregate over them.  Arrays an aggregate list does not
 * need may be NULL.  count[] of a sum / min / max is its number of non-NULL inputs (0 = the partial was SQL NULL).
 * A partial with a CG_AGG_VARIANCE aggregate is CG_EUNSUPPORTED: the rows carry no sum(x^2) (merge the words with
 * cg_partial_merge_rows instead). */
int cg_partial_merge_values(CgPartial *p, int64_t nrows, const int64_t *keys, const uint8_t *key_nulls, const int64_t *sum_hi,
							const uint64_t *sum_lo, const int64_t *count, const int64_t *minmax, const double *fsum);
/* count / exact sum / min / max of one host column (attlen 1, 2, 4, 8; float4 is widened to float8 for min / max; a float
 * sum is not computed: its result depends on the order) in one pass: the batch step of the worker_partial_agg /
 * coord_combine_agg shims (utils/aggregate_utils.c:501-607, 820-1003), which otherwise pay one fmgr call per row. */
int cg_agg_column(int32_t attlen, int32_t is_float, const void *values, const uint8_t *isnull, int64_t n, int64_t *count,
				  int64_t *sum_hi, uint64_t *sum_lo, int64_t *min_value, int64_t *max_value);

/* Raw accumulator export / merge, for the combine step and for collectives.
 * A partial is `nwords` 64-bit accumulator words per group; every word is combined
 * with one commutative op (add / min / max / float add), so partials of different
 * shards or GPUs are merged word by word -- by this library (cg_partial_merge_rows)
 * or by ncclReduce on the dense layout. */
/* at most CG_MAX_WORDS words per group: word 0 (rows) and per aggregate count(*) 0 (1 with a FILTER), count(x) 1,
 * sum 2 or 3, min / max / bit_* / bool_* 2, variance 3 to 7 (7 without a term_abs_bound); cg_partial_create refuses a
 * longer aggregate list with CG_EUNSUPPORTED */
#define CG_MAX_WORDS 32
int cg_partial_layout(const CgPartial *p, int32_t *nwords, int32_t *word_ops /* [nwords] CG_WORD_* */,
					  int32_t *is_dense, int64_t *capacity);
/* CG_WORD_AND / CG_WORD_OR: bitwise, identities ~0 and 0 (bit_and / bit_or values; bool_and / bool_or keep the truth
 * value in bit 0, an input TRUE contributes ~0 and FALSE 0) */
enum { CG_WORD_ADD = 0, CG_WORD_MIN = 1, CG_WORD_MAX = 2, CG_WORD_FADD = 3, CG_WORD_FMIN = 4, CG_WORD_FMAX = 5,
	   CG_WORD_AND = 6, CG_WORD_OR = 7 };

/* Compact occupied groups into device arrays owned by the caller (e.g. torch tensors):
 * d_keys[capacity], d_key_nulls[capacity] (may be NULL), d_words[capacity*nwords];
 * *nrows on the host. */
int cg_partial_export_device(CgPartial *p, int64_t capacity, int64_t *d_keys, uint8_t *d_key_nulls,
							 uint64_t *d_words, int64_t *nrows);
/* Merge rows (device arrays) into p: the coordinator-side combine kernel (K5). */
int cg_partial_merge_rows(CgPartial *p, const int64_t *d_keys, const uint8_t *d_key_nulls,
						  const uint64_t *d_words, int64_t nrows);
/* Plain-aggregate and direct-indexed tables only: device pointer and length (in 64-bit
 * words) of the whole accumulator array, laid out [entry][stride].  Two partials created
 * with the same arguments have identical layouts, so when every word op is CG_WORD_ADD a
 * collective (ncclReduce / ncclAllReduce, sum, int64) combines them in place. */
int cg_partial_dense_words(CgPartial *p, uint64_t **d_words, int64_t *total_words, int32_t *stride);
/* The same without a host synchronisation: pending table maintenance is only enqueued on the library's
 * stream (cg_set_stream), so a collective enqueued behind it on that stream reduces the finished table
 * and the host runs ahead.  The scan's error flags are not examined: call cg_partial_check (every rank,
 * after enqueuing the collective) before trusting the combined result. */
int cg_partial_dense_words_enqueue(CgPartial *p, uint64_t **d_words, int64_t *total_words, int32_t *stride);
/* Waits for the partial's pending work and reports what its kernels flagged. */
int cg_partial_check(CgPartial *p);
/* Read-only view of the optimistic packing (cg_partial_set_packing): C (0 = the partial has no packed words), the
 * accumulator word the packed sum drains into, the CG_PSTATE_* bits, and the packed words themselves -- one per table
 * entry, ((sum << C) + rows) mod 2^64 -- copied into h_words (NULL or capacity 0: *nwords only).  Waits for the work
 * already enqueued on the library's stream and enqueues none: the partial, its words and flags, and whether the next scan
 * may overlap the previous one are all left as they were. */
#define CG_PSTATE_PACKED_DIRTY 1u       /* packed words were added since the last drain or reset */
#define CG_PSTATE_WIDE_DIRTY 2u         /* the wide accumulator words were written since the last reset */
#define CG_PSTATE_READ_PACKED_DIRECT 4u /* a read decoded result rows straight from the packed words since the last drain */
#define CG_PSTATE_TABLE_INITIALISED 8u  /* the wide table was initialised at least once */
int cg_partial_packed_state(CgPartial *p, uint64_t *h_words, uint64_t capacity, int32_t *pack_shift, int32_t *pack_word,
							uint32_t *state, uint64_t *nwords);

/* ---------------------------------------------------------------------------------- *
 *  Hash repartition (map side): worker_partition_query_result's per-row routing
 *  executor/partitioned_intermediate_results.c:493-553 + FindShardInterval
 *  utils/shardinterval_utils.c:260-452.  Keys and payload are device arrays.
 * ---------------------------------------------------------------------------------- */
/* partition index of every row: NULL key -> 0, else binary search of hashint4/8(key) (or of
 * the raw value for range partitioning) over [mins[i], maxs[i]].  key_len 4 or 8.
 * d_index[n] (int32), d_counts[P] (int64).  Returns CG_EINVAL if a hash falls in no range. */
int cg_partition_index(const int64_t *d_keys, const uint8_t *d_nulls, int64_t n, int32_t key_len,
					   int32_t by_hash, const int32_t *mins, const int32_t *maxs, int32_t P,
					   int32_t *d_index, int64_t *d_counts);
/* Stable scatter of `ncols` int64 payload columns into partition-contiguous order:
 * d_out[c][offsets[p] .. offsets[p+1]) holds partition p's rows in input order. */
int cg_partition_scatter(const int32_t *d_index, int64_t n, int32_t P, const int64_t *const *d_cols,
						 int32_t ncols, int64_t *const *d_out, int64_t *h_offsets /* [P+1] */);
/* Same, with the partitions laid out in a caller-chosen order: h_order[p] = output position of
 * partition p (a permutation; e.g. destination-rank-major for an all-to-all);
 * h_offsets[i] .. h_offsets[i+1] then delimit the partition whose position is i. */
int cg_partition_scatter_ordered(const int32_t *d_index, int64_t n, int32_t P, const int32_t *h_order,
								 const int64_t *const *d_cols, int32_t ncols, int64_t *const *d_out,
								 int64_t *h_offsets /* [P+1] */);

/* The return rows of worker_partition_query_result (partitioned_intermediate_results.c:270-291):
 * rows_written[P] and bytes_written[P] (host arrays), the bytes being what each partition's file
 * would hold in COPY text or binary format (worker/worker_sql_task_protocol.c:91-251).  d_cols:
 * ncols device arrays of int64 values; d_nulls: per column a device byte array or NULL; col_len:
 * the binary width of every column (4 for int4, 8 for int8).  A partition without rows has 0
 * bytes unless generate_empty_results (then a binary file still holds header + trailer). */
int cg_partition_copy_bytes(const int32_t *d_index, int64_t n, int32_t P, const int64_t *const *d_cols,
							const uint8_t *const *d_nulls, const int32_t *col_len, int32_t ncols, int32_t binary,
							int32_t generate_empty_results, int64_t *rows_written, int64_t *bytes_written);

/* The partition files themselves (what TaskFileDestReceiver writes, worker/worker_sql_task_protocol.c:91-251): the COPY text or
 * binary encoding of every row, rows of a partition in input order, the P files back to back in the device buffer d_out
 * (out_capacity bytes); file p is [file_offsets[p], file_offsets[p + 1]).  Sizes equal cg_partition_copy_bytes'. */
int cg_partition_copy_serialize(const int32_t *d_index, int64_t n, int32_t P, const int64_t *const *d_cols,
								const uint8_t *const *d_nulls, const int32_t *col_len, int32_t ncols, int32_t binary,
								int32_t generate_empty_results, uint8_t *d_out, int64_t out_capacity, int64_t *file_offsets /* [P + 1] */);

/* The merge side of a dual-repartition join for the aggregate query
 *     SELECT count(*), sum(b.payload + p.payload) FROM build b JOIN probe p USING (key)
 * over two co-located partitions that are already device arrays (what the MERGE task computes with
 * read_intermediate_results() + PostgreSQL's HashJoin + Agg, planner/multi_physical_planner.c:
 * 4304-4328, executor/intermediate_results.c:789-1045).  NULL keys join nothing; the sum is exact
 * (128-bit two's complement in sum_hi:sum_lo).  The joined rows are never materialised. */
int cg_join_count_sum(const int64_t *d_build_keys, const uint8_t *d_build_nulls, const int64_t *d_build_payload,
					  int64_t nbuild, const int64_t *d_probe_keys, const uint8_t *d_probe_nulls,
					  const int64_t *d_probe_payload, int64_t nprobe, int64_t *joined_rows, int64_t *sum_hi,
					  uint64_t *sum_lo);

/* ---------------------------------------------------------------------------------- *
 *  Exchange steps across GPUs (one process per GPU on one node; NVLink / NVSwitch, on the library's streams).
 *  Data moves through a peer window -- every rank's buffers mapped into every other rank with CUDA IPC, written
 *  and read by the library's own kernels -- with NCCL underneath for bootstrap, counts and agreements, and as the
 *  data path when the mapping is refused or switched off (cg_set_option("peer_window", 0) on every rank).
 *  Replaces the libpq funnel of the adaptive executor for GPU-resident results
 *  (executor/adaptive_executor.c:3964-4189 ReceiveResults + the combine query's HashAggregate,
 *  planner/multi_logical_optimizer.c:1807-1885, 2231-2275) and the file exchange of a repartition
 *  (executor/partitioned_intermediate_results.c:115-298, executor/intermediate_results.c:789-1045).
 * ---------------------------------------------------------------------------------- */
#define CG_COMM_ID_BYTES 128
/* rank 0 creates the id; the caller ships the bytes to every rank (over the coordinator's connections) */
int cg_comm_unique_id(uint8_t *id /* [CG_COMM_ID_BYTES] */);
int cg_comm_init(const uint8_t *id, int32_t rank, int32_t nranks);    /* collective; after cg_init; id may be NULL when nranks = 1 */
int cg_comm_rank(int32_t *rank, int32_t *nranks);
int cg_comm_destroy(void);
int cg_comm_barrier(void);
int cg_comm_peer_window(void);               /* 1: the peer window carries the combine and the exchange; 0: NCCL does */
enum { CG_COMM_SUM = 0, CG_COMM_MIN = 1, CG_COMM_MAX = 2 };
/* small host-side agreement (plan constants such as the key range; timings): values[i] <- op over ranks */
int cg_comm_allreduce_i64(int64_t *values, int32_t n, int32_t op);
/* Coordinator-side combine: after the call the partial of rank `root` holds the combined aggregate.  Collective:
 * EVERY rank calls it, passing the status of its own scans in local_status -- a rank that failed still takes
 * part, and every rank then returns an error instead of some of them hanging in a collective.  Direct-indexed
 * tables with additive words are reduced in place (the packed words alone when nothing else was written -- then by
 * the ranks themselves: rank s sums slice s of every rank's words over NVLink into the root's window);
 * other tables send their compacted rows to the root, which merges them.  Asynchronous on the library's
 * stream: errors raised by kernels of any rank surface on the root at the next call that reads the partial. */
int cg_comm_combine(CgPartial *p, int32_t root, int32_t local_status);
/* Hash repartition of this rank's rows (column 0 = the key) into P partitions, partition p owned by rank
 * p mod nranks.  Peer window: routing + histogram, the counts of all ranks, then ONE kernel that is scatter and
 * all-to-all at once -- rows leave shared memory as runs straight into the owner's receive buffer.  NCCL path:
 * scatter into destination-major order and one grouped ncclSend/ncclRecv of all columns on a second stream, so
 * that the next table's routing and scatter overlap this table's exchange.  Results live in the slot (0..3)
 * until its next use.  A NULL key (d_key_nulls[i] != 0) routes its row to partition 0, but the received table carries
 * only the value columns, so the receiver cannot tell that row's key slot from a real key: a join over the received
 * rows would match it on whatever value the slot holds. */
int cg_comm_repartition_exchange(int32_t slot, const int64_t *const *d_cols, const uint8_t *d_key_nulls, int64_t n,
								 int32_t ncols, int32_t key_len, int32_t P, const int32_t *mins, const int32_t *maxs,
								 int64_t *recv_rows);
int cg_comm_exchange_wait(int32_t slot);      /* the library's compute stream waits (on the device) for the slot's exchange */
/* received columns (device pointers), rows, rows of every local partition by source rank [nlocal][nranks],
 * bytes sent to other ranks and the duration of the exchange on its stream; any pointer may be NULL */
int cg_comm_exchange_result(int32_t slot, int64_t **d_cols, int64_t *nrows, int64_t *part_counts, int32_t *nlocal,
							uint64_t *sent_bytes, double *exchange_ms);
/* the host-side plan of an exchange (exposed for tests): position[p] = place of partition p in destination-major
 * order; from counts[nranks][P] the rows this rank sends to / receives from every rank and the rows of its local
 * partitions by source rank.  counts may be NULL (positions and nlocal only). */
int cg_comm_exchange_plan(int32_t P, int32_t nranks, int32_t rank, const int64_t *counts, int32_t *position,
						  int64_t *send_rows, int64_t *recv_rows, int64_t *local_part_counts, int32_t *nlocal);
/* peer-window form: where this rank's rows land in the receive buffers of the ranks (pure host arithmetic over the
 * exchanged counts, counts[r * P + p]).  Positions [pos_begin[d], pos_begin[d + 1]) belong to rank d; rank d's buffer
 * has a column stride of total[d] rows; a row at index i of this rank's send order lands at adj[d] + i. */
int cg_comm_peer_plan(int32_t P, int32_t nranks, int32_t rank, const int64_t *counts, int32_t *pos_begin /* [nranks + 1] */,
					  int64_t *total /* [nranks] */, int64_t *adj /* [nranks] */);

/* The same join emitting its rows -- SELECT b.key, b.payload, p.payload FROM build b JOIN probe p USING (key) -- into device
 * arrays of `capacity` rows owned by the caller (row order unspecified, NULL keys join nothing).  *nrows = the number of
 * joined rows; with capacity 0 nothing is written (size the arrays, call again); a too small capacity is CG_EINVAL. */
int cg_join_rows(const int64_t *d_build_keys, const uint8_t *d_build_nulls, const int64_t *d_build_payload, int64_t nbuild,
				 const int64_t *d_probe_keys, const uint8_t *d_probe_nulls, const int64_t *d_probe_payload, int64_t nprobe,
				 int64_t capacity, int64_t *d_out_key, int64_t *d_out_build_payload, int64_t *d_out_probe_payload, int64_t *nrows);

/* One side of a join: ncols device arrays of nrows values each, in the scan kernels' decoded form (integer types
 * sign-extended to int64, bool 0 / 1, char(1) as the unsigned byte, numeric(p, s) as value * 10^s, float4 / float8 as
 * float8 bits -- what cg_comm_exchange_result delivers for int columns).  d_nulls: NULL, or per column NULL or a device
 * byte array (non-zero = NULL).  key = index of the join key column among them. */
typedef struct CgJoinSide
{
	const int64_t *const *d_cols;
	const uint8_t *const *d_nulls;
	int32_t ncols;
	int32_t key;
	int64_t nrows;
} CgJoinSide;

/* Any scan query over the equi-join of two device-resident sides, folded into `into`:
 *     SELECT <desc's group key and aggregates> FROM build b JOIN probe p ON b.key = p.key WHERE <desc's WHERE tree> GROUP BY ...
 * which is what the MERGE task of a repartition join runs (planner/multi_physical_planner.c:598-687 puts the worker
 * half of the aggregates, the GROUP BY and the WHERE over the join).
 *   Attributes.  A joined row has build->ncols + probe->ncols attributes, build columns first, then probe columns;
 *   columns[] describes them and desc refers to them by that numbering everywhere (WHERE atoms, group columns,
 *   aggregate factors, FILTER and bool-argument atoms, IN lists, column atoms).  A factor product or a column atom may
 *   mix the sides (sum(b.x * p.y), WHERE b.d < p.d).  into must come from cg_partial_create with the same desc and
 *   columns (a different aggregate list or key form is CG_EINVAL).
 *   Join.  Keys are equal when their int64 values are equal; a NULL key joins nothing, on either side; INT64_MIN is a key
 *   like any other.  The two key columns must be of one class: integer-like with equal numeric scale (int widths may
 *   differ, as int48eq allows) or char(1) with char(1).  A float key, or integer-like keys of different scales, is
 *   CG_EUNSUPPORTED.
 *   Everything else follows a scan row: three-valued WHERE, NULL inputs, FILTER, bool arguments, overflow checks,
 *   composite codes (the caller supplies key_col_min / key_col_max), dense or hash tables and the error flags.
 *   enable_qual_pushdown has no effect: there are no skip lists, so nothing is skipped.
 *   term_abs_bound must be 0 in every aggregate (CG_EINVAL otherwise): the number of joined rows is not known before the
 *   probe, so no bound * max_rows proof can hold; sums keep two limb words and every integer term is overflow-checked.
 *   Asynchronous on the library's stream unless stats is given, like cg_scan_shard: kernel-raised errors surface at the
 *   next call that reads the partial.  The join table is allocated in stream order, without a host synchronisation, so
 *   one call per local partition can be enqueued back to back.
 *   stats: rows_scanned = joined rows handed to WHERE, rows_removed_by_filter, rows_passed; kernel_ms = device time of
 *   the build and the probe-aggregate launches; bytes_scanned = 8 bytes per row for the key column and each plan column
 *   of a side, plus one byte per row for each null array read; the chunk-group fields and h2d_bytes are 0.
 *   Refusals: CG_EINVAL for a NULL pointer for a key or plan column, key or ncols out of range, nrows < 0, a nonzero
 *   term_abs_bound or a desc that does not match the partial; CG_EUNSUPPORTED for plans over the kernels' column limit
 *   (8), as for a scan.  nrows == 0 on either side is a no-op that returns CG_OK. */
int cg_join_aggregate(const CgJoinSide *build, const CgJoinSide *probe, const CgColumnDesc *columns, const CgScanDesc *desc,
					  CgPartial *into, CgScanStats *stats);

/* exact bounds from the skip lists (min/max of every chunk that survives chunk-group
 * skipping): the packed group key range and |argument| of every aggregate (0 = unknown,
 * e.g. a chunk without min/max).  Feed them to cg_partial_create / CgAggSpec.term_abs_bound. */
int cg_relation_bounds(const CgRelation *rel, const CgScanDesc *desc, int64_t *key_min, int64_t *key_max,
					   int64_t *term_abs_bound /* [naggs] */, int64_t *rows);
/* The same per group column, for a composite key (CgScanDesc.composite_key): col_min[g] / col_max[g] = bounds of column
 * group_cols[g] over the chunk groups that survive skipping; a column without any non-NULL value there gets
 * col_min > col_max.  A surviving chunk that has values but no min / max (or a float column) is CG_EUNSUPPORTED. */
int cg_relation_key_bounds(const CgRelation *rel, const CgScanDesc *desc, int64_t *col_min /* [ngroup_cols] */,
						   int64_t *col_max /* [ngroup_cols] */);
/* Composite key codes <-> key tuples under desc's codec (composite_key = 1, ngroup_cols = K, key_col_min / key_col_max):
 * values[i * K + c] / nulls[i * K + c] are column c of row i (a NULL's value is 0).  Pure host functions.  A code outside
 * [0, D) or a value outside its column's bounds is CG_EINVAL; D > 2^63 is CG_EUNSUPPORTED. */
int cg_group_key_decode(const CgScanDesc *desc, int64_t n, const int64_t *codes, int64_t *values, uint8_t *nulls);
int cg_group_key_encode(const CgScanDesc *desc, int64_t n, const int64_t *values, const uint8_t *nulls, int64_t *codes);

/* ---------------------------------------------------------------------------------- *
 *  Host-side helpers that belong to the path.
 * ---------------------------------------------------------------------------------- */
/* SelectedChunkMask (columnar_reader.c:1132-1187): mask[chunk] for one stripe; returns the
 * number of chunk groups filtered through *filtered. */
int cg_selected_chunk_mask(const CgRelation *rel, int32_t stripe_index, const CgScanDesc *desc,
						   uint8_t *mask, int64_t *filtered);

/* numeric text of a 128-bit integer with `scale` fractional digits (sum(numeric) output) and
 * of the quotient sum/count with PostgreSQL's select_div_scale rule (avg output, the
 * master-side sum(sum)/sum(count), multi_logical_optimizer.c:1807-1830).  buf >= 64 bytes. */
int cg_numeric_out(int64_t hi, uint64_t lo, int32_t scale, char *buf, size_t buflen);
int cg_numeric_div_out(int64_t hi, uint64_t lo, int32_t scale, int64_t count, char *buf, size_t buflen);
/* The final functions of a CG_AGG_VARIANCE state, as PostgreSQL's numeric_stddev_internal computes them from
 * N = n, S = sum_hi:sum_lo and Q = sumsq[0..3) (192-bit little-endian), all in units of 10^-scale (scale 0..30):
 *   NULL (*is_null = 1, buf = "") when N = 0, or N <= 1 for the sample forms;
 *   num = N * Q - S^2 at display scale 2 * scale; num <= 0 gives the text "0";
 *   otherwise den = N * (N - 1) (samp) or N^2 (pop), rscale = select_div_scale(num, den) (16 significant digits counted
 *   in base-10000 digits, at least 2 * scale, within [0, 1000]), the variance = num / den rounded half away from zero at
 *   rscale, and the standard deviation = the square root of that rounded variance, rounded half away from zero at
 *   rscale.  The text has exactly rscale fraction digits.  A buffer too small for it is CG_EINVAL. */
enum { CG_VAR_POP = 0, CG_VAR_SAMP = 1, CG_STDDEV_POP = 2, CG_STDDEV_SAMP = 3 };
int cg_numeric_var_out(int32_t final, int64_t n, int64_t sum_hi, uint64_t sum_lo, const uint64_t *sumsq /* [3] */, int32_t scale,
					   char *buf, size_t buflen, int32_t *is_null);

/* ---------------------------------------------------------------------------------- *
 *  Synthetic shard writer (bench / test tooling; the on-disk encoding of
 *  backend/columnar/columnar_writer.c:391-654, compression none).
 * ---------------------------------------------------------------------------------- */
enum { CG_GEN_UNIFORM = 0, CG_GEN_SEQUENCE = 1 };
typedef struct CgGenColumn
{
	int32_t attlen;
	int32_t kind;           /* CG_GEN_* */
	int64_t lo;             /* uniform in [lo, hi) / sequence start */
	int64_t hi;
	uint32_t null_ppm;      /* NULL probability in parts per million */
	uint32_t reserved;
} CgGenColumn;

typedef struct CgGenRelation CgGenRelation;
/* value(row, col) = lo + splitmix64(seed ^ col<<56 ^ (first_row+row)) % (hi-lo)
 * null(row, col)  = splitmix64(~seed ^ col<<56 ^ (first_row+row)) % 1000000 < null_ppm */
int cg_gen_relation(const CgGenColumn *cols, int32_t natts, uint64_t nrows, uint64_t first_row,
					uint64_t seed, uint64_t stripe_row_limit, uint32_t chunk_row_limit,
					int32_t nthreads, CgGenRelation **out);
/* Encode caller-supplied columns (values[c][row] int64 / float8 bits, nulls[c] may be NULL). */
int cg_write_relation(const CgColumnDesc *cols, int32_t natts, const int64_t *const *values,
					  const uint8_t *const *nulls, uint64_t nrows, uint64_t stripe_row_limit,
					  uint32_t chunk_row_limit, CgGenRelation **out);
/* columnar.compression of the relations written after the call: CG_COMPRESSION_NONE,
 * CG_COMPRESSION_LZ4 or CG_COMPRESSION_ZSTD (liblz4's LZ4_compress_default / libzstd's
 * ZSTD_compress at level 3, as the reference's CompressBuffer) */
int cg_gen_set_compression(int32_t compression);
int cg_gen_relation_view(const CgGenRelation *g, CgRelation *view);
void cg_gen_relation_free(CgGenRelation *g);

#ifdef __cplusplus
}
#endif
#endif /* CITUS_GPU_H */
