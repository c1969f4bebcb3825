/*
 * cg_jit.cpp -- plan-specialised fused scan kernels, compiled at run time with NVRTC.
 *
 * The reference evaluates a worker task's  Agg <- ColumnarScan  subtree with PostgreSQL's
 * expression interpreter, one row and one fmgr call at a time (ExecQual / ExecProject under
 * ExecScan, backend/columnar/columnar_customscan.c:1907-1913; nodeAgg transition functions for
 * the worker half chosen by planner/multi_logical_optimizer.c:3160-3484).  The ahead-of-time
 * kernels in cg_scan.cu / cg_scan_small.cu interpret the plan too -- loops over quals and
 * aggregates, switches on widths and kinds, dynamic picks out of the per-row register file --
 * and are bound by instruction issue (DESIGN.md section 4).  Here the plan's STRUCTURE (column
 * widths and roles, operators, aggregate kinds and factor shapes, table kind, accumulator
 * layout) is written out as straight-line CUDA and compiled for sm_90a the first time a query
 * shape is seen; the plan's VALUES (constants, key range, bounds, pointers) stay kernel
 * parameters, so `WHERE f < 50` and `WHERE f < 51` share one kernel.  Same decode / filter /
 * aggregate semantics and the same accumulator words as the interpretive kernels: both write
 * the same group table, so a scan may use this kernel for its NULL-free chunk groups and the
 * interpretive one for the rest.
 *
 * Scope: chunk groups whose plan columns have no NULLs (the value stream of such a chunk is a
 * dense array, columnar_reader.c:1542-1572); any mix of 1/2/4/8-byte integers and float4/8;
 * every plan the KPlan language can express.  Table kinds:
 *   GLOBAL  plain aggregate: per-thread registers, warp shuffles, one atomic per warp and word
 *   SMALL   tiny key domain: one private accumulator cell per lane in shared memory (no
 *           atomics), CTA-level combine at the end; a bounded integer sum needs ONE cell -- a
 *           lane sees too few rows to overflow 64 bits -- and is split into the table's
 *           (low 32, high) limbs only when flushed
 *   TABLE   direct-indexed or hash table in global memory: L2 reductions, optionally the
 *           packed count+sum word
 *
 * NVRTC and the CUDA driver are loaded with dlopen; when either is missing the library simply
 * keeps using its ahead-of-time kernels.
 */
#include <dlfcn.h>
#include <stdarg.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <mutex>
#include <string>
#include <vector>

#include <cuda.h>      /* types only (CUlaunchConfig); the driver API itself is resolved with dlsym */

#include "cg_internal.h"

/* ---- minimal NVRTC / driver API surface (opaque handles + ints) ---- */
typedef struct _nvrtcProgram *nvrtcProgram;
typedef int (*nvrtcCreateProgram_t)(nvrtcProgram *, const char *, const char *, int, const char *const *, const char *const *);
typedef int (*nvrtcCompileProgram_t)(nvrtcProgram, int, const char *const *);
typedef int (*nvrtcGetSize_t)(nvrtcProgram, size_t *);
typedef int (*nvrtcGetData_t)(nvrtcProgram, char *);
typedef int (*nvrtcDestroyProgram_t)(nvrtcProgram *);
typedef struct CUmod_st *CUmodule;
typedef struct CUfunc_st *CUfunction;
typedef int (*cuModuleLoadData_t)(CUmodule *, const void *);
typedef int (*cuModuleGetFunction_t)(CUfunction *, CUmodule, const char *);
typedef int (*cuFuncSetAttribute_t)(CUfunction, int, int);
typedef int (*cuOccupancy_t)(int *, CUfunction, int, size_t);
typedef int (*cuLaunchKernelEx_t)(const CUlaunchConfig *, CUfunction, void **, void **);
typedef int (*cuGetErrorString_t)(int, const char **);
#define CG_CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES 8

static struct
{
	bool tried_rtc = false, have_rtc = false, tried_drv = false, have_drv = false;
	nvrtcCreateProgram_t create; nvrtcCompileProgram_t compile; nvrtcGetSize_t cubin_size, log_size;
	nvrtcGetData_t cubin, log; nvrtcDestroyProgram_t destroy;
	cuModuleLoadData_t load; cuModuleGetFunction_t getfn; cuFuncSetAttribute_t setattr; cuOccupancy_t occupancy;
	cuLaunchKernelEx_t launch; cuGetErrorString_t errstr;
} g_api;

static bool load_rtc()
{
	if (g_api.tried_rtc) return g_api.have_rtc;
	g_api.tried_rtc = true;
	void *h = dlopen("libnvrtc.so.12", RTLD_NOW | RTLD_GLOBAL);
	if (!h) h = dlopen("/usr/local/cuda/lib64/libnvrtc.so.12", RTLD_NOW | RTLD_GLOBAL);
	if (!h) h = dlopen("libnvrtc.so", RTLD_NOW | RTLD_GLOBAL);
	if (!h) return false;
	g_api.create = (nvrtcCreateProgram_t) dlsym(h, "nvrtcCreateProgram");
	g_api.compile = (nvrtcCompileProgram_t) dlsym(h, "nvrtcCompileProgram");
	g_api.cubin_size = (nvrtcGetSize_t) dlsym(h, "nvrtcGetCUBINSize");
	g_api.cubin = (nvrtcGetData_t) dlsym(h, "nvrtcGetCUBIN");
	g_api.log_size = (nvrtcGetSize_t) dlsym(h, "nvrtcGetProgramLogSize");
	g_api.log = (nvrtcGetData_t) dlsym(h, "nvrtcGetProgramLog");
	g_api.destroy = (nvrtcDestroyProgram_t) dlsym(h, "nvrtcDestroyProgram");
	g_api.have_rtc = g_api.create && g_api.compile && g_api.cubin_size && g_api.cubin && g_api.log_size && g_api.log && g_api.destroy;
	return g_api.have_rtc;
}

static bool load_drv()
{
	if (g_api.tried_drv) return g_api.have_drv;
	g_api.tried_drv = true;
	void *h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
	if (!h) return false;
	g_api.load = (cuModuleLoadData_t) dlsym(h, "cuModuleLoadData");
	g_api.getfn = (cuModuleGetFunction_t) dlsym(h, "cuModuleGetFunction");
	g_api.setattr = (cuFuncSetAttribute_t) dlsym(h, "cuFuncSetAttribute");
	g_api.occupancy = (cuOccupancy_t) dlsym(h, "cuOccupancyMaxActiveBlocksPerMultiprocessor");
	g_api.launch = (cuLaunchKernelEx_t) dlsym(h, "cuLaunchKernelEx");
	g_api.errstr = (cuGetErrorString_t) dlsym(h, "cuGetErrorString");
	g_api.have_drv = g_api.load && g_api.getfn && g_api.setattr && g_api.occupancy && g_api.launch;
	return g_api.have_drv;
}

static int g_jit_level = -1;
int cg_jit_level(void)
{
	if (g_jit_level < 0) { const char *e = getenv("CG_JIT"); g_jit_level = e ? atoi(e) : 1; }
	return g_jit_level;
}
void cg_jit_set_level(int level) { g_jit_level = level < 0 ? 0 : level; }

/* ------------------------------------------------------------------------------ *
 *  Code generation.
 * ------------------------------------------------------------------------------ */
#define JIT_THREADS 256
/* a lane's private 64-bit sum cell is exact while |term| * rows-per-lane < 2^63; launches are cut so
 * that no lane sees more rows than this */
#define JIT_LANE_ROWS_CAP (1ll << 22)
#define JIT_NARROW_ROWS_CAP 160ll   /* four 10 000-row chunk groups per CTA: 40 rows per lane each */
#define JIT_MAX_CHUNK_ROWS 100000ll    /* chunk_group_row_limit's upper bound (columnar.c:50-51) */

enum { JK_GLOBAL = 0, JK_SMALL = 1, JK_TABLE = 2 };

struct JitShape
{
	int kind = JK_GLOBAL;
	int R = 2, U = 2;
	int nhot = 0;                     /* SMALL: cells per group */
	int hot0[CG_MAX_AGGS];            /* SMALL: first cell of the aggregate, -1 = none */
	bool lane1[CG_MAX_AGGS];          /* SMALL: integer sum kept in one cell per lane */
	/* SMALL, narrow cells: a lane sees at most lane_rows_cap rows per launch, so a sum whose |term| * cap < 2^31 needs only
	 * 32 bits there; two such sums (or the row count and one sum) share one 64-bit cell and one shared-memory update:
	 * half 1 = high 32 bits (two's complement), half 0 = low 32 bits holding sum(term + bias) (non-negative, so that it never
	 * borrows from the high half; the bias times the group's row count is taken off at the flush), -1 = a cell of its own */
	int half[CG_MAX_AGGS];
	int64_t bias[CG_MAX_AGGS];
	int rows_partner = -1;            /* aggregate in the high half of cell 0 (whose low half counts the rows), -1 = none */
	int ncell[CG_MAX_AGGS];           /* SMALL: cell of a filtered aggregate's no-input counter, -1 = none */
	int qcell[CG_MAX_AGGS];           /* SMALL: first of the qlimbs cells of a variance aggregate's sum(x^2), -1 = none */
	long long lane_rows_cap = (1ll << 22);
	int min_blocks = 0;               /* __launch_bounds__ second argument, 0 = none */
	size_t smem = 0;
	bool packed = false;
	int pack_agg = -1;
	uint32_t nullable = 0;            /* plan columns read through exists bitmap + rank directory where a chunk has NULLs */
};

static void addf(std::string &s, const char *fmt, ...) __attribute__((format(printf, 2, 3)));
static void addf(std::string &s, const char *fmt, ...)
{
	char buf[1024];
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(buf, sizeof buf, fmt, ap);
	va_end(ap);
	s += buf;
}

static bool agg_has_value(const KAgg &g) { return g.kind != CG_AGG_COUNT_STAR && g.kind != CG_AGG_COUNT; }
static bool agg_two_limbs(const KAgg &g) { return (g.kind == CG_AGG_SUM || g.kind == CG_AGG_VARIANCE) && !g.is_float && g.nlimbs == 2; }
static bool agg_is_var(const KAgg &g) { return g.kind == CG_AGG_VARIANCE; }

/* sum(x^2) limb l of a variance aggregate a as an expression over x^2 = qh<a>:ql<a> */
static std::string square_limb_expr(int a, int qlimbs, int l)
{
	char b[96];
	if (qlimbs == 1) snprintf(b, sizeof b, "ql%d", a);
	else snprintf(b, sizeof b, "(q%c%d %s)", l < 2 ? 'l' : 'h', a, (l & 1) ? ">> 32" : "& 0xffffffffull");
	return b;
}

static std::string agg_null_expr(const KAgg &g, const JitShape &sh);
static std::string agg_noinput_expr(const KPlan &plan, int a, const JitShape &sh);

static void choose_shape(const KPlan &plan, uint32_t nullable, JitShape *sh)
{
	sh->nullable = plan.ncols >= 32 ? nullable : (nullable & ((1u << plan.ncols) - 1u));
	sh->kind = plan.mode == CG_MODE_GLOBAL ? JK_GLOBAL : JK_TABLE;
	/* two rows per thread and step (one 16-byte load per 8-byte column), two steps loaded before any is
	 * consumed: the best of the (R, U) grid on every probed shape (tools/kernel_probe.py) */
	sh->R = 2;
	sh->U = 2;
	{
		const char *r = getenv("CG_JIT_R"), *u = getenv("CG_JIT_U");
		if (r && (atoi(r) == 2 || atoi(r) == 4)) sh->R = atoi(r);
		if (u && atoi(u) >= 1 && atoi(u) <= 4) sh->U = atoi(u);
	}
	for (int a = 0; a < CG_MAX_AGGS; a++)
	{
		sh->hot0[a] = -1; sh->lane1[a] = false; sh->half[a] = -1; sh->bias[a] = 0; sh->ncell[a] = -1; sh->qcell[a] = -1;
	}
	if (plan.mode == CG_MODE_DENSE)
	{
		static int narrow_on = -1;
		if (narrow_on < 0) { const char *e = getenv("CG_JIT_NARROW"); narrow_on = e ? atoi(e) : 1; }
		/* candidates for 32-bit halves */
		int cand[CG_MAX_AGGS], ncand = 0;
		for (int a = 0; a < plan.naggs && narrow_on; a++)
		{
			const KAgg &g = plan.aggs[a];
			if (g.kind == CG_AGG_SUM && !g.is_float && g.tbound > 0 && (__int128) g.tbound * JIT_NARROW_ROWS_CAP < ((__int128) 1 << 31)) cand[ncand++] = a;
		}
		bool taken[CG_MAX_AGGS] = {false};
		int nhot = 1;
		if (ncand > 0)
		{
			/* cell 0: rows (low) + the first candidate (high) */
			sh->rows_partner = cand[0]; sh->hot0[cand[0]] = 0; sh->half[cand[0]] = 1; sh->lane1[cand[0]] = true; taken[cand[0]] = true;
			/* further cells: a candidate without nullable inputs in the low half (biased), another one in the high half */
			for (int i = 1; i < ncand; i++)
			{
				const int x = cand[i];
				if (taken[x] || !agg_noinput_expr(plan, x, *sh).empty()) continue;
				int y = -1;
				for (int j = 1; j < ncand; j++) if (j != i && !taken[cand[j]]) { y = cand[j]; break; }
				if (y < 0) break;
				sh->hot0[x] = nhot; sh->half[x] = 0; sh->bias[x] = plan.aggs[x].tbound; sh->lane1[x] = true; taken[x] = true;
				sh->hot0[y] = nhot; sh->half[y] = 1; sh->lane1[y] = true; taken[y] = true;
				nhot++;
			}
		}
		for (int a = 0; a < plan.naggs; a++)
		{
			const KAgg &g = plan.aggs[a];
			if (!agg_has_value(g) || taken[a]) continue;
			sh->hot0[a] = nhot;
			if ((g.kind == CG_AGG_SUM || agg_is_var(g)) && !g.is_float)
			{
				/* one cell if the lane's running sum cannot overflow: the table's own single-word
				 * guarantee, or the caller's term bound times the per-lane row cap */
				bool one = g.nlimbs == 1 ||
						   (g.tbound > 0 && (__int128) g.tbound * JIT_LANE_ROWS_CAP < ((__int128) 1 << 63));
				sh->lane1[a] = one;
				nhot += one ? 1 : 2;
			}
			else
				nhot += 1;
			/* sum(x^2): a cell per limb word (a lane's limb grows by < 2^32 per row; the one-word form is bounded by the table's
			 * own guarantee) */
			if (agg_is_var(g)) { sh->qcell[a] = nhot; nhot += g.qlimbs; }
		}
		/* rejected rows are common, not rare like NULL inputs: a filtered aggregate's no-input counter gets a cell too, and
		 * so does the counter of a bool_and / bool_or, whose UNKNOWN rows are as common as its atoms' NULLs, and that of a
		 * CASE, whose NULL results are as common as its arms' WHEN trees fail */
		for (int a = 0; a < plan.naggs; a++)
			if (plan.nfexpr[a] > 0 || plan.aggs[a].barg || plan.cnarms[a] > 0) sh->ncell[a] = nhot++;
		size_t bytes = (size_t) plan.capacity * nhot * sizeof(uint64_t) * JIT_THREADS;
		if (plan.capacity <= 4096 && bytes <= 200 * 1024)
		{
			sh->kind = JK_SMALL;
			sh->nhot = nhot;
			sh->smem = bytes;
			if (ncand > 0) sh->lane_rows_cap = JIT_NARROW_ROWS_CAP;
			/* registers: four CTAs per SM when their cells fit (the compiler is held to 64 registers) */
			if (bytes + 4096 <= 55 * 1024) sh->min_blocks = 4;
			const char *mb = getenv("CG_JIT_MINB");
			if (mb) sh->min_blocks = atoi(mb);
		}
		else
		{
			/* not the shared-memory kind after all: no narrow cells, the no-input counters stay in the table */
			for (int a = 0; a < CG_MAX_AGGS; a++) { sh->half[a] = -1; sh->bias[a] = 0; sh->ncell[a] = -1; }
			sh->rows_partner = -1;
		}
	}
	if (sh->kind == JK_TABLE && plan.packed)
		for (int a = 0; a < plan.naggs && sh->pack_agg < 0; a++)
		{
			const KAgg &g = plan.aggs[a];
			if (g.kind == CG_AGG_SUM && !g.is_float && g.nlimbs == 1 && g.word0 == plan.pack_word) { sh->pack_agg = a; sh->packed = true; }
		}
}

static const char *op_identity(int op)
{
	switch (op)
	{
		case CG_WORD_MIN: return "0x7fffffffffffffffull";
		case CG_WORD_MAX: return "0x8000000000000000ull";
		case CG_WORD_FMIN: return "0xffffffffffffffffull";
		case CG_WORD_AND: return "0xffffffffffffffffull";
		case CG_WORD_OR: return "0ull";
		default: return "0ull";
	}
}

/* expression combining accumulator `acc` with value `v` (both uint64_t expressions) */
static std::string op_combine(int op, const std::string &acc, const std::string &v)
{
	switch (op)
	{
		case CG_WORD_ADD: return acc + " + " + v;
		case CG_WORD_MIN: return "(uint64_t) smin64((int64_t) " + acc + ", (int64_t) " + v + ")";
		case CG_WORD_MAX: return "(uint64_t) smax64((int64_t) " + acc + ", (int64_t) " + v + ")";
		case CG_WORD_FADD: return "(uint64_t) __double_as_longlong(__longlong_as_double((int64_t) " + acc + ") + __longlong_as_double((int64_t) " + v + "))";
		case CG_WORD_FMIN: return "umin64(" + acc + ", " + v + ")";
		case CG_WORD_AND: return "(" + acc + " & " + v + ")";
		case CG_WORD_OR: return "(" + acc + " | " + v + ")";
		default: return "umax64(" + acc + ", " + v + ")";
	}
}

/* statement applying value expression `v` to global word pointer expression `p` */
static std::string op_apply_global(int op, const std::string &p, const std::string &v)
{
	switch (op)
	{
		case CG_WORD_ADD: return "red_add(" + p + ", " + v + ");";
		case CG_WORD_MIN: return "atomicMin((long long *) (" + p + "), (long long) (" + v + "));";
		case CG_WORD_MAX: return "atomicMax((long long *) (" + p + "), (long long) (" + v + "));";
		case CG_WORD_FADD: return "atomicAdd((double *) (" + p + "), __longlong_as_double((long long) (" + v + ")));";
		case CG_WORD_FMIN: return "atomicMin((unsigned long long *) (" + p + "), (unsigned long long) (" + v + "));";
		case CG_WORD_AND: return "atomicAnd((unsigned long long *) (" + p + "), (unsigned long long) (" + v + "));";
		case CG_WORD_OR: return "atomicOr((unsigned long long *) (" + p + "), (unsigned long long) (" + v + "));";
		default: return "atomicMax((unsigned long long *) (" + p + "), (unsigned long long) (" + v + "));";
	}
}


static bool plan_has_args(const KPlan &plan)
{
	for (int a = 0; a < plan.naggs; a++)
		if (plan.nargexpr[a] > 0) return true;
	return false;
}

static bool op_is_list(int op) { return op == CG_OP_IN || op == CG_OP_NOT_IN; }

/* some WHERE or pool atom is IN / NOT IN: the kernel reads P.sets and the atoms' KSet entries */
static bool plan_has_sets(const KPlan &plan)
{
	for (int q = 0; q < plan.nquals; q++) if (op_is_list(plan.qop[q])) return true;
	for (int q = 0; q < plan.nfquals; q++) if (op_is_list(plan.fop[q])) return true;
	return false;
}

/* some WHERE or pool atom compares two columns: the prelude defines their comparison helpers */
static bool plan_has_column_atoms(const KPlan &plan)
{
	for (int q = 0; q < plan.nquals; q++) if (cg_op_is_column(plan.qop[q])) return true;
	for (int q = 0; q < plan.nfquals; q++) if (cg_op_is_column(plan.fop[q])) return true;
	return false;
}

/* The host's structs restated for NVRTC.  A plan without bool_and / bool_or arguments restates KPlan up to fexpr and
 * KAgg's barg byte as padding: its kernel reads nothing behind them (the arguments' trees are written out as code), so
 * the plan parameter it declares is a prefix of the one the host passes, and its source is the one such plans had
 * before the arguments existed -- the same kernel cache key, the same compiled code. */
/* gcol is restated with the two entries it had before composite keys: the generated code names its key columns v<c> and
 * never reads gcol, and naggs follows at the same offset either way (the padding after gcol absorbs the difference), so
 * the source of every existing plan shape stays as it was */
#define KPLAN_GCOL_RESTATED 2
static_assert(offsetof(KPlan, naggs) == offsetof(KPlan, gcol) + 4 && (offsetof(KPlan, gcol) + KPLAN_GCOL_RESTATED + 3) / 4 * 4 == offsetof(KPlan, naggs),
			  "a two-entry gcol must give KPlan's layout");

static void gen_prelude(std::string &s, const KPlan &plan)
{
	const bool args = plan_has_args(plan);
	/* plans with CASE arms restate the whole struct, plans with IN lists all but the column atoms and the arms, plans with
	 * a composite key all but the lists; the others stop at fexpr or argexpr as before */
	const bool cases = plan.ncase > 0;
	const bool sets = plan_has_sets(plan) || cases;
	const bool composite = plan.composite || sets;
	const bool tail = args || composite;
	s +=
		"typedef unsigned long long uint64_t; typedef long long int64_t; typedef unsigned int uint32_t; typedef int int32_t;\n"
		"typedef unsigned short uint16_t; typedef short int16_t; typedef unsigned char uint8_t; typedef signed char int8_t;\n"
		"struct DevChunkCol { uint64_t values_off; uint64_t exists_off; uint64_t rank_off; uint32_t value_count; uint32_t row_count; };\n";
	if (sets) s += "struct KSet { uint16_t off; uint16_t len; uint8_t steps; uint8_t nnull; uint8_t pad[2]; };\n";
	if (cases)
		addf(s,
			 "struct KCmp { int64_t mul; uint8_t col2; uint8_t right; uint8_t pad[6]; };\n"
			 "struct KArm { int64_t a[3]; int64_t b[3]; int8_t nwhen; int8_t form; int8_t nfactors; int8_t pcol[3]; int8_t when[%d]; };\n",
			 CG_MAX_QEXPR);
	s += args ? "struct KAgg { int8_t kind; int8_t nfactors; int8_t is_float; int8_t nlimbs; int8_t pcol[3]; int8_t word0; int8_t nullword; int8_t ovchk; int8_t filt; int8_t barg;"
			  : "struct KAgg { int8_t kind; int8_t nfactors; int8_t is_float; int8_t nlimbs; int8_t pcol[3]; int8_t word0; int8_t nullword; int8_t ovchk; int8_t filt; int8_t pad;";
	/* the sum(x^2) fields sit in KAgg's padding: plans without a variance aggregate restate the struct without them */
	s += cg_plan_has_variance(plan.aggs, plan.naggs) ? " int8_t qlimbs; int8_t qword;\n" : "\n";
	s += "  int64_t a[3]; int64_t b[3]; int64_t bound; int64_t tbound; };\n";
	addf(s,
		 "struct KPlan { const uint8_t *arena; const DevChunkCol *chunkcols; const uint32_t *selected; uint32_t nselected; int32_t nstaged;\n"
		 "  int32_t ncols; uint8_t slot[%d]; uint8_t len[%d]; uint8_t isfloat[%d];\n"
		 "  int32_t nquals; uint8_t qcol[%d]; uint8_t qop[%d]; int64_t qk[%d]; int64_t qlo[%d]; int64_t qhi[%d]; uint8_t qneg[%d];\n"
		 "  int32_t ngroup; uint8_t gcol[%d]; int32_t naggs; KAgg aggs[%d];\n"
		 "  int32_t mode; int32_t nwords; int32_t stride; uint64_t *table; int64_t *hkeys; uint64_t capacity; int32_t hash_shift;\n"
		 "  int64_t key_min; int64_t key_min1; uint64_t range1; uint8_t wordop[%d]; unsigned long long *stats;\n"
		 "  int8_t hot_of_word[%d]; int32_t nhot; uint64_t *packed; int32_t pack_shift; int32_t pack_word;\n"
		 "  int32_t nqexpr; int8_t qexpr[%d]; int32_t slices; uint32_t slice_rows; uint32_t max_cg_rows;\n"
		 "  int32_t nfquals; uint8_t fcol[%d]; uint8_t fop[%d]; int64_t fk[%d]; int64_t flo[%d]; int64_t fhi[%d]; uint8_t fneg[%d];\n"
		 "  int32_t nfexpr[%d]; int8_t fexpr[%d][%d];%s",
		 CG_KMAX_COLS, CG_KMAX_COLS, CG_KMAX_COLS, CG_MAX_QUALS, CG_MAX_QUALS, CG_MAX_QUALS, CG_MAX_QUALS, CG_MAX_QUALS, CG_MAX_QUALS,
		 KPLAN_GCOL_RESTATED, CG_MAX_AGGS, CG_KMAX_WORDS, CG_KMAX_WORDS, CG_MAX_QEXPR, CG_MAX_FILTER_QUALS, CG_MAX_FILTER_QUALS,
		 CG_MAX_FILTER_QUALS, CG_MAX_FILTER_QUALS, CG_MAX_FILTER_QUALS, CG_MAX_FILTER_QUALS, CG_MAX_AGGS, CG_MAX_AGGS, CG_MAX_QEXPR,
		 tail ? "\n" : " };\n");
	if (tail) addf(s, "  int32_t nargexpr[%d]; int8_t argexpr[%d][%d];%s", CG_MAX_AGGS, CG_MAX_AGGS, CG_MAX_QEXPR, composite ? "\n" : " };\n");
	if (composite) addf(s, "  int32_t composite; int64_t kmin[%d]; uint64_t kradix[%d];%s", CG_MAX_GROUP_COLS, CG_MAX_GROUP_COLS, sets ? "\n" : " };\n");
	if (sets) addf(s, "  const uint64_t *sets; KSet qset[%d]; KSet fset[%d];%s", CG_MAX_QUALS, CG_MAX_FILTER_QUALS, cases ? "\n" : " };\n");
	if (cases)
		addf(s, "  KCmp qcc[%d]; KCmp fcc[%d]; int32_t ncase; int8_t cfirst[%d]; int8_t cnarms[%d]; KArm arms[%d]; };\n", CG_MAX_QUALS,
			 CG_MAX_FILTER_QUALS, CG_MAX_AGGS, CG_MAX_AGGS, CG_MAX_CASE_ARMS);
	/* the text above must describe the host's structs exactly (without arguments: the prefix up to fexpr; with arguments
	 * only: the prefix up to argexpr; with a composite key: the prefix up to the lists; with lists: the prefix up to the
	 * column atoms' KCmp entries, which the generated code never reads -- their columns and scales are written out) */
	const auto upto = [](size_t off) { return (off + alignof(KPlan) - 1) / alignof(KPlan) * alignof(KPlan); };
	const size_t size = cases ? sizeof(KPlan) : sets ? upto(offsetof(KPlan, qcc)) : composite ? upto(offsetof(KPlan, sets))
																			   : args ? upto(offsetof(KPlan, composite)) : upto(offsetof(KPlan, nargexpr));
	addf(s, "static_assert(sizeof(DevChunkCol) == %zu, \"DevChunkCol\");\n", sizeof(DevChunkCol));
	addf(s, "static_assert(sizeof(KAgg) == %zu, \"KAgg\");\n", sizeof(KAgg));
	if (cases) addf(s, "static_assert(sizeof(KArm) == %zu, \"KArm\");\n", sizeof(KArm));
	addf(s, "static_assert(sizeof(KPlan) == %zu, \"KPlan\");\n", size);
	/* (NVRTC has no offsetof; same field order + same total size is the check) */
	s +=
		"#define EMPTY_KEY ((int64_t) 0x8000000000000000ull)\n"
		"__device__ __forceinline__ void ld16(const void *p, uint64_t &a, uint64_t &b) { asm(\"ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];\" : \"=l\"(a), \"=l\"(b) : \"l\"(p)); }\n"
		"__device__ __forceinline__ uint64_t ld8(const void *p) { uint64_t a; asm(\"ld.global.nc.L1::no_allocate.u64 %0, [%1];\" : \"=l\"(a) : \"l\"(p)); return a; }\n"
		"__device__ __forceinline__ uint64_t ld4(const void *p) { uint32_t a; asm(\"ld.global.nc.L1::no_allocate.u32 %0, [%1];\" : \"=r\"(a) : \"l\"(p)); return a; }\n"
		"__device__ __forceinline__ uint64_t ld2(const void *p) { uint16_t a; asm(\"ld.global.nc.L1::no_allocate.u16 %0, [%1];\" : \"=h\"(a) : \"l\"(p)); return a; }\n"
		"__device__ __forceinline__ uint64_t ld1(const void *p) { uint32_t a; asm(\"ld.global.nc.L1::no_allocate.u8 %0, [%1];\" : \"=r\"(a) : \"l\"(p)); return a; }\n"
		"__device__ __forceinline__ void red_add(uint64_t *p, uint64_t v) { asm volatile(\"red.global.add.u64 [%0], %1;\" :: \"l\"(p), \"l\"(v) : \"memory\"); }\n"
		"__device__ __forceinline__ int64_t smin64(int64_t a, int64_t b) { return a < b ? a : b; }\n"
		"__device__ __forceinline__ int64_t smax64(int64_t a, int64_t b) { return a > b ? a : b; }\n"
		"__device__ __forceinline__ uint64_t umin64(uint64_t a, uint64_t b) { return a < b ? a : b; }\n"
		"__device__ __forceinline__ uint64_t umax64(uint64_t a, uint64_t b) { return a > b ? a : b; }\n"
		/* [PG] float8 btree order: NaN equals NaN and is greater than everything */
		"__device__ __forceinline__ int fcmp(int64_t a, int64_t b) { double x = __longlong_as_double(a), y = __longlong_as_double(b);\n"
		"  bool xn = x != x, yn = y != y; return (xn || yn) ? ((int) xn - (int) yn) : ((x > y) - (x < y)); }\n"
		/* every NaN is the one largest code, above +inf */
		"__device__ __forceinline__ uint64_t f8_ordered(int64_t bits) { uint64_t u = (uint64_t) bits;\n"
		"  if ((u & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return ~0ull; return (u >> 63) ? ~u : (u | 0x8000000000000000ull); }\n"
		"__device__ __forceinline__ int64_t mul_ovf(int64_t x, int64_t y, bool &o) { int64_t l = (int64_t) ((uint64_t) x * (uint64_t) y);\n"
		"  o |= __mul64hi(x, y) != (l >> 63); return l; }\n"
		"__device__ __forceinline__ int64_t add_ovf(int64_t x, int64_t y, bool &o) { int64_t r = (int64_t) ((uint64_t) x + (uint64_t) y);\n"
		"  o |= ((x ^ r) & (y ^ r)) < 0; return r; }\n"
		"__device__ __noinline__ void raise_flag(unsigned long long *stats, unsigned long long flag) { atomicOr(stats + 2, flag); }\n"
		"__device__ __forceinline__ uint64_t wsum(uint64_t x) { for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o); return x; }\n"
		"__device__ __noinline__ uint64_t hash_slot_slow(const KPlan &P, int64_t key, uint64_t h) {\n"
		"  const uint64_t mask = P.capacity - 1;\n"
		"  for (uint32_t probes = 0; probes < 8192; probes++) {\n"
		"    unsigned long long *kp = (unsigned long long *) (P.hkeys + h);\n"
		"    long long cur = (long long) __ldcg(kp);\n"
		"    if (cur == key) return h;\n"
		"    if (cur == EMPTY_KEY) { long long old = (long long) atomicCAS(kp, (unsigned long long) EMPTY_KEY, (unsigned long long) key); if (old == EMPTY_KEY || old == key) return h; }\n"
		"    h = (h + 1) & mask; }\n"
		"  raise_flag(P.stats, 1ull); return ~0ull; }\n";
	if (sets)
		/* cg_set_code (cg_internal.h) and the branch-free membership search of cg_device.cuh's set_contains: a fixed number of
		 * halvings per list, L1-allocating read-only loads of the codes */
		s +=
			"__device__ __forceinline__ uint64_t set_code_i(int64_t v) { return (uint64_t) v ^ 0x8000000000000000ull; }\n"
			"__device__ __forceinline__ uint64_t set_code_f(int64_t v) { uint64_t u = (uint64_t) v; if (u == 0x8000000000000000ull) u = 0;\n"
			"  if ((u & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return ~0ull; return (u >> 63) ? ~u : (u | 0x8000000000000000ull); }\n"
			"__device__ __forceinline__ bool in_set(const uint64_t *sets, const KSet &k, uint64_t key) {\n"
			"  if (k.len == 0) return false;\n"
			"  const uint64_t *b = sets + k.off; uint32_t n = k.len;\n"
			"  for (uint32_t i = 0; i < k.steps; i++) { const uint32_t h = n >> 1; b = (__ldg(b + h) <= key) ? b + h : b; n -= h; }\n"
			"  return __ldg(b) == key; }\n";
	if (plan_has_column_atoms(plan))
		/* column atoms (cg_device.cuh, col_cmp): float sides compare their cg_set_code, integer-like sides of different scales
		 * the sign of x * m - y in 128 bits */
		s +=
			"__device__ __forceinline__ uint64_t col_code_f(int64_t v) { uint64_t u = (uint64_t) v; if (u == 0x8000000000000000ull) u = 0;\n"
			"  if ((u & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return ~0ull; return (u >> 63) ? ~u : (u | 0x8000000000000000ull); }\n"
			"__device__ __forceinline__ int cmp_scaled(int64_t x, int64_t m, int64_t y) { const int64_t h = __mul64hi(x, m), yh = y >> 63;\n"
			"  const uint64_t l = (uint64_t) x * (uint64_t) m; return h != yh ? (h < yh ? -1 : 1) : ((l > (uint64_t) y) - (l < (uint64_t) y)); }\n";
}

static bool col_nullable(const JitShape &sh, int c) { return (sh.nullable >> c) & 1u; }

/* value of plan column c, row j of step u, as an int64_t expression (widened like fetch_att) */
static std::string col_value(const KPlan &plan, const JitShape &sh, int c, int u, int j)
{
	char raw[64];
	int len = plan.len[c];
	int shift = 0;
	if (col_nullable(sh, c))
		snprintf(raw, sizeof raw, "x%d_%d_%d", c, u, j);     /* one zero-extended datum per row */
	else
	{
		int word = j * len / 8;
		shift = (j * len % 8) * 8;
		if (sh.R * len < 8) { word = 0; shift = j * len * 8; }
		snprintf(raw, sizeof raw, "w%d_%d_%d", c, u, word);
	}
	std::string x = raw;
	char buf[256];
	switch (len)
	{
		case 8: return "(int64_t) " + x;
		case 4:
			if (plan.isfloat[c]) snprintf(buf, sizeof buf, "__double_as_longlong((double) __uint_as_float((uint32_t) (%s >> %d)))", raw, shift);
			else snprintf(buf, sizeof buf, "(int64_t) (int32_t) (uint32_t) (%s >> %d)", raw, shift);
			return buf;
		case 2: snprintf(buf, sizeof buf, "(int64_t) (int16_t) (uint16_t) (%s >> %d)", raw, shift); return buf;
		default: snprintf(buf, sizeof buf, "(int64_t) (int8_t) (uint8_t) (%s >> %d)", raw, shift); return buf;
	}
}

static void gen_loads(std::string &s, const KPlan &plan, const JitShape &sh, int u)
{
	const char *T = "\t\t\t\t\t";
	for (int c = 0; c < plan.ncols; c++)
	{
		const int len = plan.len[c];
		if (col_nullable(sh, c))
		{
			/* K1 for a chunk with NULLs (DeserializeBoolArray / DeserializeDatumArray, columnar_reader.c:1506-1572):
			 * NULL rows occupy no bytes of the value stream, so row -> value index = rank directory entry of the
			 * row's 64-row block + popcount of the exists bits below it.  r is a multiple of R, so the R rows of
			 * this step share one bitmap word; bits past the last row are zero padding. */
			addf(s, "%sif (n%d) {\n", T, c);
			addf(s, "%s\tconst uint64_t bw = sb%d[(r >> 6) - wfirst];\n%s\tconst uint32_t sh = r & 63u;\n", T, c, T);
			addf(s, "%s\tuint32_t vi = sk%d[(r >> 6) - wfirst] + (uint32_t) __popcll(bw & ((1ull << sh) - 1ull));\n", T, c);
			addf(s, "%s\te%d_%d = (uint32_t) (bw >> sh) & %uu;\n", T, c, u, (1u << sh.R) - 1u);
			for (int j = 0; j < sh.R; j++)
				addf(s, "%s\tif (e%d_%d & %uu) { x%d_%d_%d = ld%d(p%d + (uint64_t) vi * %d); vi++; }\n", T, c, u, 1u << j, c, u, j, len, c, len);
			addf(s, "%s} else {\n%s\te%d_%d = %uu;\n", T, T, c, u, (1u << sh.R) - 1u);
			for (int j = 0; j < sh.R; j++)
				addf(s, "%s\tif (r + %d < rows) x%d_%d_%d = ld%d(p%d + (uint64_t) (r + %d) * %d);\n", T, j, c, u, j, len, c, j, len);
			addf(s, "%s}\n", T);
			continue;
		}
		int bytes = sh.R * len;
		if (bytes >= 16)
			for (int k = 0; k < bytes / 16; k++)
				addf(s, "%sld16(p%d + (uint64_t) r * %d + %d, w%d_%d_%d, w%d_%d_%d);\n", T, c, len, 16 * k, c, u, 2 * k, c, u, 2 * k + 1);
		else
			addf(s, "%sw%d_%d_0 = ld%d(p%d + (uint64_t) r * %d);\n", T, c, u, bytes, c, len);
	}
}

/* integer / float term of aggregate number `a` as an expression over v<c>; factor constants stay
 * kernel parameters unless the factor is the bare column */
static std::string term_expr(const KAgg &g, int a)
{
	std::string e;
	for (int f = 0; f < g.nfactors; f++)
	{
		char buf[256];
		if (g.is_float)
		{
			double fa, fb;
			memcpy(&fa, &g.a[f], 8); memcpy(&fb, &g.b[f], 8);
			if (g.a[f] == 0 && fb == 1.0) snprintf(buf, sizeof buf, "__longlong_as_double(v%d)", g.pcol[f]);
			else snprintf(buf, sizeof buf, "(__longlong_as_double(P.aggs[%d].a[%d]) + __longlong_as_double(P.aggs[%d].b[%d]) * __longlong_as_double(v%d))",
						  a, f, a, f, g.pcol[f]);
		}
		else if (g.ovchk)
		{
			/* no proven bound: every factor and product is checked (mul_ovf / add_ovf set ov<a>) */
			if (g.a[f] == 0 && g.b[f] == 1) snprintf(buf, sizeof buf, "v%d", g.pcol[f]);
			else snprintf(buf, sizeof buf, "add_ovf(P.aggs[%d].a[%d], mul_ovf(P.aggs[%d].b[%d], v%d, ov%d), ov%d)", a, f, a, f, g.pcol[f], a, a);
			e = f ? "mul_ovf(" + e + ", " + buf + ", ov" + std::to_string(a) + ")" : std::string(buf);
			continue;
		}
		else if (g.a[f] == 0 && g.b[f] == 1) snprintf(buf, sizeof buf, "v%d", g.pcol[f]);
		else snprintf(buf, sizeof buf, "(P.aggs[%d].a[%d] + P.aggs[%d].b[%d] * v%d)", a, f, a, f, g.pcol[f]);
		if (f) e += " * ";
		e += buf;
	}
	return e;
}

/* "an input of aggregate a is NULL" as an expression, or "" when no factor column is nullable */
static std::string agg_null_expr(const KAgg &g, const JitShape &sh)
{
	std::string e;
	for (int f = 0; f < g.nfactors; f++)
	{
		int c = g.pcol[f];
		if (!col_nullable(sh, c)) continue;
		bool dup = false;
		for (int f2 = 0; f2 < f; f2++) if (g.pcol[f2] == c) dup = true;
		if (dup) continue;
		char buf[32];
		snprintf(buf, sizeof buf, "z%d", c);
		if (!e.empty()) e += " || ";
		e += buf;
	}
	return e;
}

/* "aggregate a gives no input on this row" (NULL input, bool_and / bool_or argument UNKNOWN -- neither TRUE: at<a> nor
 * FALSE: af<a> --, or its FILTER is not TRUE: f<a>), or "" when it always does */
static std::string agg_noinput_expr(const KPlan &plan, int a, const JitShape &sh)
{
	const KAgg &g = plan.aggs[a];
	std::string e = g.kind == CG_AGG_COUNT_STAR ? std::string() : agg_null_expr(g, sh);
	if (plan.cnarms[a] > 0) e = "cn" + std::to_string(a);     /* the CASE's value is NULL (gen_case) */
	if (plan.nargexpr[a] > 0) e += (e.empty() ? "" : " || ") + ("(!at" + std::to_string(a) + " && !af" + std::to_string(a) + ")");
	if (plan.nfexpr[a] > 0) e += (e.empty() ? "!f" : " || !f") + std::to_string(a);
	return e;
}

/* a postfix tree over the atoms <prefix><q>; dual: with AND and OR swapped (over "is FALSE" atoms: "the tree is FALSE") */
static std::string tree_expr(int n, const int8_t *expr, const char *prefix, bool dual = false)
{
	std::vector<std::string> st;
	for (int i = 0; i < n; i++)
	{
		int t = expr[i];
		if (t >= 0) st.push_back(prefix + std::to_string(t));
		else
		{
			std::string b = st.back(); st.pop_back();
			std::string a = st.back(); st.pop_back();
			st.push_back("(" + a + (((t == CG_QX_AND) != dual) ? " && " : " || ") + b + ")");
		}
	}
	return st.back();
}

/* "the row's value is in the list of atom q" (IN / NOT IN), as the variable h<prefix><q> the row block defines first */
static std::string found_var(const char *prefix, int q) { return "h" + std::string(prefix) + std::to_string(q); }

/* one atom "column <op> constant" on plan column c, its constants in P.<arr>k / <arr>lo / <arr>hi / <arr>neg [q]; an atom
 * on a NULL input is not TRUE (three-valued logic).  IS [NOT] NULL reads only the NULL flag (in the plain form, where the
 * column has no NULL, it is a constant); IN / NOT IN read found_var(prefix, q) and the list's NULL flag P.<arr>set[q].nnull */
/* the other side of column atom q of the WHERE list (arr "q") or the pool (arr "f") */
static const KCmp &atom_cmp(const KPlan &plan, const char *arr, int q) { return arr[0] == 'q' ? plan.qcc[q] : plan.fcc[q]; }

/* "neither column of atom q is NULL" as a prefix "!z<c> && ..." ("" when neither column is nullable) */
static std::string atom_known(const KPlan &plan, const JitShape &sh, int c, int op, const char *arr, int q)
{
	std::string nn;
	if (col_nullable(sh, c)) nn += "!z" + std::to_string(c) + " && ";
	if (cg_op_is_column(op))
	{
		const int c2 = atom_cmp(plan, arr, q).col2;
		if (c2 != c && col_nullable(sh, c2)) nn += "!z" + std::to_string(c2) + " && ";
	}
	return nn;
}

static std::string atom_expr(const KPlan &plan, const JitShape &sh, int c, int op, bool neg, const char *arr, int q, const char *prefix)
{
	char buf[256], nn[32] = "";
	if (op == CG_OP_IS_NULL || op == CG_OP_IS_NOT_NULL)
	{
		if (!col_nullable(sh, c)) return op == CG_OP_IS_NULL ? "false" : "true";
		snprintf(buf, sizeof buf, "%sz%d", op == CG_OP_IS_NULL ? "" : "!", c);
		return buf;
	}
	if (cg_op_is_column(op))
	{
		/* the columns, the operator and the scale factor are the plan's shape: all of them are written out */
		const char *ops[] = {"<", "<=", "==", ">=", ">", "!="};
		const char *o = ops[op - CG_OP_COL_LT];
		const KCmp &kc = atom_cmp(plan, arr, q);
		const std::string known = atom_known(plan, sh, c, op, arr, q);
		if (plan.isfloat[c]) snprintf(buf, sizeof buf, "%s(col_code_f(v%d) %s col_code_f(v%d))", known.c_str(), c, o, kc.col2);
		else if (kc.mul == 1) snprintf(buf, sizeof buf, "%s(v%d %s v%d)", known.c_str(), c, o, kc.col2);
		/* x op y * m  <=>  sign(x - y * m) op 0  <=>  0 op sign(y * m - x) */
		else if (kc.right) snprintf(buf, sizeof buf, "%s(0 %s cmp_scaled(v%d, %lldll, v%d))", known.c_str(), o, kc.col2, (long long) kc.mul, c);
		else snprintf(buf, sizeof buf, "%s(cmp_scaled(v%d, %lldll, v%d) %s 0)", known.c_str(), c, (long long) kc.mul, kc.col2, o);
		return buf;
	}
	if (col_nullable(sh, c)) snprintf(nn, sizeof nn, "!z%d && ", c);
	if (op_is_list(op))
	{
		const std::string h = found_var(prefix, q);
		if (op == CG_OP_IN) snprintf(buf, sizeof buf, "%s%s", nn, h.c_str());
		else snprintf(buf, sizeof buf, "%s!%s && !P.%sset[%d].nnull", nn, h.c_str(), arr, q);
		return buf;
	}
	if (plan.isfloat[c])
	{
		const char *ops[] = {"<", "<=", "==", ">=", ">", "!="};
		snprintf(buf, sizeof buf, "%s(fcmp(v%d, P.%sk[%d]) %s 0)", nn, c, arr, q, ops[op]);
	}
	else if (neg)
		snprintf(buf, sizeof buf, "%s!((v%d >= P.%slo[%d]) && (v%d <= P.%shi[%d]))", nn, c, arr, q, c, arr, q);
	else
		snprintf(buf, sizeof buf, "%s(v%d >= P.%slo[%d]) && (v%d <= P.%shi[%d])", nn, c, arr, q, c, arr, q);
	return buf;
}

/* the WHERE tree over the atoms t<q> (an AND-list without a tree) */
static std::string where_expr(const KPlan &plan)
{
	char buf[32];
	if (plan.nquals == 0) return "true";
	if (plan.nqexpr == 0)
	{
		std::string e;
		for (int q = 0; q < plan.nquals; q++) { snprintf(buf, sizeof buf, "%st%d", q ? " && " : "", q); e += buf; }
		return e;
	}
	return tree_expr(plan.nqexpr, plan.qexpr, "t");
}

/* The CASE argument of aggregate a as straight-line first-TRUE selection over the WHEN trees (pool atoms u<q>): defines
 * cn<a> = the value is NULL, and it<a> (integer) or ft<a> (float) -- and ov<a> for an overflow-checked term -- from the
 * chosen arm only, so an arm that was not chosen raises nothing.  The arms' structure (their number, WHEN trees, result
 * forms and factor columns) is the query shape; their constants stay kernel parameters, P.arms[i], except that a bare
 * column factor (0 + 1 * x) is written out, as term_expr does. */
static void gen_case(std::string &s, const KPlan &plan, const JitShape &sh, int a, const char *C)
{
	const KAgg &g = plan.aggs[a];
	const bool fl = g.is_float;
	addf(s, "%sbool cn%d = true;\n%s%s %ct%d = %s;\n", C, a, C, fl ? "double" : "int64_t", fl ? 'f' : 'i', a, fl ? "0.0" : "0");
	if (!fl && g.ovchk) addf(s, "%sbool ov%d = false;\n", C, a);
	bool has_else = false;
	for (int i = plan.cfirst[a]; i < plan.cfirst[a] + plan.cnarms[a]; i++)
	{
		const KArm &A = plan.arms[i];
		const bool first = i == plan.cfirst[a];
		if (A.nwhen == 0)
		{
			addf(s, "%s%s{", C, first ? "" : "else ");
			has_else = true;
		}
		else addf(s, "%s%sif (%s) {", C, first ? "" : "else ", tree_expr(A.nwhen, A.when, "u").c_str());
		if (A.form == CG_CASE_CONST)
		{
			if (fl) addf(s, " cn%d = false; ft%d = __longlong_as_double(P.arms[%d].a[0]);", a, a, i);
			else addf(s, " cn%d = false; it%d = P.arms[%d].a[0];", a, a, i);
		}
		else if (A.form == CG_CASE_PRODUCT)
		{
			std::string nul, e;
			bool seen[CG_KMAX_COLS] = {false};
			for (int f = 0; f < A.nfactors; f++)
			{
				const int c = A.pcol[f];
				if (col_nullable(sh, c) && !seen[c]) nul += (nul.empty() ? "(z" : " || z") + std::to_string(c);
				seen[c] = true;
				char buf[256];
				const bool bare = A.a[f] == 0 && (fl ? A.b[f] == 0x3ff0000000000000ll : A.b[f] == 1);
				if (fl)
				{
					if (bare) snprintf(buf, sizeof buf, "__longlong_as_double(v%d)", c);
					else snprintf(buf, sizeof buf, "(__longlong_as_double(P.arms[%d].a[%d]) + __longlong_as_double(P.arms[%d].b[%d]) * __longlong_as_double(v%d))",
								  i, f, i, f, c);
					e += (f ? " * " : "") + std::string(buf);
				}
				else if (g.ovchk)
				{
					if (bare) snprintf(buf, sizeof buf, "v%d", c);
					else snprintf(buf, sizeof buf, "add_ovf(P.arms[%d].a[%d], mul_ovf(P.arms[%d].b[%d], v%d, ov%d), ov%d)", i, f, i, f, c, a, a);
					e = f ? "mul_ovf(" + e + ", " + buf + ", ov" + std::to_string(a) + ")" : std::string(buf);
				}
				else
				{
					if (bare) snprintf(buf, sizeof buf, "v%d", c);
					else snprintf(buf, sizeof buf, "(P.arms[%d].a[%d] + P.arms[%d].b[%d] * v%d)", i, f, i, f, c);
					e += (f ? " * " : "") + std::string(buf);
				}
			}
			if (!nul.empty()) nul += ")";
			addf(s, " cn%d = %s; %ct%d = %s;", a, nul.empty() ? "false" : nul.c_str(), fl ? 'f' : 'i', a, e.c_str());
		}
		s += " }\n";
		if (has_else) break;
	}
}

/* updates of a group entry in global memory (`e` = its word pointer): the TABLE kind, and the NULL-key group of
 * the SMALL kind.  with_packed: count(*) and the packed sum share one reduction on P.packed[slot]. */
static void gen_table_updates(std::string &s, const KPlan &plan, const JitShape &sh, const char *C, bool with_packed,
							  const std::vector<std::string> &an, const std::vector<std::string> &w0)
{
	if (with_packed)
	{
		const int pa = sh.pack_agg;
		if (an[pa].empty())
			addf(s, "%sred_add(P.packed + slot, ((uint64_t) it%d << P.pack_shift) + 1ull);\n", C, pa);
		else
			addf(s, "%sred_add(P.packed + slot, (an%d ? 0ull : ((uint64_t) it%d << P.pack_shift)) + 1ull);\n%sif (an%d) red_add(e + %d, 1ull);\n",
				 C, pa, pa, C, pa, plan.aggs[pa].nullword);
		addf(s, "%sg_rows++;\n", C);
	}
	else
		addf(s, "%sred_add(e, 1ull);\n", C);
	for (int a = 0; a < plan.naggs; a++)
	{
		const KAgg &g = plan.aggs[a];
		if ((g.kind == CG_AGG_COUNT_STAR && an[a].empty()) || (with_packed && a == sh.pack_agg)) continue;
		if (!an[a].empty()) addf(s, "%sif (an%d) red_add(e + %d, 1ull);\n", C, a, g.nullword);
		if (!agg_has_value(g)) continue;
		if (agg_is_var(g))
		{
			/* sum(x^2): one reduction per limb, none for a zero limb above the first */
			std::string q = an[a].empty() ? "{" : ("if (!an" + std::to_string(a) + ") {");
			for (int l = 0; l < g.qlimbs; l++)
				q += (l ? " if (" + square_limb_expr(a, g.qlimbs, l) + ") " : std::string(" ")) + "red_add(e + " + std::to_string(g.qword + l) +
					 ", " + square_limb_expr(a, g.qlimbs, l) + ");";
			addf(s, "%s%s }\n", C, q.c_str());
		}
		char p[32];
		snprintf(p, sizeof p, "e + %d", g.word0);
		std::string guard = an[a].empty() ? "" : ("if (!an" + std::to_string(a) + ") ");
		const int op = plan.wordop[g.word0];
		if (op == CG_WORD_AND || op == CG_WORD_OR)
		{
			/* no reduction for the identity (bit_or of 0, bool_or FALSE, bool_and TRUE), as min / max skip theirs */
			guard = "if (" + (an[a].empty() ? std::string() : "!an" + std::to_string(a) + " && ") + w0[a] + " != " + op_identity(op) + ") ";
		}
		if (agg_two_limbs(g))
			addf(s, "%s%s{ %s red_add(e + %d, (uint64_t) (it%d >> 32)); }\n", C, guard.c_str(),
				 op_apply_global(plan.wordop[g.word0], p, w0[a]).c_str(), g.word0 + 1, a);
		else
			addf(s, "%s%s{ %s }\n", C, guard.c_str(), op_apply_global(plan.wordop[g.word0], p, w0[a]).c_str());
	}
}

/* the per-row block: extraction, WHERE tree, group slot, transition functions */
static void gen_row(std::string &s, const KPlan &plan, const JitShape &sh, int u, int j)
{
	const char *T = "\t\t\t\t\t\t";
	addf(s, "\t\t\t\t\tif (r + %d < rows) {\n", j);
	for (int c = 0; c < plan.ncols; c++)
	{
		addf(s, "%sconst int64_t v%d = %s;\n", T, c, col_value(plan, sh, c, u, j).c_str());
		if (col_nullable(sh, c)) addf(s, "%sconst bool z%d = !((e%d_%d >> %d) & 1u);\n", T, c, c, u, j);
	}
	/* list membership of the IN / NOT IN atoms (the lists stay kernel parameters: P.sets, P.qset / P.fset) */
	auto gen_found = [&](int n, const uint8_t *col, const uint8_t *op, const char *arr, const char *prefix) {
		for (int q = 0; q < n; q++)
			if (op_is_list(op[q]))
				addf(s, "%sconst bool %s = in_set(P.sets, P.%sset[%d], set_code_%c(v%d));\n", T, found_var(prefix, q).c_str(), arr, q,
					 plan.isfloat[col[q]] ? 'f' : 'i', col[q]);
	};
	/* K3: the WHERE tree; an atom on a NULL input is not TRUE (three-valued logic) */
	gen_found(plan.nquals, plan.qcol, plan.qop, "q", "t");
	for (int q = 0; q < plan.nquals; q++)
		addf(s, "%sconst bool t%d = %s;\n", T, q, atom_expr(plan, sh, plan.qcol[q], plan.qop[q], plan.qneg[q], "q", q, "t").c_str());
	/* aggregate FILTERs: atoms u<q> of their own pool, f<a> = aggregate a's tree is TRUE */
	gen_found(plan.nfquals, plan.fcol, plan.fop, "f", "u");
	for (int q = 0; q < plan.nfquals; q++)
		addf(s, "%sconst bool u%d = %s;\n", T, q, atom_expr(plan, sh, plan.fcol[q], plan.fop[q], plan.fneg[q], "f", q, "u").c_str());
	for (int a = 0; a < plan.naggs; a++)
		if (plan.nfexpr[a] > 0) addf(s, "%sconst bool f%d = %s;\n", T, a, tree_expr(plan.nfexpr[a], plan.fexpr[a], "u").c_str());
	/* bool_and / bool_or arguments, three-valued on two rails: uf<q> = atom q is FALSE (not NULL, not TRUE); at<a> = the
	 * argument is TRUE, af<a> = it is FALSE (the same tree with AND / OR swapped over the uf<q>); neither = UNKNOWN */
	if (plan_has_args(plan))
	{
		for (int q = 0; q < plan.nfquals; q++)
		{
			const int c = plan.fcol[q];
			const int op = plan.fop[q];
			std::string nn = col_nullable(sh, c) ? "!z" + std::to_string(c) + " && " : std::string();
			if (op == CG_OP_IS_NULL || op == CG_OP_IS_NOT_NULL) addf(s, "%sconst bool uf%d = !u%d;\n", T, q, q);     /* never UNKNOWN */
			else if (op == CG_OP_IN) addf(s, "%sconst bool uf%d = %s!%s && !P.fset[%d].nnull;\n", T, q, nn.c_str(), found_var("u", q).c_str(), q);
			else if (op == CG_OP_NOT_IN) addf(s, "%sconst bool uf%d = %s%s;\n", T, q, nn.c_str(), found_var("u", q).c_str());
			else if (cg_op_is_column(op)) addf(s, "%sconst bool uf%d = %s!u%d;\n", T, q, atom_known(plan, sh, c, op, "f", q).c_str(), q);
			else if (col_nullable(sh, c)) addf(s, "%sconst bool uf%d = !z%d && !u%d;\n", T, q, c, q);
			else addf(s, "%sconst bool uf%d = !u%d;\n", T, q, q);
		}
		for (int a = 0; a < plan.naggs; a++)
			if (plan.nargexpr[a] > 0)
				addf(s, "%sconst bool at%d = %s;\n%sconst bool af%d = %s;\n", T, a, tree_expr(plan.nargexpr[a], plan.argexpr[a], "u").c_str(), T, a,
					 tree_expr(plan.nargexpr[a], plan.argexpr[a], "uf", true).c_str());
	}
	addf(s, "%sconst bool pass = %s;\n", T, where_expr(plan).c_str());
	addf(s, "%sif (!pass) removed++;\n%selse {\n", T, T);
	const char *B = "\t\t\t\t\t\t\t";
	/* group slot; a NULL key is its own group (the entry behind the addressable ones) */
	std::string zkey;
	if (plan.composite)
	{
		/* the composite code (cg_plan.cpp): a NULL is digit 0, so there is no NULL group; kok = every value within its
		 * column's bounds */
		std::string code, ok;
		for (int g = 0; g < plan.ngroup; g++)
		{
			const int c = plan.gcol[g];
			addf(s, "%sconst uint64_t kd%d = (uint64_t) v%d - (uint64_t) P.kmin[%d];\n", B, g, c, g);
			char digit[64], in[96];
			if (col_nullable(sh, c))
			{
				snprintf(digit, sizeof digit, "(z%d ? 0ull : kd%d + 1ull)", c, g);
				snprintf(in, sizeof in, "(z%d || kd%d < P.kradix[%d] - 1ull)", c, g, g);
			}
			else
			{
				snprintf(digit, sizeof digit, "(kd%d + 1ull)", g);
				snprintf(in, sizeof in, "kd%d < P.kradix[%d] - 1ull", g, g);
			}
			code = g ? "(" + code + ") * P.kradix[" + std::to_string(g) + "] + " + digit : std::string(digit);
			ok += (g ? " && " : "") + std::string(in);
		}
		addf(s, "%sconst bool kok = %s;\n%sconst uint64_t kcode = %s;\n", B, ok.c_str(), B, code.c_str());
	}
	else if (plan.mode != CG_MODE_GLOBAL)
	{
		if (plan.ngroup == 1) { if (col_nullable(sh, plan.gcol[0])) zkey = "z" + std::to_string(plan.gcol[0]); }
		else
		{
			if (col_nullable(sh, plan.gcol[0])) zkey = "z" + std::to_string(plan.gcol[0]);
			if (col_nullable(sh, plan.gcol[1])) zkey += (zkey.empty() ? "z" : " || z") + std::to_string(plan.gcol[1]);
		}
	}
	if (plan.mode == CG_MODE_DENSE && plan.composite)
		addf(s, "%suint64_t slot = kcode;\n%sbool ok = kok;\n%sif (!ok) raise_flag(P.stats, %lluull);\n", B, B, B,
			 (unsigned long long) CG_ERRFLAG_KEY_RANGE);
	else if (plan.mode == CG_MODE_HASH && plan.composite)
		/* a code is never EMPTY_KEY (it is >= 0) */
		addf(s,
			 "%sconst int64_t key = (int64_t) kcode;\n%suint64_t slot;\n"
			 "%sif (!kok) { raise_flag(P.stats, %lluull); slot = ~0ull; }\n"
			 "%selse { uint64_t h = ((uint64_t) key * 0x9E3779B97F4A7C15ull) >> P.hash_shift;\n"
			 "%s  long long cur = (long long) __ldcg((unsigned long long *) (P.hkeys + h));\n"
			 "%s  slot = (cur == key) ? h : hash_slot_slow(P, key, h); }\n"
			 "%sbool ok = slot != ~0ull;\n",
			 B, B, B, (unsigned long long) CG_ERRFLAG_KEY_RANGE, B, B, B, B);
	else if (plan.mode == CG_MODE_DENSE)
	{
		if (plan.ngroup == 1)
		{
			if (zkey.empty())
				addf(s, "%suint64_t slot = (uint64_t) v%d - (uint64_t) P.key_min;\n%sbool ok = slot < P.capacity;\n", B, plan.gcol[0], B);
			else
				addf(s, "%suint64_t slot = %s ? P.capacity : (uint64_t) v%d - (uint64_t) P.key_min;\n%sbool ok = %s || slot < P.capacity;\n", B,
					 zkey.c_str(), plan.gcol[0], B, zkey.c_str());
			addf(s, "%sif (!ok) raise_flag(P.stats, %lluull);\n", B, (unsigned long long) CG_ERRFLAG_KEY_RANGE);
		}
		else
		{
			addf(s,
				 "%sconst uint64_t ka = (uint64_t) (int64_t) (int32_t) v%d - (uint64_t) P.key_min, kb = (uint64_t) (int64_t) (int32_t) v%d - (uint64_t) P.key_min1;\n"
				 "%suint64_t slot = ka * P.range1 + kb;\n%sbool ok = kb < P.range1 && slot < P.capacity;\n",
				 B, plan.gcol[0], plan.gcol[1], B, B);
			if (zkey.empty())
				addf(s, "%sif (!ok) raise_flag(P.stats, %lluull);\n", B, (unsigned long long) CG_ERRFLAG_KEY_RANGE);
			else
				addf(s, "%sif (%s) { raise_flag(P.stats, %lluull); ok = false; }\n%selse if (!ok) raise_flag(P.stats, %lluull);\n", B, zkey.c_str(),
					 (unsigned long long) CG_ERRFLAG_NULL_MULTIKEY, B, (unsigned long long) CG_ERRFLAG_KEY_RANGE);
		}
	}
	else if (plan.mode == CG_MODE_HASH)
	{
		if (plan.ngroup == 1) addf(s, "%sconst int64_t key = v%d;\n", B, plan.gcol[0]);
		else addf(s, "%sconst int64_t key = (int64_t) ((uint64_t) (uint32_t) v%d | ((uint64_t) (uint32_t) v%d << 32));\n", B, plan.gcol[0], plan.gcol[1]);
		addf(s, "%suint64_t slot;\n", B);
		if (!zkey.empty())
		{
			if (plan.ngroup == 1) addf(s, "%sif (%s) slot = P.capacity;\n%selse ", B, zkey.c_str(), B);
			else addf(s, "%sif (%s) { raise_flag(P.stats, %lluull); slot = ~0ull; }\n%selse ", B, zkey.c_str(),
					  (unsigned long long) CG_ERRFLAG_NULL_MULTIKEY, B);
		}
		else s += B;
		addf(s,
			 "if (key == EMPTY_KEY) slot = P.capacity + 1;\n"
			 "%selse { uint64_t h = ((uint64_t) key * 0x9E3779B97F4A7C15ull) >> P.hash_shift;\n"
			 "%s  long long cur = (long long) __ldcg((unsigned long long *) (P.hkeys + h));\n"
			 "%s  slot = (cur == key) ? h : hash_slot_slow(P, key, h); }\n"
			 "%sbool ok = slot != ~0ull;\n", B, B, B, B);
	}
	else
		addf(s, "%sconst bool ok = true;\n", B);
	addf(s, "%sif (ok) {\n", B);
	const char *C = "\t\t\t\t\t\t\t\t";
	/* no-input flags (NULL input, or FILTER not TRUE) and terms; a rejected row raises no error of its term */
	std::vector<std::string> an(plan.naggs), w0v(plan.naggs);
	for (int a = 0; a < plan.naggs; a++)
	{
		const KAgg &g = plan.aggs[a];
		if (plan.cnarms[a] > 0) gen_case(s, plan, sh, a, C);
		an[a] = agg_noinput_expr(plan, a, sh);
		if (!an[a].empty()) addf(s, "%sconst bool an%d = %s;\n", C, a, an[a].c_str());
		if (!agg_has_value(g)) continue;
		if (g.barg)
		{
			/* bool_and / bool_or: TRUE = all ones (the identity of AND), FALSE = 0 (that of OR) */
			w0v[a] = "(at" + std::to_string(a) + " ? 0xffffffffffffffffull : 0ull)";
			continue;
		}
		const bool cs = plan.cnarms[a] > 0;     /* gen_case defined the term */
		std::string e = cs ? std::string() : term_expr(g, a);
		if (g.is_float) { if (!cs) addf(s, "%sconst double ft%d = %s;\n", C, a, e.c_str()); }
		else
		{
			if (g.ovchk && !cs) addf(s, "%sbool ov%d = false;\n", C, a);
			if (!cs) addf(s, "%sconst int64_t it%d = %s;\n", C, a, e.c_str());
			if (g.ovchk)
				addf(s, "%sif (%sov%d) raise_flag(P.stats, %lluull);\n", C, an[a].empty() ? "" : ("!an" + std::to_string(a) + " && ").c_str(),
					 a, (unsigned long long) CG_ERRFLAG_TERM_OVERFLOW);
			if ((g.kind == CG_AGG_SUM && g.nlimbs == 1) || (agg_is_var(g) && g.bound > 0))
				addf(s, "%sif (%s(it%d > P.aggs[%d].bound || it%d < -P.aggs[%d].bound)) raise_flag(P.stats, %lluull);\n", C,
					 an[a].empty() ? "" : ("!an" + std::to_string(a) + " && ").c_str(), a, a, a, a, (unsigned long long) CG_ERRFLAG_SUM_BOUND);
			if (agg_is_var(g))
				/* x^2 = qh:ql from |x| (x = INT64_MIN gives 2^126) */
				addf(s, "%sconst uint64_t qa%d = it%d < 0 ? 0ull - (uint64_t) it%d : (uint64_t) it%d;\n"
						"%sconst uint64_t ql%d = qa%d * qa%d, qh%d = __umul64hi(qa%d, qa%d);\n",
					 C, a, a, a, a, C, a, a, a, a, a, a);
		}
		/* the word-0 value the aggregate contributes */
		char buf[128];
		if (g.kind == CG_AGG_SUM || agg_is_var(g))
		{
			if (g.is_float) snprintf(buf, sizeof buf, "(uint64_t) __double_as_longlong(ft%d)", a);
			else if (g.nlimbs == 1) snprintf(buf, sizeof buf, "(uint64_t) it%d", a);
			else snprintf(buf, sizeof buf, "(uint64_t) (uint32_t) it%d", a);
		}
		else if (g.is_float) snprintf(buf, sizeof buf, "f8_ordered(__double_as_longlong(ft%d))", a);
		else snprintf(buf, sizeof buf, "(uint64_t) it%d", a);
		w0v[a] = buf;
	}
	if (sh.kind == JK_GLOBAL)
	{
		addf(s, "%sg_rows++;\n", C);
		for (int a = 0; a < plan.naggs; a++)
		{
			const KAgg &g = plan.aggs[a];
			if (!an[a].empty()) addf(s, "%sif (an%d) g_n%d++;\n", C, a, a);
			if (!agg_has_value(g)) continue;
			char acc[32];
			snprintf(acc, sizeof acc, "g_a%d_0", a);
			std::string guard = an[a].empty() ? "" : ("if (!an" + std::to_string(a) + ") ");
			if (agg_two_limbs(g))
				addf(s, "%s%s{ %s = %s; g_a%d_1 += (uint64_t) (it%d >> 32); }\n", C, guard.c_str(), acc,
					 op_combine(plan.wordop[g.word0], acc, w0v[a]).c_str(), a, a);
			else
				addf(s, "%s%s%s = %s;\n", C, guard.c_str(), acc, op_combine(plan.wordop[g.word0], acc, w0v[a]).c_str());
			if (agg_is_var(g))
			{
				std::string q = guard + "{";
				for (int l = 0; l < g.qlimbs; l++) q += " g_q" + std::to_string(a) + "_" + std::to_string(l) + " += " + square_limb_expr(a, g.qlimbs, l) + ";";
				addf(s, "%s%s }\n", C, q.c_str());
			}
		}
	}
	else if (sh.kind == JK_SMALL)
	{
		const char *D = C;
		std::string inner = C;
		if (!zkey.empty())
		{
			/* the NULL group has no shared-memory cells: (rare) global reductions on its table entry */
			addf(s, "%sif (%s) {\n%s\tuint64_t *e = P.table + P.capacity * %dull;\n", C, zkey.c_str(), C, plan.stride);
			std::string CC = std::string(C) + "\t";
			gen_table_updates(s, plan, sh, CC.c_str(), false, an, w0v);
			addf(s, "%s} else {\n", C);
			inner += "\t";
			D = inner.c_str();
		}
		addf(s, "%suint64_t *e = mine + (uint32_t) slot * %du;\n", D, sh.nhot * JIT_THREADS);
		/* one update per cell: the contributions of the (at most two) aggregates that share it are added together */
		std::vector<std::string> cellexpr(sh.nhot);
		cellexpr[0] = "1ull";
		for (int a = 0; a < plan.naggs; a++)
		{
			const KAgg &g = plan.aggs[a];
			/* a filtered aggregate's no-input counter has a cell; the NULL-input counters of the others stay on global
			 * reductions (rare) */
			if (sh.ncell[a] >= 0)
			{
				std::string &ce = cellexpr[sh.ncell[a]];
				ce = ce.empty() ? "(uint64_t) an" + std::to_string(a) : ce + " + (uint64_t) an" + std::to_string(a);
			}
			else if (!an[a].empty()) addf(s, "%sif (an%d) red_add(P.table + slot * %dull + %d, 1ull);\n", D, a, plan.stride, g.nullword);
			if (!agg_has_value(g)) continue;
			if (sh.half[a] >= 0)
			{
				char buf[160];
				if (sh.half[a] == 1) snprintf(buf, sizeof buf, "((uint64_t) it%d << 32)", a);
				else snprintf(buf, sizeof buf, "(uint64_t) (uint32_t) (it%d + %lldll)", a, (long long) sh.bias[a]);
				std::string term = an[a].empty() ? std::string(buf) : ("(an" + std::to_string(a) + " ? 0ull : " + buf + ")");
				std::string &ce = cellexpr[sh.hot0[a]];
				ce = ce.empty() ? term : (ce + " + " + term);
				continue;
			}
			char cell[48];
			snprintf(cell, sizeof cell, "e[%d]", sh.hot0[a] * JIT_THREADS);
			std::string guard = an[a].empty() ? "" : ("if (!an" + std::to_string(a) + ") ");
			if ((g.kind == CG_AGG_SUM || agg_is_var(g)) && !g.is_float)
			{
				if (sh.lane1[a]) addf(s, "%s%s%s += (uint64_t) it%d;\n", D, guard.c_str(), cell, a);
				else
					addf(s, "%s%s{ %s += (uint64_t) (uint32_t) it%d; e[%d] += (uint64_t) (it%d >> 32); }\n", D, guard.c_str(), cell, a,
						 (sh.hot0[a] + 1) * JIT_THREADS, a);
			}
			else
				addf(s, "%s%s%s = %s;\n", D, guard.c_str(), cell, op_combine(plan.wordop[g.word0], cell, w0v[a]).c_str());
			if (agg_is_var(g))
			{
				std::string q = guard + "{";
				for (int l = 0; l < g.qlimbs; l++)
					q += " e[" + std::to_string((sh.qcell[a] + l) * JIT_THREADS) + "] += " + square_limb_expr(a, g.qlimbs, l) + ";";
				addf(s, "%s%s }\n", D, q.c_str());
			}
		}
		for (int k = 0; k < sh.nhot; k++)
			if (!cellexpr[k].empty()) addf(s, "%se[%d] += %s;\n", D, k * JIT_THREADS, cellexpr[k].c_str());
		if (!zkey.empty()) addf(s, "%s}\n", C);
	}
	else
	{
		addf(s, "%suint64_t *e = P.table + slot * %dull;\n", C, plan.stride);
		gen_table_updates(s, plan, sh, C, sh.packed, an, w0v);
	}
	addf(s, "%s}\n%s}\n\t\t\t\t\t}\n", B, T);
}

/* the generated kernel's signature and the opening brace of its body */
#define JIT_ENTRY "cg_jit_scan(const __grid_constant__ KPlan P)\n{\n"

static std::string gen_source(const KPlan &plan, const JitShape &sh)
{
	std::string s;
	s.reserve(32768);
	gen_prelude(s, plan);
	if (sh.min_blocks > 0)
		addf(s, "extern \"C\" __global__ void __launch_bounds__(%d, %d) %s", JIT_THREADS, sh.min_blocks, JIT_ENTRY);
	else
		addf(s, "extern \"C\" __global__ void __launch_bounds__(%d) %s", JIT_THREADS, JIT_ENTRY);
	s += "\tconst uint32_t tid = threadIdx.x;\n\tuint32_t removed = 0;\n\tunsigned long long scanned = 0;\n\tuint64_t g_rows = 0;\n";
	if (sh.kind == JK_GLOBAL)
		for (int a = 0; a < plan.naggs; a++)
		{
			const KAgg &g = plan.aggs[a];
			if (!agg_noinput_expr(plan, a, sh).empty()) addf(s, "\tuint64_t g_n%d = 0;\n", a);
			if (!agg_has_value(g)) continue;
			addf(s, "\tuint64_t g_a%d_0 = %s, g_a%d_1 = 0;\n", a, op_identity(plan.wordop[g.word0]), a);
			for (int l = 0; agg_is_var(g) && l < g.qlimbs; l++) addf(s, "\tuint64_t g_q%d_%d = 0;\n", a, l);
		}
	if (sh.kind == JK_SMALL || sh.nullable)
		s += "\textern __shared__ uint64_t s_acc[];\n";
	if (sh.kind != JK_SMALL && sh.nullable)
		s += "\tuint64_t *s_nb = s_acc;\n";
	if (sh.kind == JK_SMALL)
	{
		addf(s, "\tconst uint32_t cells = (uint32_t) P.capacity * %du;\n", sh.nhot);
		if (sh.nullable) addf(s, "\tuint64_t *s_nb = s_acc + (size_t) cells * %d;\n", JIT_THREADS);
		addf(s, "\tfor (uint32_t i = 0; i < cells; i++) {\n\t\tuint64_t id = 0ull;\n\t\tswitch (i %% %du) {\n", sh.nhot);
		for (int a = 0; a < plan.naggs; a++)
		{
			const KAgg &g = plan.aggs[a];
			if (!agg_has_value(g)) continue;
			if (strcmp(op_identity(plan.wordop[g.word0]), "0ull") != 0)
				addf(s, "\t\t\tcase %d: id = %s; break;\n", sh.hot0[a], op_identity(plan.wordop[g.word0]));
		}
		addf(s, "\t\t\tdefault: break;\n\t\t}\n\t\ts_acc[(size_t) i * %d + tid] = id;\n\t}\n\tuint64_t *mine = s_acc + tid;\n", JIT_THREADS);
	}
	if (sh.nullable)
	{
		/* exists bitmap words and rank directory entries of the unit's rows are staged in shared memory once per unit: the
		 * per-row lookups then cost shared-memory latency and the value loads depend on nothing in global memory */
		int nn = 0;
		for (int c = 0; c < plan.ncols; c++) if (col_nullable(sh, c)) nn++;
		s += "\tconst uint32_t NW = P.max_cg_rows / 64u + 2u;\n";
		int ni = 0;
		for (int c = 0; c < plan.ncols; c++)
			if (col_nullable(sh, c))
			{
				addf(s, "\tuint64_t *sb%d = s_nb + %du * NW;\n\tuint32_t *sk%d = (uint32_t *) (s_nb + %du * NW) + %du * NW;\n", c, ni, c, nn, ni);
				ni++;
			}
	}
	/* work unit = (chunk group, row range [row0, rows)): launches with few chunk groups cut them into slices */
	s += "\tconst uint32_t nunits = P.nselected * (uint32_t) P.slices;\n"
		 "\tfor (uint32_t unit = blockIdx.x; unit < nunits; unit += gridDim.x)\n\t{\n"
		 "\t\tconst uint32_t ci = P.slices == 1 ? unit : unit / (uint32_t) P.slices;\n"
		 "\t\tconst uint32_t sl = P.slices == 1 ? 0u : unit - ci * (uint32_t) P.slices;\n";
	addf(s, "\t\tconst DevChunkCol *cc = P.chunkcols + (uint64_t) P.selected[ci] * %dull;\n", plan.nstaged);
	s += "\t\tconst uint32_t chunk_rows = __ldg(&cc[0].row_count);\n"
		 "\t\tconst uint32_t row0 = sl * P.slice_rows;\n"
		 "\t\tconst uint32_t rows = min(chunk_rows, row0 + P.slice_rows);\n";
	for (int c = 0; c < plan.ncols; c++)
	{
		addf(s, "\t\tconst uint8_t *p%d = P.arena + __ldg(&cc[%d].values_off);\n", c, plan.slot[c]);
		if (col_nullable(sh, c))
			addf(s, "\t\tconst uint64_t *b%d = (const uint64_t *) (P.arena + __ldg(&cc[%d].exists_off));\n"
					"\t\tconst uint32_t *k%d = (const uint32_t *) (P.arena + __ldg(&cc[%d].rank_off));\n"
					"\t\tconst bool n%d = __ldg(&cc[%d].value_count) != chunk_rows;\n",
				 c, plan.slot[c], c, plan.slot[c], c, plan.slot[c]);
	}
	if (sh.nullable)
	{
		s += "\t\tconst uint32_t wfirst = row0 >> 6, wcount = rows > row0 ? ((rows + 63u) >> 6) - wfirst : 0u;\n\t\t__syncthreads();\n";
		for (int c = 0; c < plan.ncols; c++)
			if (col_nullable(sh, c))
				addf(s, "\t\tif (n%d) for (uint32_t i = tid; i < wcount; i += %du) { sb%d[i] = b%d[wfirst + i]; sk%d[i] = k%d[wfirst + i]; }\n", c,
					 JIT_THREADS, c, c, c, c);
		s += "\t\t__syncthreads();\n";
	}
	s += "\t\tscanned += (tid == 0 && sl == 0) ? chunk_rows : 0;\n";
	if (plan.ncols == 0)
	{
		/* count(*) without any column */
		s += "\t\tif (tid == 0 && sl == 0) g_rows += chunk_rows;\n\t}\n";
	}
	else
	{
		addf(s, "\t\tfor (uint32_t base = row0; base < rows; base += %du)\n\t\t{\n", JIT_THREADS * sh.R * sh.U);
		for (int u = 0; u < sh.U; u++)
			for (int c = 0; c < plan.ncols; c++)
			{
				if (col_nullable(sh, c))
				{
					s += "\t\t\tuint64_t ";
					for (int k = 0; k < sh.R; k++) addf(s, "%sx%d_%d_%d = 0", k ? ", " : "", c, u, k);
					addf(s, "; uint32_t e%d_%d = 0;\n", c, u);
					continue;
				}
				int nw = sh.R * plan.len[c] / 8;
				if (nw < 1) nw = 1;
				s += "\t\t\tuint64_t ";
				for (int k = 0; k < nw; k++) addf(s, "%sw%d_%d_%d = 0", k ? ", " : "", c, u, k);
				s += ";\n";
			}
		for (int u = 0; u < sh.U; u++)
		{
			addf(s, "\t\t\t{\n\t\t\t\tconst uint32_t r = base + (%du + tid) * %du;\n\t\t\t\tif (r < rows) {\n", u * JIT_THREADS, sh.R);
			gen_loads(s, plan, sh, u);
			s += "\t\t\t\t}\n\t\t\t}\n";
		}
		for (int u = 0; u < sh.U; u++)
		{
			addf(s, "\t\t\t{\n\t\t\t\tconst uint32_t r = base + (%du + tid) * %du;\n\t\t\t\tif (r < rows) {\n", u * JIT_THREADS, sh.R);
			for (int j = 0; j < sh.R; j++) gen_row(s, plan, sh, u, j);
			s += "\t\t\t\t}\n\t\t\t}\n";
		}
		s += "\t\t}\n\t}\n";
	}
	/* epilogue */
	s += "\tunsigned long long rem = wsum(removed), scn = wsum(scanned);\n"
		 "\tif ((tid & 31) == 0) { if (scn) atomicAdd(P.stats + 0, scn); if (rem) atomicAdd(P.stats + 1, rem); }\n";
	if (sh.kind == JK_TABLE && sh.packed)
		addf(s, "\t{ uint64_t added = wsum(g_rows); if ((tid & 31) == 0 && added) atomicAdd(P.stats + %d, (unsigned long long) added); }\n",
			 CG_STAT_PACKED_ADDED);
	if (sh.kind == JK_GLOBAL)
	{
		s += "\t{ uint64_t n = wsum(g_rows); if ((tid & 31) == 0 && n) red_add(P.table, n); }\n";
		for (int a = 0; a < plan.naggs; a++)
		{
			const KAgg &g = plan.aggs[a];
			if (!agg_noinput_expr(plan, a, sh).empty())
				addf(s, "\t{ uint64_t n = wsum(g_n%d); if ((tid & 31) == 0 && n) red_add(P.table + %d, n); }\n", a, g.nullword);
			if (!agg_has_value(g)) continue;
			int op = plan.wordop[g.word0];
			if (op == CG_WORD_AND || op == CG_WORD_OR)
			{
				/* one redux.sync per 32-bit half instead of five shuffle rounds */
				const char *rd = op == CG_WORD_AND ? "__reduce_and_sync" : "__reduce_or_sync";
				addf(s, "\t{ uint64_t x = g_a%d_0;\n\t  x = ((uint64_t) %s(0xffffffffu, (uint32_t) (x >> 32)) << 32) | (uint64_t) %s(0xffffffffu, (uint32_t) x);\n",
					 a, rd, rd);
			}
			else
				addf(s, "\t{ uint64_t x = g_a%d_0;\n\t  for (int o = 16; o > 0; o >>= 1) { uint64_t y = __shfl_xor_sync(0xffffffffu, x, o); x = %s; }\n", a,
					 op_combine(op, "x", "y").c_str());
			char p[48];
			snprintf(p, sizeof p, "P.table + %d", g.word0);
			addf(s, "\t  if ((tid & 31) == 0 && x != %s) { %s }\n", op_identity(op), op_apply_global(op, p, "x").c_str());
			if (agg_two_limbs(g))
				addf(s, "\t  uint64_t x1 = wsum(g_a%d_1); if ((tid & 31) == 0 && x1) red_add(P.table + %d, x1);\n", a, g.word0 + 1);
			for (int l = 0; agg_is_var(g) && l < g.qlimbs; l++)
				addf(s, "\t  { uint64_t q = wsum(g_q%d_%d); if ((tid & 31) == 0 && q) red_add(P.table + %d, q); }\n", a, l, g.qword + l);
			s += "\t}\n";
		}
	}
	if (sh.kind == JK_SMALL)
	{
		/* flush: combine the 256 lanes of every cell, one global atomic per touched word of this CTA */
		addf(s, "\t__syncthreads();\n\tfor (uint32_t i = tid; i < cells; i += %d) {\n\t\tconst uint64_t *col = s_acc + (size_t) i * %d;\n"
				"\t\tuint64_t *ge = P.table + (uint64_t) (i / %du) * %dull;\n\t\tswitch (i %% %du) {\n",
			 JIT_THREADS, JIT_THREADS, sh.nhot, plan.stride, sh.nhot);
		/* emits the statements that add the exact lane total `S` (int64_t) of aggregate a to the group's table words */
		auto add_total = [&](int a) -> std::string {
			const KAgg &g = plan.aggs[a];
			char b[256];
			if (g.nlimbs == 2)
				snprintf(b, sizeof b, "{ const uint64_t l_ = (uint64_t) (uint32_t) S, h_ = (uint64_t) (S >> 32); if (l_) red_add(ge + %d, l_); if (h_) red_add(ge + %d, h_); }",
						 g.word0, g.word0 + 1);
			else
				snprintf(b, sizeof b, "{ if (S) red_add(ge + %d, (uint64_t) S); }", g.word0);
			return b;
		};
		if (sh.rows_partner < 0)
			addf(s, "\t\t\tcase 0: { uint64_t x = 0; for (uint32_t k = 0; k < %d; k++) x += col[(k + tid) %% %d]; if (x) red_add(ge, x); break; }\n",
				 JIT_THREADS, JIT_THREADS);
		else
			addf(s, "\t\t\tcase 0: { uint64_t r_ = 0; int64_t S = 0; for (uint32_t k = 0; k < %d; k++) { const uint64_t x = col[(k + tid) %% %d]; r_ += (uint32_t) x; S += (int64_t) (int32_t) (uint32_t) (x >> 32); }\n"
					"\t\t\t\tif (r_) red_add(ge, r_); %s break; }\n",
				 JIT_THREADS, JIT_THREADS, add_total(sh.rows_partner).c_str());
		/* paired cells: low half = sum(term + bias) of aggregate x over the group's rows of a lane, high half = aggregate y */
		for (int cell = 1; cell < sh.nhot; cell++)
		{
			int x = -1, y = -1;
			for (int a = 0; a < plan.naggs; a++)
				if (sh.hot0[a] == cell && sh.half[a] == 0) x = a; else if (sh.hot0[a] == cell && sh.half[a] == 1) y = a;
			if (x < 0 || y < 0) continue;
			addf(s, "\t\t\tcase %d: { uint64_t lo_ = 0, r_ = 0; int64_t hi_ = 0; const uint64_t *rows_ = s_acc + (size_t) (i - %d) * %d;\n"
					"\t\t\t\tfor (uint32_t k = 0; k < %d; k++) { const uint64_t v_ = col[(k + tid) %% %d]; lo_ += (uint32_t) v_; hi_ += (int64_t) (int32_t) (uint32_t) (v_ >> 32); r_ += (uint32_t) rows_[(k + tid) %% %d]; }\n"
					"\t\t\t\t{ const int64_t S = (int64_t) lo_ - (int64_t) r_ * %lldll; %s }\n"
					"\t\t\t\t{ const int64_t S = hi_; %s } break; }\n",
				 cell, cell, JIT_THREADS, JIT_THREADS, JIT_THREADS, JIT_THREADS, (long long) sh.bias[x], add_total(x).c_str(), add_total(y).c_str());
		}
		for (int a = 0; a < plan.naggs; a++)
		{
			const KAgg &g = plan.aggs[a];
			if (sh.ncell[a] >= 0)
				addf(s, "\t\t\tcase %d: { uint64_t x = 0; for (uint32_t k = 0; k < %d; k++) x += col[(k + tid) %% %d]; if (x) red_add(ge + %d, x); break; }\n",
					 sh.ncell[a], JIT_THREADS, JIT_THREADS, g.nullword);
			if (!agg_has_value(g) || sh.half[a] >= 0) continue;
			int op = plan.wordop[g.word0];
			char p[32];
			snprintf(p, sizeof p, "ge + %d", g.word0);
			for (int l = 0; agg_is_var(g) && l < g.qlimbs; l++)
				addf(s, "\t\t\tcase %d: { uint64_t x = 0; for (uint32_t k = 0; k < %d; k++) x += col[(k + tid) %% %d]; if (x) red_add(ge + %d, x); break; }\n",
					 sh.qcell[a] + l, JIT_THREADS, JIT_THREADS, g.qword + l);
			if ((g.kind == CG_AGG_SUM || agg_is_var(g)) && !g.is_float)
			{
				if (sh.lane1[a] && g.nlimbs == 2)
					/* exact 64-bit lane sums -> the table's (low 32 unsigned, high signed) limbs */
					addf(s,
						 "\t\t\tcase %d: { uint64_t lo = 0, hi = 0; for (uint32_t k = 0; k < %d; k++) { int64_t x = (int64_t) col[(k + tid) %% %d]; lo += (uint64_t) (uint32_t) x; hi += (uint64_t) (x >> 32); }\n"
						 "\t\t\t\tif (lo) red_add(ge + %d, lo); if (hi) red_add(ge + %d, hi); break; }\n",
						 sh.hot0[a], JIT_THREADS, JIT_THREADS, g.word0, g.word0 + 1);
				else
				{
					addf(s, "\t\t\tcase %d: { uint64_t x = 0; for (uint32_t k = 0; k < %d; k++) x += col[(k + tid) %% %d]; if (x) red_add(ge + %d, x); break; }\n",
						 sh.hot0[a], JIT_THREADS, JIT_THREADS, g.word0);
					if (!sh.lane1[a])
						addf(s, "\t\t\tcase %d: { uint64_t x = 0; for (uint32_t k = 0; k < %d; k++) x += col[(k + tid) %% %d]; if (x) red_add(ge + %d, x); break; }\n",
							 sh.hot0[a] + 1, JIT_THREADS, JIT_THREADS, g.word0 + 1);
				}
			}
			else
				addf(s,
					 "\t\t\tcase %d: { uint64_t x = %s; for (uint32_t k = 0; k < %d; k++) { uint64_t y = col[(k + tid) %% %d]; x = %s; }\n"
					 "\t\t\t\tif (x != %s) { %s } break; }\n",
					 sh.hot0[a], op_identity(op), JIT_THREADS, JIT_THREADS, op_combine(op, "x", "y").c_str(), op_identity(op),
					 op_apply_global(op, p, "x").c_str());
		}
		s += "\t\t\tdefault: break;\n\t\t}\n\t}\n";
	}
	s += "}\n";
	return s;
}

/* ------------------------------------------------------------------------------ *
 *  Compilation cache and launch.
 * ------------------------------------------------------------------------------ */
struct JitKernel
{
	std::string cubin;
	CUfunction fn = nullptr;
	int occupancy = 0;
	size_t smem_configured = 0;
	bool failed = false;
};

static std::map<std::string, JitKernel> g_cache;
static std::mutex g_cache_mutex;
static unsigned long long g_jit_compiles = 0, g_jit_launches = 0;

/* compiles a plan's generated source as it is launched: the kernel's first statement lets the next scan launch of a
 * chain start as soon as every CTA of this one runs (cg_chain_scan, cg_host.cpp) */
static int compile_source(const std::string &plan_src, std::string *cubin)
{
	if (!load_rtc()) return cg_set_error(CG_EUNSUPPORTED, "libnvrtc is not available");
	const size_t body = plan_src.find(JIT_ENTRY);
	if (body == std::string::npos) return cg_set_error(CG_EINVAL, "generated source without the kernel entry");
	const size_t at = body + strlen(JIT_ENTRY);
	const std::string src = plan_src.substr(0, at) + "\tasm volatile(\"griddepcontrol.launch_dependents;\" ::: \"memory\");\n" + plan_src.substr(at);
	nvrtcProgram prog = nullptr;
	if (g_api.create(&prog, src.c_str(), "cg_jit_scan.cu", 0, nullptr, nullptr) != 0)
		return cg_set_error(CG_ECUDA, "nvrtcCreateProgram failed");
	const char *opts[] = {"--gpu-architecture=sm_90a", "-lineinfo", "--std=c++17"};
	int rc = g_api.compile(prog, 3, opts);
	if (rc != 0)
	{
		size_t n = 0;
		g_api.log_size(prog, &n);
		std::string log(n + 1, '\0');
		if (n) g_api.log(prog, &log[0]);
		g_api.destroy(&prog);
		if (getenv("CG_JIT_DUMP")) fprintf(stderr, "%s\n", src.c_str());
		return cg_set_error(CG_ECUDA, "nvrtc: %.400s", log.c_str());
	}
	size_t n = 0;
	g_api.cubin_size(prog, &n);
	cubin->assign(n, '\0');
	g_api.cubin(prog, &(*cubin)[0]);
	g_api.destroy(&prog);
	g_jit_compiles++;
	return CG_OK;
}

/* source of the kernel a plan would get (tests, EXPLAIN-style inspection) */
int cg_jit_source_for(const KPlan &plan, uint32_t nullable, std::string *src, int *kind)
{
	JitShape sh;
	choose_shape(plan, nullable, &sh);
	*src = gen_source(plan, sh);
	if (kind) *kind = sh.kind;
	return CG_OK;
}

/*
 * Launches the plan-specialised kernel over plan.selected[0 .. nselected).  *launched = false
 * (and CG_OK) when the JIT is unavailable -- the caller then uses its ahead-of-time kernels.
 * *used_packed tells the caller that packed words were written.
 */
int cg_launch_scan_jit(CgContext *ctx, const KPlan &plan, uint32_t nullable, cudaStream_t stream, bool *launched, bool *used_packed,
					   bool *packed_only)
{
	*launched = false;
	*used_packed = false;
	if (packed_only) *packed_only = false;
	if (cg_jit_level() <= 0 || plan.nselected == 0) return CG_OK;
	if (!load_rtc() || !load_drv()) return CG_OK;
	JitShape sh;
	choose_shape(plan, nullable, &sh);
	std::string src = gen_source(plan, sh);
	/* one compilation per distinct source, also when several host threads scan at once */
	std::unique_lock<std::mutex> lock(g_cache_mutex);
	JitKernel *k = &g_cache[src];
	if (k->failed) return CG_OK;
	if (!k->fn)
	{
		int rc = compile_source(src, &k->cubin);
		if (rc) { k->failed = true; fprintf(stderr, "[cg] jit disabled for this plan: %s\n", cg_last_error()); return CG_OK; }
		CUmodule mod = nullptr;
		int e = g_api.load(&mod, k->cubin.data());
		if (e == 0) e = g_api.getfn(&k->fn, mod, "cg_jit_scan");
		if (e != 0)
		{
			k->failed = true; k->fn = nullptr;
			fprintf(stderr, "[cg] jit: loading the compiled kernel failed (CUresult %d)\n", e);
			return CG_OK;
		}
		if (getenv("CG_JIT_DUMP")) fprintf(stderr, "%s\n", src.c_str());
	}
	/* dynamic shared memory: the SMALL kind's cells + the staged exists bitmaps / rank directories of nullable columns */
	KPlan sized = plan;
	size_t smem = sh.smem;
	if (sh.nullable)
	{
		int nn = 0;
		for (int c = 0; c < plan.ncols; c++) if (col_nullable(sh, c)) nn++;
		if (sized.max_cg_rows == 0) sized.max_cg_rows = (uint32_t) JIT_MAX_CHUNK_ROWS;
		smem += (size_t) nn * (sized.max_cg_rows / 64u + 2u) * 12u + 16u;
	}
	if (smem > 220 * 1024) { lock.unlock(); return CG_OK; }        /* does not fit: the caller's ahead-of-time kernels take it */
	if (smem > k->smem_configured || k->occupancy == 0)
	{
		if (smem > 48 * 1024)
		{
			int e = g_api.setattr(k->fn, CG_CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int) smem);
			if (e != 0) return cg_set_error(CG_ECUDA, "cuFuncSetAttribute(%zu bytes of shared memory) failed: %d", smem, e);
		}
		k->smem_configured = smem;
		int occ = 0;
		if (g_api.occupancy(&occ, k->fn, JIT_THREADS, smem) != 0 || occ < 1) occ = 1;
		k->occupancy = occ;
	}
	lock.unlock();
	const uint32_t grid_full = (uint32_t) (ctx->sm_count * k->occupancy);
	/* SMALL with single-cell sums: bound the rows a lane can see in one launch */
	uint32_t max_cgs_per_launch = UINT32_MAX;
	if (sh.kind == JK_SMALL)
	{
		const int64_t cg_rows = plan.max_cg_rows ? (int64_t) plan.max_cg_rows : JIT_MAX_CHUNK_ROWS;
		int64_t rows_per_cg_lane = ((cg_rows + JIT_THREADS * sh.R - 1) / (JIT_THREADS * sh.R)) * sh.R;
		int64_t cgs_per_cta = sh.lane_rows_cap / rows_per_cg_lane;
		if (cgs_per_cta < 1) { fprintf(stderr, "[cg] jit: chunk groups of %lld rows exceed the narrow cells' per-lane row cap\n", (long long) cg_rows); return CG_OK; }
		int64_t cap = cgs_per_cta * (int64_t) grid_full;
		if (cap < (int64_t) UINT32_MAX) max_cgs_per_launch = (uint32_t) cap;
	}
	for (uint32_t first = 0; first < plan.nselected; )
	{
		KPlan piece = sized;
		piece.selected = plan.selected + first;
		piece.nselected = std::min(plan.nselected - first, max_cgs_per_launch);
		piece.slices = 1; piece.slice_rows = 1u << 30;
		if (piece.nselected < 2 * grid_full && plan.max_cg_rows > 0)
		{
			/* the step is a multiple of 64 rows, so slices start on a word of the exists bitmaps / rank directories */
			cg_choose_slices(piece.nselected, grid_full, (uint32_t) (JIT_THREADS * sh.R * sh.U), plan.max_cg_rows, &piece.slices, &piece.slice_rows);
		}
		uint32_t grid = (uint32_t) std::min<uint64_t>(grid_full, (uint64_t) piece.nselected * (uint64_t) piece.slices);
		void *args[] = {&piece};
		bool overlap;
		int rc = cg_chain_scan(ctx, stream, true, &overlap);
		if (rc) return rc;
		CUlaunchAttribute attr;
		memset(&attr, 0, sizeof attr);
		attr.id = CU_LAUNCH_ATTRIBUTE_PROGRAMMATIC_STREAM_SERIALIZATION;
		attr.value.programmaticStreamSerializationAllowed = 1;
		CUlaunchConfig cfg;
		memset(&cfg, 0, sizeof cfg);
		cfg.gridDimX = grid; cfg.gridDimY = 1; cfg.gridDimZ = 1;
		cfg.blockDimX = JIT_THREADS; cfg.blockDimY = 1; cfg.blockDimZ = 1;
		cfg.sharedMemBytes = (unsigned) smem;
		cfg.hStream = (CUstream) stream;
		cfg.attrs = &attr;
		cfg.numAttrs = overlap ? 1 : 0;
		int e = g_api.launch(&cfg, k->fn, args, nullptr);
		if (e != 0)
		{
			const char *msg = nullptr;
			if (g_api.errstr) g_api.errstr(e, &msg);
			return cg_set_error(CG_ECUDA, "cuLaunchKernelEx of the plan-specialised kernel failed: %s", msg ? msg : "?");
		}
		g_cg_launches++;
		g_jit_launches++;
		first += piece.nselected;
	}
	*launched = true;
	*used_packed = sh.packed;
	if (packed_only && sh.packed)
	{
		/* nothing but the packed word is written when the plan is count(*) + the packed sum over NULL-free inputs */
		bool only = true;
		for (int a = 0; a < plan.naggs; a++)
			if ((plan.aggs[a].kind != CG_AGG_COUNT_STAR && a != sh.pack_agg) || plan.nfexpr[a] > 0) only = false;
		if (!agg_null_expr(plan.aggs[sh.pack_agg], sh).empty()) only = false;
		*packed_only = only;
	}
	return CG_OK;
}

extern "C" uint64_t cg_jit_launches(void) { return g_jit_launches; }
extern "C" uint64_t cg_jit_compiles(void) { return g_jit_compiles; }

/*
 * Generates and compiles (no launch, no GPU needed) the kernel a query shape would get:
 * the CPU-side check that every plan form produces valid sm_90a code.  kind: 0 plain
 * aggregate, 1 shared-memory cells, 2 global table.  source/source_len may be NULL/0.
 */
extern "C" int cg_jit_compile_check_nullable(const CgScanDesc *desc, const CgColumnDesc *columns, int32_t natts, int64_t key_min,
											 int64_t key_max, int64_t max_rows, uint32_t nullable_atts, int32_t *kind, char *source,
											 size_t source_len)
{
	if (!desc || !columns) return cg_set_error(CG_EINVAL, "NULL argument");
	CgPartial part;
	int rc = cg_partial_shape(&part, desc, columns, natts, key_min, key_max, max_rows);
	if (rc) return rc;
	/* packing as cg_partial_create would choose it, so that the packed form of the generated code is checked too */
	for (int a = 0; a < desc->naggs && !part.d_packed && (part.mode == CG_MODE_DENSE || part.mode == CG_MODE_HASH); a++)
	{
		const KAgg &k = part.aggs[a];
		if (k.kind != CG_AGG_SUM || k.is_float || k.nlimbs != 1 || k.bound <= 0) continue;
		part.d_packed = (uint64_t *) 16; part.pack_shift = 16; part.pack_word = k.word0; part.packing_enabled = true;
	}
	KPlan plan;
	bool all8 = false;
	rc = cg_build_plan(desc, columns, natts, nullptr, &part, &plan, &all8);
	part.d_packed = nullptr;
	if (rc) return rc;
	plan.nstaged = natts;
	/* attribute mask -> plan-column mask */
	uint32_t nullable = 0;
	for (int c = 0; c < plan.ncols; c++)
		if (plan.slot[c] < 32 && ((nullable_atts >> plan.slot[c]) & 1u)) nullable |= 1u << c;
	std::string src;
	int k = 0;
	cg_jit_source_for(plan, nullable, &src, &k);
	if (kind) *kind = k;
	if (source && source_len) { strncpy(source, src.c_str(), source_len - 1); source[source_len - 1] = '\0'; }
	std::string cubin;
	return compile_source(src, &cubin);
}

extern "C" int cg_jit_compile_check(const CgScanDesc *desc, const CgColumnDesc *columns, int32_t natts, int64_t key_min,
									int64_t key_max, int64_t max_rows, int32_t *kind, char *source, size_t source_len)
{
	return cg_jit_compile_check_nullable(desc, columns, natts, key_min, key_max, max_rows, 0u, kind, source, source_len);
}
