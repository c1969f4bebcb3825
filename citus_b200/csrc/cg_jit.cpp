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

#include "cg_internal.h"

/* ---- minimal NVRTC / driver API surface (headers are not needed: opaque handles + ints) ---- */
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
typedef int (*cuLaunchKernel_t)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, void *, void **, void **);
typedef int (*cuGetErrorString_t)(int, const char **);
#define CG_CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES 8

static struct
{
	bool tried_rtc = false, have_rtc = false, tried_drv = false, have_drv = false;
	nvrtcCreateProgram_t create; nvrtcCompileProgram_t compile; nvrtcGetSize_t cubin_size, log_size;
	nvrtcGetData_t cubin, log; nvrtcDestroyProgram_t destroy;
	cuModuleLoadData_t load; cuModuleGetFunction_t getfn; cuFuncSetAttribute_t setattr; cuOccupancy_t occupancy;
	cuLaunchKernel_t launch; cuGetErrorString_t errstr;
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
	g_api.launch = (cuLaunchKernel_t) dlsym(h, "cuLaunchKernel");
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
static bool agg_two_limbs(const KAgg &g) { return g.kind == CG_AGG_SUM && !g.is_float && g.nlimbs == 2; }

static std::string agg_null_expr(const KAgg &g, const JitShape &sh);

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
	for (int a = 0; a < CG_MAX_AGGS; a++) { sh->hot0[a] = -1; sh->lane1[a] = false; sh->half[a] = -1; sh->bias[a] = 0; }
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
				if (taken[x] || !agg_null_expr(plan.aggs[x], *sh).empty()) continue;
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
			if (g.kind == CG_AGG_SUM && !g.is_float)
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
		}
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
			/* not the shared-memory kind after all: no narrow cells */
			for (int a = 0; a < CG_MAX_AGGS; a++) { sh->half[a] = -1; sh->bias[a] = 0; }
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
		default: return "atomicMax((unsigned long long *) (" + p + "), (unsigned long long) (" + v + "));";
	}
}


static void gen_prelude(std::string &s)
{
	s +=
		"typedef unsigned long long uint64_t; typedef long long int64_t; typedef unsigned int uint32_t; typedef int int32_t;\n"
		"typedef unsigned short uint16_t; typedef short int16_t; typedef unsigned char uint8_t; typedef signed char int8_t;\n"
		"struct DevChunkCol { uint64_t values_off; uint64_t exists_off; uint64_t rank_off; uint32_t value_count; uint32_t row_count; };\n"
		"struct KAgg { int8_t kind; int8_t nfactors; int8_t is_float; int8_t nlimbs; int8_t pcol[3]; int8_t word0; int8_t nullword; int8_t ovchk; int8_t pad[2];\n"
		"  int64_t a[3]; int64_t b[3]; int64_t bound; int64_t tbound; };\n";
	addf(s,
		 "struct KPlan { const uint8_t *arena; const DevChunkCol *chunkcols; const uint32_t *selected; uint32_t nselected; int32_t nstaged;\n"
		 "  int32_t ncols; uint8_t slot[%d]; uint8_t len[%d]; uint8_t isfloat[%d];\n"
		 "  int32_t nquals; uint8_t qcol[%d]; uint8_t qop[%d]; int64_t qk[%d]; int64_t qlo[%d]; int64_t qhi[%d]; uint8_t qneg[%d];\n"
		 "  int32_t ngroup; uint8_t gcol[%d]; int32_t naggs; KAgg aggs[%d];\n"
		 "  int32_t mode; int32_t nwords; int32_t stride; uint64_t *table; int64_t *hkeys; uint64_t capacity; int32_t hash_shift;\n"
		 "  int64_t key_min; int64_t key_min1; uint64_t range1; uint8_t wordop[%d]; unsigned long long *stats;\n"
		 "  int8_t hot_of_word[%d]; int32_t nhot; uint64_t *packed; int32_t pack_shift; int32_t pack_word;\n"
		 "  int32_t nqexpr; int8_t qexpr[%d]; int32_t slices; uint32_t slice_rows; uint32_t max_cg_rows; };\n",
		 CG_KMAX_COLS, CG_KMAX_COLS, CG_KMAX_COLS, CG_MAX_QUALS, CG_MAX_QUALS, CG_MAX_QUALS, CG_MAX_QUALS, CG_MAX_QUALS, CG_MAX_QUALS,
		 CG_MAX_GROUP_COLS, CG_MAX_AGGS, CG_KMAX_WORDS, CG_KMAX_WORDS, CG_MAX_QEXPR);
	/* the text above must describe the host's structs exactly */
	addf(s, "static_assert(sizeof(DevChunkCol) == %zu, \"DevChunkCol\");\n", sizeof(DevChunkCol));
	addf(s, "static_assert(sizeof(KAgg) == %zu, \"KAgg\");\n", sizeof(KAgg));
	addf(s, "static_assert(sizeof(KPlan) == %zu, \"KPlan\");\n", sizeof(KPlan));
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
	std::vector<std::string> st;
	for (int i = 0; i < plan.nqexpr; i++)
	{
		int t = plan.qexpr[i];
		if (t >= 0) { snprintf(buf, sizeof buf, "t%d", t); st.push_back(buf); }
		else
		{
			std::string b = st.back(); st.pop_back();
			std::string a = st.back(); st.pop_back();
			st.push_back("(" + a + (t == CG_QX_AND ? " && " : " || ") + b + ")");
		}
	}
	return st.back();
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
		if (g.kind == CG_AGG_COUNT_STAR || (with_packed && a == sh.pack_agg)) continue;
		if (!an[a].empty()) addf(s, "%sif (an%d) red_add(e + %d, 1ull);\n", C, a, g.nullword);
		if (!agg_has_value(g)) continue;
		char p[32];
		snprintf(p, sizeof p, "e + %d", g.word0);
		std::string guard = an[a].empty() ? "" : ("if (!an" + std::to_string(a) + ") ");
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
	/* K3: the WHERE tree; an atom on a NULL input is not TRUE (three-valued logic) */
	for (int q = 0; q < plan.nquals; q++)
	{
		int c = plan.qcol[q];
		char nn[32] = "";
		if (col_nullable(sh, c)) snprintf(nn, sizeof nn, "!z%d && ", c);
		if (plan.isfloat[c])
		{
			const char *ops[] = {"<", "<=", "==", ">=", ">", "!="};
			addf(s, "%sconst bool t%d = %s(fcmp(v%d, P.qk[%d]) %s 0);\n", T, q, nn, c, q, ops[plan.qop[q]]);
		}
		else if (plan.qneg[q])
			addf(s, "%sconst bool t%d = %s!((v%d >= P.qlo[%d]) && (v%d <= P.qhi[%d]));\n", T, q, nn, c, q, c, q);
		else
			addf(s, "%sconst bool t%d = %s(v%d >= P.qlo[%d]) && (v%d <= P.qhi[%d]);\n", T, q, nn, c, q, c, q);
	}
	addf(s, "%sconst bool pass = %s;\n", T, where_expr(plan).c_str());
	addf(s, "%sif (!pass) removed++;\n%selse {\n", T, T);
	const char *B = "\t\t\t\t\t\t\t";
	/* group slot; a NULL key is its own group (the entry behind the addressable ones) */
	std::string zkey;
	if (plan.mode != CG_MODE_GLOBAL)
	{
		if (plan.ngroup == 1) { if (col_nullable(sh, plan.gcol[0])) zkey = "z" + std::to_string(plan.gcol[0]); }
		else
		{
			if (col_nullable(sh, plan.gcol[0])) zkey = "z" + std::to_string(plan.gcol[0]);
			if (col_nullable(sh, plan.gcol[1])) zkey += (zkey.empty() ? "z" : " || z") + std::to_string(plan.gcol[1]);
		}
	}
	if (plan.mode == CG_MODE_DENSE)
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
	/* NULL-input flags and terms */
	std::vector<std::string> an(plan.naggs), w0v(plan.naggs);
	for (int a = 0; a < plan.naggs; a++)
	{
		const KAgg &g = plan.aggs[a];
		if (g.kind == CG_AGG_COUNT_STAR) continue;
		an[a] = agg_null_expr(g, sh);
		if (!an[a].empty()) addf(s, "%sconst bool an%d = %s;\n", C, a, an[a].c_str());
		if (!agg_has_value(g)) continue;
		std::string e = term_expr(g, a);
		if (g.is_float) addf(s, "%sconst double ft%d = %s;\n", C, a, e.c_str());
		else
		{
			if (g.ovchk) addf(s, "%sbool ov%d = false;\n", C, a);
			addf(s, "%sconst int64_t it%d = %s;\n", C, a, e.c_str());
			if (g.ovchk)
				addf(s, "%sif (%sov%d) raise_flag(P.stats, %lluull);\n", C, an[a].empty() ? "" : ("!an" + std::to_string(a) + " && ").c_str(),
					 a, (unsigned long long) CG_ERRFLAG_TERM_OVERFLOW);
			if (g.kind == CG_AGG_SUM && g.nlimbs == 1)
				addf(s, "%sif (%s(it%d > P.aggs[%d].bound || it%d < -P.aggs[%d].bound)) raise_flag(P.stats, %lluull);\n", C,
					 an[a].empty() ? "" : ("!an" + std::to_string(a) + " && ").c_str(), a, a, a, a, (unsigned long long) CG_ERRFLAG_SUM_BOUND);
		}
		/* the word-0 value the aggregate contributes */
		char buf[128];
		if (g.kind == CG_AGG_SUM)
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
			if (g.kind == CG_AGG_COUNT_STAR) continue;
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
			if (g.kind == CG_AGG_COUNT_STAR) continue;
			/* NULL-input counters stay on global reductions (rare) */
			if (!an[a].empty()) addf(s, "%sif (an%d) red_add(P.table + slot * %dull + %d, 1ull);\n", D, a, plan.stride, g.nullword);
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
			if (g.kind == CG_AGG_SUM && !g.is_float)
			{
				if (sh.lane1[a]) addf(s, "%s%s%s += (uint64_t) it%d;\n", D, guard.c_str(), cell, a);
				else
					addf(s, "%s%s{ %s += (uint64_t) (uint32_t) it%d; e[%d] += (uint64_t) (it%d >> 32); }\n", D, guard.c_str(), cell, a,
						 (sh.hot0[a] + 1) * JIT_THREADS, a);
			}
			else
				addf(s, "%s%s%s = %s;\n", D, guard.c_str(), cell, op_combine(plan.wordop[g.word0], cell, w0v[a]).c_str());
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

static std::string gen_source(const KPlan &plan, const JitShape &sh)
{
	std::string s;
	s.reserve(32768);
	gen_prelude(s);
	if (sh.min_blocks > 0)
		addf(s, "extern \"C\" __global__ void __launch_bounds__(%d, %d) cg_jit_scan(const __grid_constant__ KPlan P)\n{\n", JIT_THREADS, sh.min_blocks);
	else
		addf(s, "extern \"C\" __global__ void __launch_bounds__(%d) cg_jit_scan(const __grid_constant__ KPlan P)\n{\n", JIT_THREADS);
	s += "\tconst uint32_t tid = threadIdx.x;\n\tuint32_t removed = 0;\n\tunsigned long long scanned = 0;\n\tuint64_t g_rows = 0;\n";
	if (sh.kind == JK_GLOBAL)
		for (int a = 0; a < plan.naggs; a++)
		{
			const KAgg &g = plan.aggs[a];
			if (g.kind != CG_AGG_COUNT_STAR && !agg_null_expr(g, sh).empty()) addf(s, "\tuint64_t g_n%d = 0;\n", a);
			if (!agg_has_value(g)) continue;
			addf(s, "\tuint64_t g_a%d_0 = %s, g_a%d_1 = 0;\n", a, op_identity(plan.wordop[g.word0]), a);
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
			if (g.kind != CG_AGG_COUNT_STAR && !agg_null_expr(g, sh).empty())
				addf(s, "\t{ uint64_t n = wsum(g_n%d); if ((tid & 31) == 0 && n) red_add(P.table + %d, n); }\n", a, g.nullword);
			if (!agg_has_value(g)) continue;
			int op = plan.wordop[g.word0];
			addf(s, "\t{ uint64_t x = g_a%d_0;\n\t  for (int o = 16; o > 0; o >>= 1) { uint64_t y = __shfl_xor_sync(0xffffffffu, x, o); x = %s; }\n", a,
				 op_combine(op, "x", "y").c_str());
			char p[48];
			snprintf(p, sizeof p, "P.table + %d", g.word0);
			addf(s, "\t  if ((tid & 31) == 0 && x != %s) { %s }\n", op_identity(op), op_apply_global(op, p, "x").c_str());
			if (agg_two_limbs(g))
				addf(s, "\t  uint64_t x1 = wsum(g_a%d_1); if ((tid & 31) == 0 && x1) red_add(P.table + %d, x1);\n", a, g.word0 + 1);
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
			if (!agg_has_value(g) || sh.half[a] >= 0) continue;
			int op = plan.wordop[g.word0];
			char p[32];
			snprintf(p, sizeof p, "ge + %d", g.word0);
			if (g.kind == CG_AGG_SUM && !g.is_float)
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

static int compile_source(const std::string &src, std::string *cubin)
{
	if (!load_rtc()) return cg_set_error(CG_EUNSUPPORTED, "libnvrtc is not available");
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
		int e = g_api.launch(k->fn, grid, 1, 1, JIT_THREADS, 1, 1, (unsigned) smem, (void *) stream, args, nullptr);
		if (e != 0)
		{
			const char *msg = nullptr;
			if (g_api.errstr) g_api.errstr(e, &msg);
			return cg_set_error(CG_ECUDA, "cuLaunchKernel of the plan-specialised kernel failed: %s", msg ? msg : "?");
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
			if (plan.aggs[a].kind != CG_AGG_COUNT_STAR && a != sh.pack_agg) only = false;
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
