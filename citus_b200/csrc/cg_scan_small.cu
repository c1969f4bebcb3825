/*
 * cg_scan_small.cu -- the fused scan kernel for GROUP BY over a tiny key domain
 * (TPC-H Q1: l_returnflag x l_linestatus, a handful of groups x many aggregates).
 *
 * With a few groups every row of a warp hits the same few table entries: global (or even
 * shared-memory) atomics per row would serialise on those addresses.  Instead the group
 * table lives in shared memory ("shared-memory staging of the group-by hash table"), one
 * private copy per LANE: a row is a plain load / add / store on the lane's own accumulators
 * -- no atomics, no warp collectives; the CTA combines its lanes' tables and flushes them to
 * the global direct-indexed table once, at the end.
 *
 * Semantics, decode and the general (interpretive) plan are those of cg_scan.cu: any column
 * width, NULLs through the rank directory, range/float quals, one or two group columns
 * (composite direct index), count/sum/min/max over products of up to three affine factors.
 * Reference: the worker HashAggregate of the task (PG nodeAgg) over ColumnarScan --
 * SURVEY.md 3.3; aggregate split planner/multi_logical_optimizer.c:3160-3484.
 */
#include "cg_internal.h"

#define CGS_THREADS 256

#include "cg_device.cuh"

/* direct index of a (composite) group key; false = not representable (flag raised) */
template <int NCC>
__device__ __forceinline__ bool small_slot(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask, uint32_t &slot)
{
	int c0 = P.gcol[0];
	if (P.ngroup == 1)
	{
		if ((nullmask >> c0) & 1u) { slot = (uint32_t) P.capacity; return true; }   /* the NULL group */
		uint64_t s = (uint64_t) pick<NCC>(v, c0) - (uint64_t) P.key_min;
		if (s >= P.capacity) { atomicOr(P.stats + 2, CG_ERRFLAG_KEY_RANGE); return false; }
		slot = (uint32_t) s;
		return true;
	}
	int c1 = P.gcol[1];
	if (((nullmask >> c0) | (nullmask >> c1)) & 1u) { atomicOr(P.stats + 2, CG_ERRFLAG_NULL_MULTIKEY); return false; }
	uint64_t a = (uint64_t) (int64_t) (int32_t) pick<NCC>(v, c0) - (uint64_t) P.key_min;
	uint64_t b = (uint64_t) (int64_t) (int32_t) pick<NCC>(v, c1) - (uint64_t) P.key_min1;
	if (b >= P.range1 || a * P.range1 + b >= P.capacity) { atomicOr(P.stats + 2, CG_ERRFLAG_KEY_RANGE); return false; }
	slot = (uint32_t) (a * P.range1 + b);
	return true;
}

__device__ __forceinline__ uint64_t warp_reduce_op(uint64_t x, int op)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
	{
		uint64_t y = __shfl_xor_sync(0xffffffffu, x, o);
		x = word_combine(op, x, y);
	}
	return x;
}

/* the values one row contributes: per aggregate (word0 value, second limb, NULL-input flag) */
template <int NCC>
struct RowTerms
{
	uint64_t w0[CG_MAX_AGGS];
	uint64_t w1[CG_MAX_AGGS];
	uint32_t nullbits;      /* bit a: aggregate a saw a NULL input */
};

template <int NCC>
__device__ __forceinline__ bool eval_quals(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask)
{
	return eval_where<NCC>(P, v, nullmask);
}

template <int NCC>
__device__ __forceinline__ void eval_terms(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask, RowTerms<NCC> &t)
{
	/* a row an aggregate's FILTER rejects is no input of it, like a NULL input; so is a row whose bool_and / bool_or
	 * argument is UNKNOWN */
	uint32_t argtrue;
	t.nullbits = eval_filters<NCC>(P, v, nullmask, &argtrue);
#pragma unroll
	for (int a = 0; a < CG_MAX_AGGS; a++)
	{
		t.w0[a] = 0; t.w1[a] = 0;
		if (a < P.naggs)
		{
			const KAgg &g = P.aggs[a];
			if (g.kind == CG_AGG_COUNT_STAR) continue;
			bool isnull = (t.nullbits >> a) & 1u;
			int64_t it = 1;
			double ft = 1.0;
#pragma unroll
			for (int f = 0; f < 3; f++)
				if (f < g.nfactors)
				{
					int c = g.pcol[f];
					isnull = isnull || ((nullmask >> c) & 1u);
					if (g.is_float) ft *= __longlong_as_double(g.a[f]) + __longlong_as_double(g.b[f]) * __longlong_as_double(pick<NCC>(v, c));
				}
			if (!g.is_float) it = int_term<NCC>(g, v, isnull, P.stats);
			if (isnull) { t.nullbits |= 1u << a; continue; }
			if (g.kind == CG_AGG_COUNT) continue;
			if (g.kind == CG_AGG_SUM)
			{
				if (g.is_float) t.w0[a] = (uint64_t) __double_as_longlong(ft);
				else if (g.nlimbs == 1)
				{
					if (it > g.bound || it < -g.bound) atomicOr(P.stats + 2, CG_ERRFLAG_SUM_BOUND);
					t.w0[a] = (uint64_t) it;
				}
				else { t.w0[a] = (uint64_t) (uint32_t) it; t.w1[a] = (uint64_t) (it >> 32); }
			}
			else if (g.barg)
				t.w0[a] = ((argtrue >> a) & 1u) ? ~0ull : 0ull;
			else
				t.w0[a] = g.is_float ? f8_ordered(__double_as_longlong(ft)) : (uint64_t) it;
		}
	}
}

/*
 * Accumulate one row into the lane's PRIVATE accumulators in shared memory, laid out
 * [group][hot word][lane] so that the 32 lanes of a warp always touch 32 consecutive words (no
 * bank conflicts) and never each other's: plain load / combine / store, no atomics, no
 * warp collectives.  (64-bit shared-memory atomics are CAS spin loops on this part --
 * ATOMS.CAST.SPIN -- and warp-level segmented reductions cost ~100 instructions per row.)
 * Only the words every row touches get a cell; NULL-input counters and the NULL-key group
 * are rare and go straight to the global table.
 */
template <int NCC>
__device__ __forceinline__ void small_accumulate(const KPlan &P, uint64_t *mine, uint32_t slot, const RowTerms<NCC> &t)
{
	if (slot >= (uint32_t) P.capacity)
	{
		/* the NULL-key group */
		uint64_t *ge = P.table + (uint64_t) slot * (uint64_t) P.stride;
		atomicAdd((unsigned long long *) ge, 1ull);
#pragma unroll
		for (int a = 0; a < CG_MAX_AGGS; a++)
			if (a < P.naggs)
			{
				const KAgg &g = P.aggs[a];
				if ((t.nullbits >> a) & 1u) { atomicAdd((unsigned long long *) ge + g.nullword, 1ull); continue; }
				if (g.kind == CG_AGG_COUNT_STAR || g.kind == CG_AGG_COUNT) continue;
				word_apply_global(ge + g.word0, P.wordop[g.word0], t.w0[a]);
				if (g.kind == CG_AGG_SUM && !g.is_float && g.nlimbs == 2)
					atomicAdd((unsigned long long *) ge + g.word0 + 1, (unsigned long long) t.w1[a]);
			}
		return;
	}
	uint64_t *e = mine + (size_t) slot * (uint32_t) P.nhot * CGS_THREADS;
	e[0] += 1ull;
#pragma unroll
	for (int a = 0; a < CG_MAX_AGGS; a++)
		if (a < P.naggs)
		{
			const KAgg &g = P.aggs[a];
			if ((t.nullbits >> a) & 1u)
			{
				/* a filtered aggregate's no-input counter has a cell (rejected rows are common) */
				if (g.filt || g.barg) e[P.hot_of_word[g.nullword] * CGS_THREADS] += 1ull;
				else atomicAdd((unsigned long long *) P.table + (uint64_t) slot * (uint64_t) P.stride + g.nullword, 1ull);
				continue;
			}
			if (g.kind == CG_AGG_COUNT_STAR || g.kind == CG_AGG_COUNT) continue;
			uint64_t *w = e + P.hot_of_word[g.word0] * CGS_THREADS;
			if (g.kind == CG_AGG_SUM && !g.is_float)
			{
				*w += t.w0[a];
				if (g.nlimbs == 2) w[CGS_THREADS] += t.w1[a];
			}
			else
				*w = word_combine(P.wordop[g.word0], *w, t.w0[a]);
		}
}

template <int NCC, bool ALL8>
__global__ void __launch_bounds__(CGS_THREADS)
cg_scan_small_kernel(const __grid_constant__ KPlan P)
{
	extern __shared__ uint64_t s_acc[];        /* [capacity][nhot][CGS_THREADS] */
	const uint32_t tid = threadIdx.x;
	const uint32_t cells = (uint32_t) P.capacity * (uint32_t) P.nhot;
	for (uint32_t i = 0; i < cells; i++)
	{
		/* cell -> word: the hot words are in ascending word order */
		uint32_t hw = i % (uint32_t) P.nhot, word = 0;
		for (uint32_t w = 0; w < (uint32_t) P.nwords; w++) if (P.hot_of_word[w] == (int) hw) word = w;
		s_acc[(size_t) i * CGS_THREADS + tid] = word_identity(P.wordop[word]);
	}
	uint64_t *mine = s_acc + tid;               /* this lane's private accumulators */

	uint32_t removed = 0;
	unsigned long long scanned = 0;
	for (uint32_t ci = blockIdx.x; ci < P.nselected; ci += gridDim.x)
	{
		const DevChunkCol *cc = P.chunkcols + (uint64_t) P.selected[ci] * (uint64_t) P.nstaged;
		const uint8_t *vptr[NCC];
		uint32_t hasnull = 0;
		const uint32_t rows = __ldg(&cc[0].row_count);
#pragma unroll
		for (int c = 0; c < NCC; c++)
			if (c < P.ncols)
			{
				const DevChunkCol *d = cc + P.slot[c];
				vptr[c] = P.arena + __ldg(&d->values_off);
				if (__ldg(&d->value_count) != rows) hasnull |= 1u << c;
			}
		scanned += (tid == 0) ? rows : 0;
		/* all lanes of a warp iterate together: lanes past the end carry no row */
		for (uint32_t base = 0; base < rows; base += CGS_THREADS * 2)
		{
			const uint32_t r = base + tid * 2;
			int64_t v0[NCC], v1[NCC];
			uint32_t n0 = 0, n1 = 0;
			if (r < rows)
			{
#pragma unroll
				for (int c = 0; c < NCC; c++)
					if (c < P.ncols)
					{
						int len = ALL8 ? 8 : P.len[c];
						bool isf = P.isfloat[c];
						if ((hasnull >> c) & 1u)
						{
							const DevChunkCol *d = cc + P.slot[c];
							const uint64_t *bm = (const uint64_t *) (P.arena + __ldg(&d->exists_off));
							const uint32_t *rk = (const uint32_t *) (P.arena + __ldg(&d->rank_off));
							uint64_t w = ldg_stream8(bm + (r >> 6));
							uint32_t sh = r & 63u;
							uint32_t before = __ldg(rk + (r >> 6)) + __popcll(w & ((1ull << sh) - 1ull));
							uint32_t e0 = (uint32_t) (w >> sh) & 1u, e1 = (uint32_t) (w >> (sh + 1)) & 1u;
							v0[c] = e0 ? load_scalar(vptr[c] + (uint64_t) before * len, len, isf) : 0;
							v1[c] = (e1 && r + 1 < rows) ? load_scalar(vptr[c] + (uint64_t) (before + e0) * len, len, isf) : 0;
							n0 |= (e0 ^ 1u) << c;
							n1 |= (e1 ^ 1u) << c;
						}
						else
							load_pair(vptr[c], r, len, isf, v0[c], v1[c]);
					}
			}
#pragma unroll
			for (int half = 0; half < 2; half++)
			{
				const bool valid = r + half < rows;
				int slot = -1;
				RowTerms<NCC> t;
				t.nullbits = 0;
				if (valid)
				{
					const uint32_t nm = half ? n1 : n0;
					bool pass = half ? eval_quals<NCC>(P, v1, nm) : eval_quals<NCC>(P, v0, nm);
					if (!pass) removed++;
					else
					{
						uint32_t s;
						bool ok = half ? small_slot<NCC>(P, v1, nm, s) : small_slot<NCC>(P, v0, nm, s);
						if (ok)
						{
							slot = (int) s;
							if (half) eval_terms<NCC>(P, v1, nm, t); else eval_terms<NCC>(P, v0, nm, t);
						}
					}
				}
				if (slot >= 0) small_accumulate<NCC>(P, mine, (uint32_t) slot, t);
			}
		}
	}

	/* flush: combine the 256 lanes of every cell, one global atomic per touched word of this CTA */
	__syncthreads();
	for (uint32_t i = tid; i < cells; i += CGS_THREADS)
	{
		uint32_t hw = i % (uint32_t) P.nhot, word = 0;
		for (uint32_t w = 0; w < (uint32_t) P.nwords; w++) if (P.hot_of_word[w] == (int) hw) word = w;
		const int op = P.wordop[word];
		const uint64_t *col = s_acc + (size_t) i * CGS_THREADS;
		uint64_t x = word_identity(op);
		for (uint32_t k = 0; k < CGS_THREADS; k++) x = word_combine(op, x, col[(k + tid) % CGS_THREADS]);
		if (x != word_identity(op))
			word_apply_global(P.table + (uint64_t) (i / (uint32_t) P.nhot) * (uint64_t) P.stride + word, op, x);
	}
	unsigned long long rem = warp_reduce_op(removed, CG_WORD_ADD);
	unsigned long long scn = warp_reduce_op(scanned, CG_WORD_ADD);
	if ((tid & 31) == 0)
	{
		if (scn) atomicAdd(P.stats + 0, scn);
		if (rem) atomicAdd(P.stats + 1, rem);
	}
}

template <int NCC, bool ALL8>
static int launch_small_variant(CgContext *ctx, const KPlan &plan, size_t smem, cudaStream_t stream)
{
	static size_t configured = 0, occ_smem = ~(size_t) 0;
	static int occ = 0;
	if (smem > configured)
	{
		CG_CUDA(cudaFuncSetAttribute(cg_scan_small_kernel<NCC, ALL8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
		configured = smem;
	}
	if (smem != occ_smem)
	{
		CG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, cg_scan_small_kernel<NCC, ALL8>, CGS_THREADS, smem));
		if (occ < 1) occ = 1;
		occ_smem = smem;
	}
	uint32_t grid = (uint32_t) (ctx->sm_count * occ);
	if (grid > plan.nselected) grid = plan.nselected;
	if (grid == 0) return CG_OK;
	cg_scan_small_kernel<NCC, ALL8><<<grid, CGS_THREADS, smem, stream>>>(plan);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

/* the words that get per-lane cells: word 0, every aggregate's value words and the no-input counters of filtered
 * aggregates */
static int hot_words(const KPlan &plan, int8_t *hot)
{
	bool is_hot[CG_KMAX_WORDS] = {false};
	is_hot[0] = true;
	for (int a = 0; a < plan.naggs; a++)
	{
		const KAgg &g = plan.aggs[a];
		if (g.filt || g.barg) is_hot[g.nullword] = true;
		if (g.kind == CG_AGG_COUNT_STAR || g.kind == CG_AGG_COUNT) continue;
		is_hot[g.word0] = true;
		if (g.kind == CG_AGG_SUM && !g.is_float && g.nlimbs == 2) is_hot[g.word0 + 1] = true;
	}
	int n = 0;
	for (int w = 0; w < CG_KMAX_WORDS; w++) hot[w] = (w < plan.nwords && is_hot[w]) ? (int8_t) n++ : (int8_t) -1;
	return n;
}

/* true when private accumulators for every lane fit the CTA's shared memory */
bool cg_small_eligible(const KPlan &plan)
{
	if (plan.mode != CG_MODE_DENSE) return false;
	int8_t hot[CG_KMAX_WORDS];
	size_t bytes = (size_t) plan.capacity * hot_words(plan, hot) * sizeof(uint64_t) * CGS_THREADS;
	return bytes <= 200 * 1024;
}

int cg_launch_scan_small(CgContext *ctx, const KPlan &plan_in, bool all8, cudaStream_t stream)
{
	KPlan plan = plan_in;
	plan.nhot = hot_words(plan, plan.hot_of_word);
	size_t smem = (size_t) plan.capacity * plan.nhot * sizeof(uint64_t) * CGS_THREADS;
	if (plan.ncols <= 4)
		return all8 ? launch_small_variant<4, true>(ctx, plan, smem, stream) : launch_small_variant<4, false>(ctx, plan, smem, stream);
	return all8 ? launch_small_variant<CG_KMAX_COLS, true>(ctx, plan, smem, stream)
				: launch_small_variant<CG_KMAX_COLS, false>(ctx, plan, smem, stream);
}
