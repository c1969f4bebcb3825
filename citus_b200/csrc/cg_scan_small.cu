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
 * Semantics, decode and the general (interpretive) plan are those of cg_scan.cu, through the same
 * row helpers (cg_device.cuh): any column
 * width, NULLs through the rank directory, range/float quals, one or two group columns
 * (composite direct index), count/sum/min/max over products of up to three affine factors.
 * Reference: the worker HashAggregate of the task (PG nodeAgg) over ColumnarScan --
 * SURVEY.md 3.3; aggregate split planner/multi_logical_optimizer.c:3160-3484.
 */
#include "cg_internal.h"

#define CGS_THREADS 256

#include "cg_device.cuh"

/*
 * Accumulate one row into the lane's PRIVATE accumulators in shared memory, laid out
 * [group][hot word][lane] so that the 32 lanes of a warp always touch 32 consecutive words (no
 * bank conflicts) and never each other's: plain load / combine / store, no atomics, no
 * warp collectives.  (64-bit shared-memory atomics are CAS spin loops on this part --
 * ATOMS.CAST.SPIN -- and warp-level segmented reductions cost ~100 instructions per row.)
 * Only the words every row touches get a cell; NULL-input counters and the NULL-key group
 * are rare and go straight to the global table.
 */
template <int NCC, bool VAR, bool CASE = false>
__device__ __forceinline__ void small_accumulate(const KPlan &P, uint64_t *mine, uint32_t slot, const int64_t (&v)[NCC], uint32_t nullmask)
{
	uint64_t *e = mine + (size_t) slot * (uint32_t) P.nhot * CGS_THREADS;
	e[0] += 1ull;
	auto term = [&](int a, const KAgg &g, bool noinput, uint64_t w0, uint64_t w1) {
		if (noinput)
		{
			/* a filtered aggregate's no-input counter has a cell (rejected rows are common), and so has a CASE's (arms that
			 * give NULL are as common) */
			if (g.filt || g.barg || (CASE && P.cnarms[a] > 0)) e[P.hot_of_word[g.nullword] * CGS_THREADS] += 1ull;
			else atomicAdd((unsigned long long *) P.table + (uint64_t) slot * (uint64_t) P.stride + g.nullword, 1ull);
			return;
		}
		uint64_t *w = e + P.hot_of_word[g.word0] * CGS_THREADS;
		if ((g.kind == CG_AGG_SUM || (VAR && g.kind == CG_AGG_VARIANCE)) && !g.is_float)
		{
			*w += w0;
			if (two_sum_limbs<VAR>(g)) w[CGS_THREADS] += w1;
		}
		else
			*w = word_combine(P.wordop[g.word0], *w, w0);
	};
	if constexpr (VAR)
		/* sum(x^2): every limb word has a cell of its own (consecutive words: consecutive cells) */
		row_terms<NCC, CG_MAX_AGGS, true, CASE>(P, v, nullmask, term, [&](int, const KAgg &g, uint64_t lo, uint64_t hi) {
			uint64_t *q = e + P.hot_of_word[g.qword] * CGS_THREADS;
			if (g.qlimbs == 1) *q += lo;
			else
			{
#pragma unroll
				for (int l = 0; l < 4; l++)
					if (l < g.qlimbs) q[l * CGS_THREADS] += square_limb(lo, hi, l);
			}
		});
	else
		row_terms<NCC, CG_MAX_AGGS, false, CASE>(P, v, nullmask, term);
}

/* K3 + K4 of one row: WHERE, the group's direct index, the terms into the group's cells (the NULL-key group's go to its
 * global entry) */
template <int NCC, bool VAR, bool CASE = false>
__device__ __forceinline__ void small_row(const KPlan &P, uint64_t *mine, const int64_t (&v)[NCC], uint32_t nullmask, uint32_t &removed)
{
	if (!eval_where<NCC>(P, v, nullmask))
	{
		removed++;
		return;
	}
	int64_t key;
	bool key_null;
	if (!group_key<NCC>(P, v, nullmask, key, key_null)) return;
	const uint64_t slot = dense_slot_of_packed(P, key, key_null);
	if (slot == ~0ull) return;
	if (key_null) global_accumulate<NCC, CG_MAX_AGGS, VAR, CASE>(P, P.table + slot * (uint64_t) P.stride, v, nullmask);
	else small_accumulate<NCC, VAR, CASE>(P, mine, (uint32_t) slot, v, nullmask);
}

template <int NCC, bool ALL8, bool VAR = false, bool CASE = false>
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
		for (uint32_t r = tid * 2; r < rows; r += CGS_THREADS * 2)
		{
			int64_t v0[NCC], v1[NCC];
			uint32_t n0 = 0, n1 = 0;
#pragma unroll
			for (int c = 0; c < NCC; c++)
				if (c < P.ncols)
				{
					int len = ALL8 ? 8 : P.len[c];
					if ((hasnull >> c) & 1u)
					{
						const DevChunkCol *d = cc + P.slot[c];
						load_pair_nullable(vptr[c], (const uint64_t *) (P.arena + __ldg(&d->exists_off)),
										   (const uint32_t *) (P.arena + __ldg(&d->rank_off)), r, rows, len, P.isfloat[c], c, v0[c], v1[c],
										   n0, n1);
					}
					else
						load_pair(vptr[c], r, len, P.isfloat[c], v0[c], v1[c]);
				}
			small_row<NCC, VAR, CASE>(P, mine, v0, n0, removed);
			if (r + 1 < rows) small_row<NCC, VAR, CASE>(P, mine, v1, n1, removed);
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
	unsigned long long rem = warp_reduce_word(removed, CG_WORD_ADD);
	unsigned long long scn = warp_reduce_word(scanned, CG_WORD_ADD);
	if ((tid & 31) == 0)
	{
		if (scn) atomicAdd(P.stats + 0, scn);
		if (rem) atomicAdd(P.stats + 1, rem);
	}
}

template <int NCC, bool ALL8, bool VAR = false, bool CASE = false>
static int launch_small_variant(CgContext *ctx, const KPlan &plan, size_t smem, cudaStream_t stream)
{
	static size_t configured = 0, occ_smem = ~(size_t) 0;
	static int occ = 0;
	if (smem > configured)
	{
		CG_CUDA(cudaFuncSetAttribute(cg_scan_small_kernel<NCC, ALL8, VAR, CASE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
		configured = smem;
	}
	if (smem != occ_smem)
	{
		CG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, cg_scan_small_kernel<NCC, ALL8, VAR, CASE>, CGS_THREADS, smem));
		if (occ < 1) occ = 1;
		occ_smem = smem;
	}
	uint32_t grid = (uint32_t) (ctx->sm_count * occ);
	if (grid > plan.nselected) grid = plan.nselected;
	if (grid == 0) return CG_OK;
	bool overlap;
	int rc = cg_chain_scan(ctx, stream, false, &overlap);     /* does not trigger its dependents early: ends a chain */
	if (rc) return rc;
	cg_scan_small_kernel<NCC, ALL8, VAR, CASE><<<grid, CGS_THREADS, smem, stream>>>(plan);
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
		if (g.filt || g.barg || plan.cnarms[a] > 0) is_hot[g.nullword] = true;
		if (g.kind == CG_AGG_COUNT_STAR || g.kind == CG_AGG_COUNT) continue;
		is_hot[g.word0] = true;
		if (two_sum_limbs<true>(g)) is_hot[g.word0 + 1] = true;
		if (g.kind == CG_AGG_VARIANCE)
			for (int l = 0; l < g.qlimbs; l++) is_hot[g.qword + l] = true;
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
	if (plan.ncase > 0) return launch_small_variant<CG_KMAX_COLS, false, true, true>(ctx, plan, smem, stream);
	if (cg_plan_has_variance(plan.aggs, plan.naggs)) return launch_small_variant<CG_KMAX_COLS, false, true>(ctx, plan, smem, stream);
	if (plan.ncols <= 4)
		return all8 ? launch_small_variant<4, true>(ctx, plan, smem, stream) : launch_small_variant<4, false>(ctx, plan, smem, stream);
	return all8 ? launch_small_variant<CG_KMAX_COLS, true>(ctx, plan, smem, stream)
				: launch_small_variant<CG_KMAX_COLS, false>(ctx, plan, smem, stream);
}
