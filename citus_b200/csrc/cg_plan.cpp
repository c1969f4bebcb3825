/*
 * cg_plan.cpp -- turns a CgScanDesc into the kernel plan and the accumulator-word layout
 * of a partial aggregate.
 *
 * The worker half of each aggregate follows planner/multi_logical_optimizer.c:3160-3484
 * (WorkerAggregateExpressionList): count -> count, sum -> sum, min/max -> min/max,
 * avg -> sum + count (the caller asks for sum; the non-NULL count rides along as the
 * aggregate's count word).  Transition semantics follow PostgreSQL's nodeAgg:
 * strict transition functions skip NULL inputs; sum/min/max over no non-NULL input is NULL.
 */
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "cg_internal.h"

static thread_local char g_errbuf[512];

int cg_set_error(int code, const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_errbuf, sizeof g_errbuf, fmt, ap);
	va_end(ap);
	return code;
}

extern "C" const char *cg_last_error(void) { return g_errbuf; }

static int validate_desc(const CgScanDesc *d, const CgColumnDesc *columns, int natts)
{
	if (d->nquals < 0 || d->nquals > CG_MAX_QUALS) return cg_set_error(CG_EINVAL, "nquals %d out of range", d->nquals);
	if (d->naggs < 0 || d->naggs > CG_MAX_AGGS) return cg_set_error(CG_EINVAL, "naggs %d out of range", d->naggs);
	if (d->ngroup_cols < 0 || d->ngroup_cols > CG_MAX_GROUP_COLS)
		return cg_set_error(CG_EINVAL, "ngroup_cols %d out of range", d->ngroup_cols);
	for (int c = 0; c < natts; c++)
	{
		int l = columns[c].attlen;
		const int cls = cg_type_class(columns[c]);
		if (l == -1)
		{
			if (cls != CG_TYPE_NUMERIC && cls != CG_TYPE_BPCHAR1)
				return cg_set_error(CG_EUNSUPPORTED, "column %d: varlena type other than numeric(p,s) / char(1)", c);
			if (cls == CG_TYPE_NUMERIC && (cg_type_scale(columns[c]) < 0 || cg_type_scale(columns[c]) > 18))
				return cg_set_error(CG_EUNSUPPORTED, "column %d: numeric scale %d", c, cg_type_scale(columns[c]));
			continue;
		}
		if (cls == CG_TYPE_NUMERIC || cls == CG_TYPE_BPCHAR1) return cg_set_error(CG_EINVAL, "column %d: varlena class with attlen %d", c, l);
		if (l != 1 && l != 2 && l != 4 && l != 8)
			return cg_set_error(CG_EUNSUPPORTED, "column %d: attlen %d (only fixed-width by-value types)", c, l);
		if (columns[c].type_class == CG_TYPE_FLOAT && l != 4 && l != 8)
			return cg_set_error(CG_EINVAL, "column %d: float with attlen %d", c, l);
	}
	for (int q = 0; q < d->nquals; q++)
	{
		if (d->quals[q].column < 0 || d->quals[q].column >= natts)
			return cg_set_error(CG_EINVAL, "qual %d: column %d out of range", q, d->quals[q].column);
		if (d->quals[q].op < CG_OP_LT || d->quals[q].op > CG_OP_NE)
			return cg_set_error(CG_EINVAL, "qual %d: bad operator", q);
	}
	if (d->nqual_expr < 0 || d->nqual_expr > CG_MAX_QEXPR) return cg_set_error(CG_EINVAL, "nqual_expr %d out of range", d->nqual_expr);
	if (d->nqual_expr > 0)
	{
		/* well-formed postfix: every operator finds two operands, one value is left */
		int depth = 0;
		for (int i = 0; i < d->nqual_expr; i++)
		{
			int t = d->qual_expr[i];
			if (t >= 0) { if (t >= d->nquals) return cg_set_error(CG_EINVAL, "qual_expr refers to atom %d of %d", t, d->nquals); depth++; }
			else if (t == CG_QX_AND || t == CG_QX_OR) { if (depth < 2) return cg_set_error(CG_EINVAL, "qual_expr: operator without operands"); depth--; }
			else return cg_set_error(CG_EINVAL, "qual_expr: bad token %d", t);
		}
		if (depth != 1) return cg_set_error(CG_EINVAL, "qual_expr leaves %d values", depth);
	}
	for (int g = 0; g < d->ngroup_cols; g++)
	{
		int c = d->group_cols[g];
		if (c < 0 || c >= natts) return cg_set_error(CG_EINVAL, "group column %d out of range", c);
		if (columns[c].type_class == CG_TYPE_FLOAT)
			return cg_set_error(CG_EUNSUPPORTED, "GROUP BY on a float column");
		if (d->ngroup_cols == 2 && cg_decoded_len(columns[c]) > 4)
			return cg_set_error(CG_EUNSUPPORTED, "two-column GROUP BY needs columns of at most 4 bytes");
	}
	for (int a = 0; a < d->naggs; a++)
	{
		const CgAggSpec &s = d->aggs[a];
		if (s.kind < CG_AGG_COUNT_STAR || s.kind > CG_AGG_MAX) return cg_set_error(CG_EINVAL, "aggregate %d: bad kind", a);
		if (s.nfactors < 0 || s.nfactors > 3) return cg_set_error(CG_EINVAL, "aggregate %d: nfactors", a);
		if (s.kind != CG_AGG_COUNT_STAR && s.nfactors == 0)
			return cg_set_error(CG_EINVAL, "aggregate %d needs an argument", a);
		for (int f = 0; f < s.nfactors; f++)
		{
			if (s.column[f] < 0 || s.column[f] >= natts)
				return cg_set_error(CG_EINVAL, "aggregate %d: column out of range", a);
			bool colf = columns[s.column[f]].type_class == CG_TYPE_FLOAT;
			if (s.kind != CG_AGG_COUNT && colf != (s.is_float != 0))
				return cg_set_error(CG_EINVAL, "aggregate %d: integer/float mismatch with column %d", a, s.column[f]);
		}
	}
	return CG_OK;
}

/*
 * Accumulator words of a group: word 0 = rows in the group (count(*) and occupancy);
 * then per aggregate
 *   count(x)      1 ADD word counting NULL inputs (count = rows - it)
 *   sum(int)      1 ADD word if |term| * max_rows < 2^63 (term_abs_bound given), else the
 *                 two-limb form (low 32 bits unsigned, term >> 32 signed), + NULL-input count
 *   sum(float8)   1 FADD word + NULL-input count
 *   min/max       1 MIN/MAX (FMIN/FMAX on the order-preserving float encoding) + NULL-input count
 * Counting the NULL inputs instead of the non-NULL ones keeps NULL-free data (the common
 * case) at one atomic per aggregate and row, while "no non-NULL input => SQL NULL" and
 * count(x) stay exact: non-NULL inputs = rows in group - NULL inputs.
 */
static int layout_partial(CgPartial *p, const CgColumnDesc *columns)
{
	const CgScanDesc &d = p->desc;
	int nw = 1;
	memset(p->wordop, CG_WORD_ADD, sizeof p->wordop);
	for (int a = 0; a < d.naggs; a++)
	{
		const CgAggSpec &s = d.aggs[a];
		KAgg &k = p->aggs[a];
		memset(&k, 0, sizeof k);
		k.kind = (int8_t) s.kind;
		k.nfactors = (int8_t) s.nfactors;
		k.is_float = (int8_t) (s.is_float != 0);
		for (int f = 0; f < 3; f++) { k.a[f] = s.a[f]; k.b[f] = s.b[f]; }
		k.nlimbs = 1;
		k.tbound = (s.kind == CG_AGG_SUM && !s.is_float && s.term_abs_bound > 0) ? s.term_abs_bound : 0;
		/* an integer argument other than a bare column can leave int64 ([PG] int8mul / int8pl raise "bigint out of
		 * range", numeric is exact): unless the caller proved a bound, the kernels check every factor and product */
		k.ovchk = (int8_t) (!s.is_float && (s.kind == CG_AGG_SUM || s.kind == CG_AGG_MIN || s.kind == CG_AGG_MAX) &&
							k.tbound == 0 && !(s.nfactors == 1 && s.a[0] == 0 && s.b[0] == 1));
		switch (s.kind)
		{
			case CG_AGG_COUNT_STAR:
				k.word0 = 0;
				break;
			case CG_AGG_COUNT:
				k.word0 = (int8_t) nw; k.nullword = (int8_t) nw; p->wordop[nw++] = CG_WORD_ADD;
				break;
			case CG_AGG_SUM:
				k.word0 = (int8_t) nw;
				if (s.is_float) p->wordop[nw++] = CG_WORD_FADD;
				else
				{
					p->wordop[nw++] = CG_WORD_ADD;
					bool one = false;
					if (s.term_abs_bound > 0 && p->max_rows > 0)
					{
						__int128 worst = (__int128) s.term_abs_bound * (__int128) p->max_rows;
						one = worst < ((__int128) 1 << 63);
					}
					if (one) { k.nlimbs = 1; k.bound = s.term_abs_bound; }
					else { k.nlimbs = 2; p->wordop[nw++] = CG_WORD_ADD; }
				}
				k.nullword = (int8_t) nw; p->wordop[nw++] = CG_WORD_ADD;
				break;
			default:
				k.word0 = (int8_t) nw;
				if (s.kind == CG_AGG_MIN) p->wordop[nw++] = s.is_float ? CG_WORD_FMIN : CG_WORD_MIN;
				else p->wordop[nw++] = s.is_float ? CG_WORD_FMAX : CG_WORD_MAX;
				k.nullword = (int8_t) nw; p->wordop[nw++] = CG_WORD_ADD;
				break;
		}
		if (nw > CG_KMAX_WORDS) return cg_set_error(CG_EUNSUPPORTED, "too many accumulator words (%d)", nw);
	}
	(void) columns;
	p->nwords = nw;
	return CG_OK;
}

/* host-only part of cg_partial_create: accumulator layout, table kind and capacity */
int cg_partial_shape(CgPartial *p, const CgScanDesc *desc, const CgColumnDesc *columns, int32_t natts,
					 int64_t key_min, int64_t key_max, int64_t max_rows)
{
	int rc = validate_desc(desc, columns, natts);
	if (rc) return rc;
	p->desc = *desc;
	p->columns.assign(columns, columns + natts);
	p->key_min = key_min;
	p->key_max = key_max;
	p->max_rows = max_rows;
	rc = layout_partial(p, columns);
	if (rc) return rc;

	const uint64_t kDenseLimit = 1ull << 26;
	if (desc->ngroup_cols == 0)
	{
		p->mode = CG_MODE_GLOBAL;
		p->capacity = 1; p->entries = 1; p->stride = p->nwords;
	}
	else if (desc->ngroup_cols == 2 &&
			 (int32_t) (uint32_t) key_min <= (int32_t) (uint32_t) key_max &&
			 (int32_t) ((uint64_t) key_min >> 32) <= (int32_t) ((uint64_t) key_max >> 32) &&
			 ((uint64_t) ((int64_t) (int32_t) (uint32_t) key_max - (int32_t) (uint32_t) key_min) + 1) *
				 ((uint64_t) ((int64_t) (int32_t) ((uint64_t) key_max >> 32) - (int32_t) ((uint64_t) key_min >> 32)) + 1) < kDenseLimit)
	{
		/* two group columns: key_min / key_max carry the per-column bounds packed like the key
		 * (low 32 bits: first column); composite direct index */
		int64_t min0 = (int32_t) (uint32_t) key_min, max0 = (int32_t) (uint32_t) key_max;
		int64_t min1 = (int32_t) ((uint64_t) key_min >> 32), max1 = (int32_t) ((uint64_t) key_max >> 32);
		p->mode = CG_MODE_DENSE;
		p->key_min = min0;
		p->key_min1 = min1;
		p->range1 = (uint64_t) (max1 - min1) + 1;
		p->capacity = ((uint64_t) (max0 - min0) + 1) * p->range1;
		p->entries = p->capacity + 1;
		int s = 1; while (s < p->nwords) s <<= 1;
		p->stride = s;
	}
	else if (desc->ngroup_cols == 1 && key_min <= key_max && ((uint64_t) key_max - (uint64_t) key_min) < kDenseLimit)
	{
		p->mode = CG_MODE_DENSE;
		p->capacity = ((uint64_t) key_max - (uint64_t) key_min) + 1;
		p->entries = p->capacity + 1;            /* + the NULL group */
		int s = 1; while (s < p->nwords) s <<= 1;   /* power-of-two stride: an entry never straddles a sector pair */
		p->stride = s;
	}
	else
	{
		p->mode = CG_MODE_HASH;
		/* load factor <= 1/4: ~7 of 8 lookups end at the home slot (the probe loop diverges a warp) */
		uint64_t want = desc->expected_groups > 0 ? (uint64_t) desc->expected_groups * 4 : (1ull << 22);
		uint64_t cap = 1024; while (cap < want) cap <<= 1;
		p->capacity = cap;
		p->entries = cap + 2;                    /* + NULL group + the key equal to the EMPTY sentinel */
		int s = 1; while (s < p->nwords) s <<= 1;
		p->stride = s;
	}
	return CG_OK;
}

extern "C" int cg_partial_create(const CgScanDesc *desc, const CgColumnDesc *columns, int32_t natts,
								 int64_t key_min, int64_t key_max, int64_t max_rows, CgPartial **out)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (!desc || !columns || !out) return cg_set_error(CG_EINVAL, "NULL argument");
	CgPartial *p = new CgPartial();
	int rc = cg_partial_shape(p, desc, columns, natts, key_min, key_max, max_rows);
	if (rc) { delete p; return rc; }
	/* CG_COMM_TAIL words behind the accumulator words travel with them in a combine (cg_comm.cu) */
	size_t bytes = ((size_t) p->entries * p->stride + CG_COMM_TAIL) * sizeof(uint64_t);
	size_t key_bytes = p->mode == CG_MODE_HASH ? (((size_t) p->entries * sizeof(int64_t) + 255) & ~(size_t) 255) : 0;
	if (cudaMalloc(&p->d_table, bytes + key_bytes) != cudaSuccess)
	{
		delete p;
		return cg_set_error(CG_ENOMEM, "cudaMalloc of %zu bytes for the group table failed", bytes + key_bytes);
	}
	if (key_bytes) p->d_hkeys = (int64_t *) ((uint8_t *) p->d_table + bytes);
	if (cudaMalloc(&p->d_stats, 8 * sizeof(unsigned long long)) != cudaSuccess ||
		cudaMalloc(&p->d_out_count, 2 * sizeof(unsigned long long)) != cudaSuccess)
	{
		cg_partial_free(p);
		return cg_set_error(CG_ENOMEM, "cudaMalloc failed");
	}
	/* optimistic packing: direct-indexed table, count + the first single-word integer sum.
	 * |term| <= bound < 2^R and at most 2^C - 1 rows per group between drains keep
	 * (sum << C) + count inside 64 bits when R + 2C <= 63. */
	if (p->mode == CG_MODE_DENSE || p->mode == CG_MODE_HASH)
	{
		static int env_pack = -1;
		if (env_pack < 0) { const char *e = getenv("CG_PACKING"); env_pack = e ? atoi(e) : 1; }
		for (int a = 0; a < desc->naggs && env_pack && !p->d_packed; a++)
		{
			const KAgg &k = p->aggs[a];
			if (k.kind != CG_AGG_SUM || k.is_float || k.nlimbs != 1 || k.bound <= 0) continue;
			int R = 0;
			while (R < 62 && ((int64_t) 1 << R) <= k.bound) R++;
			int Cbits = (63 - R) / 2;
			if (Cbits < 12) continue;
			if (Cbits > 24) Cbits = 24;
			if (cudaMalloc(&p->d_packed, ((size_t) p->entries + CG_COMM_TAIL) * sizeof(uint64_t)) != cudaSuccess)
			{
				cg_partial_free(p);
				return cg_set_error(CG_ENOMEM, "cudaMalloc for the packed accumulators failed");
			}
			p->pack_shift = Cbits;
			p->pack_word = k.word0;
			p->packing_enabled = true;
		}
	}
	rc = cg_launch_table_init(p, ctx->compute);
	if (rc) { cg_partial_free(p); return rc; }
	*out = p;
	return CG_OK;
}

extern "C" void cg_partial_free(CgPartial *p)
{
	if (!p) return;
	cudaFree(p->d_table); cudaFree(p->d_stats); cudaFree(p->d_out_keys); cudaFree(p->d_out_words); cudaFree(p->d_packed);
	cudaFree(p->d_out_nulls); cudaFree(p->d_out_count);
	if (p->h_out) cudaFreeHost(p->h_out);
	if (p->h_ret) cudaFreeHost(p->h_ret);
	delete p;
}

extern "C" int cg_partial_reset(CgPartial *p)
{
	CgContext *ctx = cg_ctx();
	if (!ctx || !p) return CG_EINVAL;
	return cg_launch_table_init(p, ctx->compute);
}

extern "C" int cg_partial_set_packing(CgPartial *p, int32_t enable)
{
	if (!p) return cg_set_error(CG_EINVAL, "NULL partial");
	if (p->packed_dirty) return cg_set_error(CG_EINVAL, "reset the partial before changing its packing mode");
	p->packing_enabled = enable != 0 && p->d_packed != nullptr;
	return CG_OK;
}

extern "C" int cg_partial_layout(const CgPartial *p, int32_t *nwords, int32_t *word_ops, int32_t *is_dense, int64_t *capacity)
{
	if (!p) return cg_set_error(CG_EINVAL, "NULL partial");
	if (nwords) *nwords = p->nwords;
	if (word_ops) for (int i = 0; i < p->nwords; i++) word_ops[i] = p->wordop[i];
	if (is_dense) *is_dense = p->mode == CG_MODE_DENSE;
	if (capacity) *capacity = (int64_t) p->capacity;
	return CG_OK;
}

/*
 * Kernel plan: deduplicated projection (columnar_customscan.c:1813-1851 ColumnarAttrNeeded:
 * only the columns the quals, group keys and aggregate arguments reference are read).
 */
int cg_build_plan(const CgScanDesc *desc, const CgColumnDesc *columns, int natts,
				  const std::vector<int32_t> *slot_of_att, CgPartial *partial, KPlan *plan, bool *all8)
{
	int rc = validate_desc(desc, columns, natts);
	if (rc) return rc;
	/* the partial must have been created for the same aggregate list */
	if (partial->desc.naggs != desc->naggs || partial->desc.ngroup_cols != desc->ngroup_cols)
		return cg_set_error(CG_EINVAL, "partial aggregate was created for a different query shape");
	for (int a = 0; a < desc->naggs; a++)
		if (memcmp(&partial->desc.aggs[a], &desc->aggs[a], sizeof(CgAggSpec)) != 0)
			return cg_set_error(CG_EINVAL, "partial aggregate was created for a different aggregate list");

	memset(plan, 0, sizeof *plan);
	int pcol_of_att[256];
	if (natts > 256) return cg_set_error(CG_EUNSUPPORTED, "more than 256 attributes");
	for (int c = 0; c < natts; c++) pcol_of_att[c] = -1;
	int ncols = 0;
	auto use = [&](int att) -> int {
		if (pcol_of_att[att] >= 0) return pcol_of_att[att];
		if (ncols == CG_KMAX_COLS) return -1;
		int slot = slot_of_att ? (*slot_of_att)[att] : att;
		if (slot < 0) return -2;
		plan->slot[ncols] = (uint8_t) slot;
		plan->len[ncols] = (uint8_t) cg_decoded_len(columns[att]);       /* a varlena column reaches the kernels decoded to a fixed width */
		plan->isfloat[ncols] = (uint8_t) (columns[att].type_class == CG_TYPE_FLOAT);
		pcol_of_att[att] = ncols;
		return ncols++;
	};
#define USE_OR_FAIL(dst, att)                                                                       \
	do {                                                                                            \
		int pc__ = use(att);                                                                        \
		if (pc__ == -1) return cg_set_error(CG_EUNSUPPORTED, "query reads more than %d columns", CG_KMAX_COLS); \
		if (pc__ == -2) return cg_set_error(CG_EINVAL, "column %d is not staged in this shard", att);  \
		dst = pc__;                                                                                 \
	} while (0)

	plan->nquals = desc->nquals;
	for (int q = 0; q < desc->nquals; q++)
	{
		int pc; USE_OR_FAIL(pc, desc->quals[q].column);
		plan->qcol[q] = (uint8_t) pc;
		plan->qop[q] = (uint8_t) desc->quals[q].op;
		plan->qk[q] = desc->quals[q].konst;
		{
			int64_t k = desc->quals[q].konst, lo = INT64_MIN, hi = INT64_MAX;
			bool neg = false;
			switch (desc->quals[q].op)
			{
				case CG_OP_LT: if (k == INT64_MIN) { lo = 1; hi = 0; } else hi = k - 1; break;
				case CG_OP_LE: hi = k; break;
				case CG_OP_EQ: lo = hi = k; break;
				case CG_OP_GE: lo = k; break;
				case CG_OP_GT: if (k == INT64_MAX) { lo = 1; hi = 0; } else lo = k + 1; break;
				default: lo = hi = k; neg = true; break;
			}
			plan->qlo[q] = lo; plan->qhi[q] = hi; plan->qneg[q] = neg;
		}
		if (columns[desc->quals[q].column].type_class == CG_TYPE_FLOAT && columns[desc->quals[q].column].attlen == 4)
		{
			/* float4 column values are promoted to float8; so is the constant (already float8 bits) */
		}
	}
	plan->slices = 1; plan->slice_rows = 1u << 30; plan->max_cg_rows = 0;
	plan->nqexpr = desc->nqual_expr;
	for (int i = 0; i < desc->nqual_expr; i++) plan->qexpr[i] = desc->qual_expr[i];
	plan->ngroup = desc->ngroup_cols;
	for (int g = 0; g < desc->ngroup_cols; g++)
	{
		int pc; USE_OR_FAIL(pc, desc->group_cols[g]);
		plan->gcol[g] = (uint8_t) pc;
	}
	plan->naggs = desc->naggs;
	for (int a = 0; a < desc->naggs; a++)
	{
		plan->aggs[a] = partial->aggs[a];
		for (int f = 0; f < desc->aggs[a].nfactors; f++)
		{
			int pc; USE_OR_FAIL(pc, desc->aggs[a].column[f]);
			plan->aggs[a].pcol[f] = (int8_t) pc;
		}
	}
	plan->ncols = ncols;
	bool a8 = true;
	for (int c = 0; c < ncols; c++) if (plan->len[c] != 8) a8 = false;
	*all8 = a8;

	plan->mode = partial->mode;
	plan->nwords = partial->nwords;
	plan->stride = partial->stride;
	plan->table = partial->d_table;
	plan->hkeys = partial->d_hkeys;
	plan->capacity = partial->capacity;
	plan->hash_shift = 64;
	for (uint64_t c = partial->capacity; c > 1; c >>= 1) plan->hash_shift--;
	plan->key_min = partial->key_min;
	plan->key_min1 = partial->key_min1;
	plan->range1 = partial->range1;
	memcpy(plan->wordop, partial->wordop, sizeof plan->wordop);
	plan->stats = partial->d_stats;
	plan->packed = partial->packing_enabled ? partial->d_packed : nullptr;
	plan->pack_shift = partial->pack_shift;
	plan->pack_word = partial->pack_word;
	return CG_OK;
}


/*
 * Specialised-kernel eligibility: 8-byte integer columns only; the WHERE list reduces to at
 * most two column ranges (btree conjuncts on one column intersect; a lone <> is a negated
 * point range); at most one group column; aggregates are count(*) and up to three
 * sum(column); every column plays exactly one role.  Anything else runs on the general
 * kernel.  NULLs are handled outside: the fast kernel only sees chunk groups whose plan
 * columns have none.
 */
bool cg_build_fast_plan(const CgScanDesc *desc, const KPlan &plan, bool all8, FPlan *fast)
{
	if (!all8 || plan.ngroup > 1 || plan.nqexpr != 0) return false;
	for (int c = 0; c < plan.ncols; c++) if (plan.isfloat[c]) return false;
	memset(fast, 0, sizeof *fast);
	bool used[CG_KMAX_COLS] = {false};
	int role = 0;

	/* ranges per plan column */
	int qcols[CG_KMAX_COLS]; int nqc = 0;
	int64_t lo[CG_KMAX_COLS], hi[CG_KMAX_COLS]; bool neg[CG_KMAX_COLS]; int nconj[CG_KMAX_COLS];
	for (int q = 0; q < plan.nquals; q++)
	{
		int c = plan.qcol[q], i;
		for (i = 0; i < nqc; i++) if (qcols[i] == c) break;
		if (i == nqc) { qcols[nqc] = c; lo[i] = INT64_MIN; hi[i] = INT64_MAX; neg[i] = false; nconj[i] = 0; nqc++; }
		int64_t k = plan.qk[q];
		if (neg[i]) return false;
		nconj[i]++;
		switch (plan.qop[q])
		{
			case CG_OP_LT: if (k == INT64_MIN) { lo[i] = 1; hi[i] = 0; } else hi[i] = std::min(hi[i], k - 1); break;
			case CG_OP_LE: hi[i] = std::min(hi[i], k); break;
			case CG_OP_EQ: lo[i] = std::max(lo[i], k); hi[i] = std::min(hi[i], k); break;
			case CG_OP_GE: lo[i] = std::max(lo[i], k); break;
			case CG_OP_GT: if (k == INT64_MAX) { lo[i] = 1; hi[i] = 0; } else lo[i] = std::max(lo[i], k + 1); break;
			default:
				if (nconj[i] != 1) return false;
				neg[i] = true; lo[i] = hi[i] = k;
				break;
		}
	}
	if (nqc > 2) return false;
	for (int i = 0; i < nqc; i++)
	{
		if (lo[i] > hi[i]) { lo[i] = 1; hi[i] = 0; }     /* empty range: nothing passes */
		fast->slot[role++] = plan.slot[qcols[i]];
		fast->qlo[i] = lo[i]; fast->qhi[i] = hi[i]; fast->qneg[i] = neg[i];
		used[qcols[i]] = true;
	}
	fast->nquals = nqc;
	if (plan.ngroup == 1)
	{
		if (used[plan.gcol[0]]) return false;
		used[plan.gcol[0]] = true;
		fast->slot[role++] = plan.slot[plan.gcol[0]];
	}
	int ns = 0;
	for (int a = 0; a < plan.naggs; a++)
	{
		const KAgg &g = plan.aggs[a];
		if (g.kind == CG_AGG_COUNT_STAR) continue;
		if (g.kind != CG_AGG_SUM || g.is_float || g.nfactors != 1 || g.a[0] != 0 || g.b[0] != 1) return false;
		if (ns == 3 || used[g.pcol[0]]) return false;
		used[g.pcol[0]] = true;
		fast->slot[role++] = plan.slot[g.pcol[0]];
		fast->sword[ns] = (uint8_t) g.word0;
		fast->slimbs[ns] = (uint8_t) g.nlimbs;
		fast->sbound[ns] = g.bound;
		ns++;
	}
	fast->nsums = ns;
	fast->mode = plan.mode;
	fast->packed = nullptr;
	fast->pack_sum = -1;
	if (plan.packed && plan.mode != CG_MODE_GLOBAL)
		for (int i = 0; i < ns; i++)
			if (fast->sword[i] == plan.pack_word && fast->slimbs[i] == 1)
			{
				fast->packed = plan.packed;
				fast->pack_shift = plan.pack_shift;
				fast->pack_sum = i;
			}
	if (fast->pack_sum > 0)
	{
		/* the kernel packs sum number 0: move the packed sum to the front of the sum roles */
		int i = fast->pack_sum, base = role - ns;
		std::swap(fast->slot[base], fast->slot[base + i]);
		std::swap(fast->sword[0], fast->sword[i]);
		std::swap(fast->slimbs[0], fast->slimbs[i]);
		std::swap(fast->sbound[0], fast->sbound[i]);
		fast->pack_sum = 0;
	}
	{
		/* tuning switches (measurements only): CG_FAST_FLAGS overrides the default */
		static int env_flags = -1;
		if (env_flags < 0) { const char *e = getenv("CG_FAST_FLAGS"); env_flags = e ? atoi(e) : (int) CG_FAST_PAIRED; }
		fast->flags = (uint32_t) env_flags;
		bool single = true;
		for (int i = 0; i < ns; i++) if (fast->slimbs[i] != 1) single = false;
		if (!single) fast->flags &= ~CG_FAST_PAIRED;
	}
	fast->arena = plan.arena; fast->chunkcols = plan.chunkcols; fast->selected = plan.selected;
	fast->nselected = plan.nselected; fast->nstaged = plan.nstaged;
	fast->table = plan.table; fast->hkeys = plan.hkeys; fast->capacity = plan.capacity; fast->stride = plan.stride;
	fast->hash_shift = plan.hash_shift;
	fast->key_min = plan.key_min; fast->stats = plan.stats;
	fast->slices = 1; fast->slice_rows = 1u << 30; fast->max_cg_rows = plan.max_cg_rows;
	(void) desc;
	return true;
}
