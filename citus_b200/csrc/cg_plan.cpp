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

/* a postfix tree over atoms [0, natoms): every operator finds two operands, one value is left */
static int validate_postfix(const char *what, const int8_t *expr, int n, int natoms)
{
	int depth = 0;
	for (int i = 0; i < n; i++)
	{
		int t = expr[i];
		if (t >= 0) { if (t >= natoms) return cg_set_error(CG_EINVAL, "%s refers to atom %d of %d", what, t, natoms); depth++; }
		else if (t == CG_QX_AND || t == CG_QX_OR) { if (depth < 2) return cg_set_error(CG_EINVAL, "%s: operator without operands", what); depth--; }
		else return cg_set_error(CG_EINVAL, "%s: bad token %d", what, t);
	}
	if (depth != 1) return cg_set_error(CG_EINVAL, "%s leaves %d values", what, depth);
	return CG_OK;
}

static int validate_atoms(const char *what, const CgQual *quals, int n, int natts, int nin_lists)
{
	for (int q = 0; q < n; q++)
	{
		if (quals[q].column < 0 || quals[q].column >= natts)
			return cg_set_error(CG_EINVAL, "%s %d: column %d out of range", what, q, quals[q].column);
		if (quals[q].op < CG_OP_LT || (quals[q].op > CG_OP_IS_NOT_NULL && !cg_op_is_column(quals[q].op)))
			return cg_set_error(CG_EINVAL, "%s %d: bad operator", what, q);
		if (cg_op_is_column(quals[q].op) && (quals[q].konst < 0 || quals[q].konst >= natts))
			return cg_set_error(CG_EINVAL, "%s %d: other column %lld out of range", what, q, (long long) quals[q].konst);
		if ((quals[q].op == CG_OP_IN || quals[q].op == CG_OP_NOT_IN) && (quals[q].konst < 0 || quals[q].konst >= nin_lists))
			return cg_set_error(CG_EINVAL, "%s %d: list %lld of %d", what, q, (long long) quals[q].konst, nin_lists);
		if ((quals[q].op == CG_OP_IS_NULL || quals[q].op == CG_OP_IS_NOT_NULL) && quals[q].konst != 0)
			return cg_set_error(CG_EINVAL, "%s %d: IS [NOT] NULL with a constant", what, q);
	}
	return CG_OK;
}

/* the IN / NOT IN list table (CgScanDesc.in_lists / in_values) */
static int validate_lists(const CgScanDesc *d)
{
	if (d->nin_lists < 0 || d->nin_lists > CG_MAX_IN_LISTS) return cg_set_error(CG_EINVAL, "nin_lists %d out of range", d->nin_lists);
	if (d->nin_values < 0 || d->nin_values > CG_MAX_IN_VALUES) return cg_set_error(CG_EINVAL, "nin_values %d out of range", d->nin_values);
	for (int l = 0; l < d->nin_lists; l++)
	{
		const CgInList &L = d->in_lists[l];
		if (L.first < 0 || L.nvalues < 0 || L.nnulls < 0) return cg_set_error(CG_EINVAL, "list %d: negative field", l);
		if ((int64_t) L.nvalues + L.nnulls == 0) return cg_set_error(CG_EINVAL, "list %d is empty", l);
		if ((int64_t) L.first + L.nvalues > d->nin_values)
			return cg_set_error(CG_EINVAL, "list %d: values [%d, %lld) beyond nin_values %d", l, L.first, (long long) L.first + L.nvalues, d->nin_values);
	}
	return CG_OK;
}

static inline bool op_is_list(int op) { return op == CG_OP_IN || op == CG_OP_NOT_IN; }

/* the comparison class of a column atom's side: integer-like (int, bool, numeric), char(1) or float */
enum { CMP_INTEGER = 0, CMP_CHAR = 1, CMP_FLOAT = 2 };
static int cmp_class(const CgColumnDesc &c)
{
	const int cls = cg_type_class(c);
	return cls == CG_TYPE_FLOAT ? CMP_FLOAT : cls == CG_TYPE_BPCHAR1 ? CMP_CHAR : CMP_INTEGER;
}

/* column atoms compare two columns of one class (include/citus_gpu.h, CgQual) */
static int validate_column_atoms(const char *what, const CgQual *quals, int n, const CgColumnDesc *columns)
{
	for (int q = 0; q < n; q++)
	{
		if (!cg_op_is_column(quals[q].op)) continue;
		const int a = quals[q].column, b = (int) quals[q].konst;
		if (cmp_class(columns[a]) != cmp_class(columns[b]))
			return cg_set_error(CG_EUNSUPPORTED, "%s %d: columns %d and %d are of different comparison classes", what, q, a, b);
	}
	return CG_OK;
}

std::vector<int64_t> cg_where_lists(const CgScanDesc *d)
{
	std::vector<int64_t> out;
	for (int q = 0; q < d->nquals && q < CG_MAX_QUALS; q++)
	{
		if (!op_is_list(d->quals[q].op) || d->quals[q].konst < 0 || d->quals[q].konst >= d->nin_lists || d->nin_lists > CG_MAX_IN_LISTS) continue;
		const CgInList &L = d->in_lists[d->quals[q].konst];
		out.push_back(q); out.push_back(L.nvalues); out.push_back(L.nnulls);
		for (int i = 0; i < L.nvalues && L.first + i < CG_MAX_IN_VALUES; i++) out.push_back(d->in_values[L.first + i]);
	}
	return out;
}

/* the columns of an aggregate argument's factors, under the rules of the aggregate's kind */
static int validate_factor_columns(int a, int kind, bool is_float, const int32_t *column, int nfactors, const CgColumnDesc *columns, int natts)
{
	for (int f = 0; f < nfactors; f++)
	{
		if (column[f] < 0 || column[f] >= natts) return cg_set_error(CG_EINVAL, "aggregate %d: column out of range", a);
		const int cls = cg_type_class(columns[column[f]]);
		if (kind == CG_AGG_VARIANCE)
		{
			/* the exact integer state of numeric_stddev_internal: a float argument has no such state */
			if (cls == CG_TYPE_BPCHAR1) return cg_set_error(CG_EINVAL, "aggregate %d: variance over a char(1) column", a);
			if (is_float || cls == CG_TYPE_FLOAT) return cg_set_error(CG_EUNSUPPORTED, "aggregate %d: variance / stddev of a float argument", a);
		}
		else if (kind != CG_AGG_COUNT && (cls == CG_TYPE_FLOAT) != is_float)
			return cg_set_error(CG_EINVAL, "aggregate %d: integer/float mismatch with column %d", a, column[f]);
	}
	return CG_OK;
}

/* CASE arguments (CgScanDesc.case_arms; include/citus_gpu.h states the rules) */
static int validate_case(const CgScanDesc *d, const CgColumnDesc *columns, int natts)
{
	if (d->ncase_arms < 0 || d->ncase_arms > CG_MAX_CASE_ARMS) return cg_set_error(CG_EINVAL, "ncase_arms %d out of range", d->ncase_arms);
	for (int a = 0; a < CG_MAX_AGGS; a++)
	{
		const int n = d->case_narms[a], first = d->case_first[a];
		if (n < 0) return cg_set_error(CG_EINVAL, "case_narms[%d] = %d", a, n);
		if (n == 0) continue;
		if (a >= d->naggs) return cg_set_error(CG_EINVAL, "CASE of aggregate %d of %d", a, d->naggs);
		const CgAggSpec &s = d->aggs[a];
		if (s.kind != CG_AGG_COUNT && s.kind != CG_AGG_SUM && s.kind != CG_AGG_MIN && s.kind != CG_AGG_MAX && s.kind != CG_AGG_VARIANCE)
			return cg_set_error(CG_EINVAL, "aggregate %d: a CASE argument on a kind that takes none", a);
		if (s.nfactors != 0) return cg_set_error(CG_EINVAL, "aggregate %d: a CASE argument with factors (the arms carry the terms)", a);
		if (first < 0 || (int64_t) first + n > d->ncase_arms)
			return cg_set_error(CG_EINVAL, "aggregate %d: arms [%d, %lld) outside [0, %d)", a, first, (long long) first + n, d->ncase_arms);
		for (int i = first; i < first + n; i++)
		{
			const CgCaseArm &A = d->case_arms[i];
			int rc;
			if (A.nwhen < 0 || A.nwhen > CG_MAX_QEXPR) return cg_set_error(CG_EINVAL, "arm %d: nwhen %d out of range", i, A.nwhen);
			if (A.nwhen == 0 && i != first + n - 1) return cg_set_error(CG_EINVAL, "aggregate %d: the ELSE arm %d is not its last arm", a, i);
			if (A.nwhen > 0 && (rc = validate_postfix("CASE WHEN tree", A.when, A.nwhen, d->nfilter_quals))) return rc;
			if (A.form != CG_CASE_NULL && A.form != CG_CASE_CONST && A.form != CG_CASE_PRODUCT)
				return cg_set_error(CG_EINVAL, "arm %d: bad result form %d", i, A.form);
			if (A.form != CG_CASE_PRODUCT) continue;
			if (A.nfactors < 1 || A.nfactors > 3) return cg_set_error(CG_EINVAL, "arm %d: nfactors %d", i, A.nfactors);
			if ((rc = validate_factor_columns(a, s.kind, s.is_float != 0, A.column, A.nfactors, columns, natts))) return rc;
		}
		if (s.kind == CG_AGG_VARIANCE && s.is_float) return cg_set_error(CG_EUNSUPPORTED, "aggregate %d: variance / stddev of a float argument", a);
	}
	return CG_OK;
}

static int validate_desc(const CgScanDesc *d, const CgColumnDesc *columns, int natts)
{
	if (d->nquals < 0 || d->nquals > CG_MAX_QUALS) return cg_set_error(CG_EINVAL, "nquals %d out of range", d->nquals);
	if (d->naggs < 0 || d->naggs > CG_MAX_AGGS) return cg_set_error(CG_EINVAL, "naggs %d out of range", d->naggs);
	if (d->composite_key != 0 && d->composite_key != 1) return cg_set_error(CG_EINVAL, "composite_key %d", d->composite_key);
	/* the packed key form holds at most two columns */
	if (d->ngroup_cols < (d->composite_key ? 1 : 0) || d->ngroup_cols > (d->composite_key ? CG_MAX_GROUP_COLS : 2))
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
	int rc = validate_lists(d);
	if (rc) return rc;
	if ((rc = validate_atoms("qual", d->quals, d->nquals, natts, d->nin_lists))) return rc;
	if ((rc = validate_column_atoms("qual", d->quals, d->nquals, columns))) return rc;
	if (d->nqual_expr < 0 || d->nqual_expr > CG_MAX_QEXPR) return cg_set_error(CG_EINVAL, "nqual_expr %d out of range", d->nqual_expr);
	if (d->nqual_expr > 0 && (rc = validate_postfix("qual_expr", d->qual_expr, d->nqual_expr, d->nquals))) return rc;
	if (d->nfilter_quals < 0 || d->nfilter_quals > CG_MAX_FILTER_QUALS)
		return cg_set_error(CG_EINVAL, "nfilter_quals %d out of range", d->nfilter_quals);
	if ((rc = validate_atoms("filter qual", d->filter_quals, d->nfilter_quals, natts, d->nin_lists))) return rc;
	if ((rc = validate_column_atoms("filter qual", d->filter_quals, d->nfilter_quals, columns))) return rc;
	for (int a = 0; a < CG_MAX_AGGS; a++)
	{
		const int n = d->nfilter_expr[a];
		if (n < 0 || n > CG_MAX_QEXPR) return cg_set_error(CG_EINVAL, "nfilter_expr[%d] = %d out of range", a, n);
		if (n > 0 && a >= d->naggs) return cg_set_error(CG_EINVAL, "filter of aggregate %d of %d", a, d->naggs);
		if (n > 0 && (rc = validate_postfix("filter_expr", d->filter_expr[a], n, d->nfilter_quals))) return rc;
		/* predicate arguments: only bool_and / bool_or have one, and they must (checked with the aggregates below) */
		const int m = d->narg_expr[a];
		if (m == 0) continue;
		if (a >= d->naggs || !cg_kind_is_bool(d->aggs[a].kind)) return cg_set_error(CG_EINVAL, "predicate argument on aggregate %d, which takes none", a);
		if (m < 0 || m > CG_MAX_QEXPR) return cg_set_error(CG_EINVAL, "narg_expr[%d] = %d out of range", a, m);
		if ((rc = validate_postfix("arg_expr", d->arg_expr[a], m, d->nfilter_quals))) return rc;
	}
	for (int g = 0; g < d->ngroup_cols; g++)
	{
		int c = d->group_cols[g];
		if (c < 0 || c >= natts) return cg_set_error(CG_EINVAL, "group column %d out of range", c);
		if (columns[c].type_class == CG_TYPE_FLOAT)
			return cg_set_error(CG_EUNSUPPORTED, "GROUP BY on a float column");
		if (!d->composite_key && d->ngroup_cols == 2 && cg_decoded_len(columns[c]) > 4)
			return cg_set_error(CG_EUNSUPPORTED, "two-column GROUP BY needs columns of at most 4 bytes");
	}
	if ((rc = validate_case(d, columns, natts))) return rc;
	for (int a = 0; a < d->naggs; a++)
	{
		const CgAggSpec &s = d->aggs[a];
		if (s.kind < CG_AGG_COUNT_STAR || s.kind > CG_AGG_VARIANCE) return cg_set_error(CG_EINVAL, "aggregate %d: bad kind", a);
		if (s.nfactors < 0 || s.nfactors > 3) return cg_set_error(CG_EINVAL, "aggregate %d: nfactors", a);
		if (d->case_narms[a] > 0) continue;     /* the arms carry the argument (validate_case) */
		if (s.kind > CG_AGG_MAX && s.kind != CG_AGG_VARIANCE && s.term_abs_bound != 0)
			return cg_set_error(CG_EINVAL, "aggregate %d: term_abs_bound on bit / bool kind", a);
		if (s.kind == CG_AGG_VARIANCE)
		{
			/* the exact integer state of numeric_stddev_internal: a float argument has no such state */
			if (s.nfactors < 1) return cg_set_error(CG_EINVAL, "aggregate %d needs an argument", a);
			for (int f = 0; f < s.nfactors; f++)
			{
				if (s.column[f] < 0 || s.column[f] >= natts) return cg_set_error(CG_EINVAL, "aggregate %d: column out of range", a);
				if (cg_type_class(columns[s.column[f]]) == CG_TYPE_BPCHAR1)
					return cg_set_error(CG_EINVAL, "aggregate %d: variance over a char(1) column", a);
				if (s.is_float || cg_type_class(columns[s.column[f]]) == CG_TYPE_FLOAT)
					return cg_set_error(CG_EUNSUPPORTED, "aggregate %d: variance / stddev of a float argument", a);
			}
			continue;
		}
		if (cg_kind_is_bool(s.kind))
		{
			/* the argument is a predicate tree, not factors */
			if (s.nfactors != 0) return cg_set_error(CG_EINVAL, "aggregate %d: bool_and / bool_or with factors", a);
			if (d->narg_expr[a] < 1) return cg_set_error(CG_EINVAL, "aggregate %d: bool_and / bool_or without a predicate argument", a);
			continue;
		}
		if (cg_kind_is_bit(s.kind))
		{
			/* one bare integer column: bitwise ops on the sign-extended words are exact for every width */
			if (s.nfactors != 1 || s.a[0] != 0 || s.b[0] != 1 || s.is_float)
				return cg_set_error(CG_EINVAL, "aggregate %d: bit_and / bit_or take one bare integer column", a);
			if (s.column[0] < 0 || s.column[0] >= natts) return cg_set_error(CG_EINVAL, "aggregate %d: column out of range", a);
			if (columns[s.column[0]].type_class != CG_TYPE_INT)
				return cg_set_error(CG_EINVAL, "aggregate %d: bit_and / bit_or over a column that is not an integer type", a);
			continue;
		}
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
 * The composite group key codec (CgScanDesc.composite_key; include/citus_gpu.h states the code).  This block is the only
 * code that knows it: the kernels receive kmin / kradix per column and compute the digits the same way, everything behind
 * them sees a one-column key over [0, D).  A column of bounds [lo, hi] has hi - lo + 1 values plus NULL (digit 0); an
 * all-NULL column (lo > hi) has NULL only.  D is computed in 128 bits: K radixes of up to 2^64 + 1 each.
 */
int cg_key_codec(const CgScanDesc *d, uint64_t *radix, unsigned __int128 *domain)
{
	if (!d->composite_key) return cg_set_error(CG_EINVAL, "the descriptor has no composite key");
	const int K = d->ngroup_cols;
	if (K < 1 || K > CG_MAX_GROUP_COLS) return cg_set_error(CG_EINVAL, "composite key over %d columns", K);
	const unsigned __int128 limit = (unsigned __int128) 1 << 63;
	unsigned __int128 D = 1;
	for (int g = 0; g < K; g++)
	{
		const int64_t lo = d->key_col_min[g], hi = d->key_col_max[g];
		const unsigned __int128 r = lo > hi ? 1 : (unsigned __int128) ((__int128) hi - (__int128) lo) + 2;
		D *= r;                       /* D <= 2^63 before, r <= 2^64 + 1: no 128-bit overflow */
		if (D > limit) return cg_set_error(CG_EUNSUPPORTED, "composite key domain exceeds 2^63 (column %d: [%lld, %lld])", g, (long long) lo, (long long) hi);
		radix[g] = (uint64_t) r;
	}
	*domain = D;
	return CG_OK;
}

uint64_t cg_key_codec_id(const CgScanDesc *d)
{
	if (!d->composite_key) return 0;
	/* FNV-1a over the column count and the bounds */
	uint64_t h = 0xcbf29ce484222325ull;
	auto mix = [&](uint64_t x) { for (int i = 0; i < 8; i++) { h ^= (x >> (8 * i)) & 0xff; h *= 0x100000001b3ull; } };
	mix((uint64_t) d->ngroup_cols);
	for (int g = 0; g < d->ngroup_cols && g < CG_MAX_GROUP_COLS; g++) { mix((uint64_t) d->key_col_min[g]); mix((uint64_t) d->key_col_max[g]); }
	return h | 1;                     /* never 0, the value of the other key forms */
}

extern "C" int cg_group_key_encode(const CgScanDesc *desc, int64_t n, const int64_t *values, const uint8_t *nulls, int64_t *codes)
{
	if (!desc || n < 0 || (n > 0 && (!values || !codes))) return cg_set_error(CG_EINVAL, "NULL argument");
	uint64_t radix[CG_MAX_GROUP_COLS];
	unsigned __int128 D;
	int rc = cg_key_codec(desc, radix, &D);
	if (rc) return rc;
	const int K = desc->ngroup_cols;
	for (int64_t i = 0; i < n; i++)
	{
		uint64_t code = 0;
		for (int g = 0; g < K; g++)
		{
			uint64_t digit = 0;
			if (!(nulls && nulls[i * K + g]))
			{
				const int64_t v = values[i * K + g];
				if (v < desc->key_col_min[g] || v > desc->key_col_max[g])
					return cg_set_error(CG_EINVAL, "row %lld: key column %d value %lld outside [%lld, %lld]", (long long) i, g, (long long) v,
										(long long) desc->key_col_min[g], (long long) desc->key_col_max[g]);
				digit = (uint64_t) v - (uint64_t) desc->key_col_min[g] + 1;
			}
			code = code * radix[g] + digit;     /* < D <= 2^63 */
		}
		codes[i] = (int64_t) code;
	}
	return CG_OK;
}

extern "C" int cg_group_key_decode(const CgScanDesc *desc, int64_t n, const int64_t *codes, int64_t *values, uint8_t *nulls)
{
	if (!desc || n < 0 || (n > 0 && (!codes || !values || !nulls))) return cg_set_error(CG_EINVAL, "NULL argument");
	uint64_t radix[CG_MAX_GROUP_COLS];
	unsigned __int128 D;
	int rc = cg_key_codec(desc, radix, &D);
	if (rc) return rc;
	const int K = desc->ngroup_cols;
	for (int64_t i = 0; i < n; i++)
	{
		if (codes[i] < 0 || (unsigned __int128) codes[i] >= D)
			return cg_set_error(CG_EINVAL, "row %lld: code %lld outside the key domain", (long long) i, (long long) codes[i]);
		uint64_t c = (uint64_t) codes[i];
		for (int g = K - 1; g >= 0; g--)
		{
			const uint64_t digit = c % radix[g];
			c /= radix[g];
			nulls[i * K + g] = digit == 0;
			values[i * K + g] = digit == 0 ? 0 : (int64_t) ((uint64_t) desc->key_col_min[g] + digit - 1);
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
 *   bit_and/or    1 AND/OR word (identity ~0 / 0) over the sign-extended values + NULL-input count
 *   bool_and/or   1 AND/OR word whose bit 0 is the result (a TRUE input contributes ~0, a FALSE one 0, so TRUE is the
 *                 identity of bool_and and FALSE that of bool_or) + a count of the rows that gave no input (UNKNOWN)
 *   variance      sum(x) in sum's one-word or two-limb form under sum's rule; then sum(x^2) in ADD words:
 *                   1 word    when B^2 * max_rows < 2^63 (B = term_abs_bound)
 *                   2 limbs   (x^2 low 32 bits, x^2 >> 32) when B < 2^32
 *                   4 limbs   the four 32-bit limbs of the unsigned 128-bit x^2 (x = INT64_MIN gives 2^126)
 *                 + NULL-input count: 3 to 7 words.  Every limb word grows by < 2^32 per row (the merge kernel's carry
 *                 chain keeps it so for merged rows: limb l's carry goes to limb l + 1)
 * Counting the NULL inputs instead of the non-NULL ones keeps NULL-free data (the common
 * case) at one atomic per aggregate and row, while "no non-NULL input => SQL NULL" and
 * count(x) stay exact: non-NULL inputs = rows in group - NULL inputs.
 * An aggregate with a FILTER counts in that word every row that gave no input (NULL input or
 * filter not TRUE); a filtered count(*) gets one such ADD word (count = rows - it).  Every
 * word stays additive or min/max, so combines and merges need not know about filters.
 */
static int layout_partial(CgPartial *p, const CgColumnDesc *columns)
{
	const CgScanDesc &d = p->desc;
	int nw = 1;
	memset(p->wordop, CG_WORD_ADD, sizeof p->wordop);
	/* appends one word; past CG_KMAX_WORDS it only counts (the aggregate list is refused below, nothing is written) */
	auto push = [&](int op) {
		if (nw < CG_KMAX_WORDS) p->wordop[nw] = (uint8_t) op;
		nw++;
	};
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
		k.tbound = (cg_kind_sums(s.kind) && !s.is_float && s.term_abs_bound > 0) ? s.term_abs_bound : 0;
		/* an integer argument other than a bare column can leave int64 ([PG] int8mul / int8pl raise "bigint out of
		 * range", numeric is exact): unless the caller proved a bound, the kernels check every factor and product */
		k.ovchk = (int8_t) (!s.is_float && (cg_kind_sums(s.kind) || s.kind == CG_AGG_MIN || s.kind == CG_AGG_MAX) &&
							k.tbound == 0 && !(s.nfactors == 1 && s.a[0] == 0 && s.b[0] == 1));
		k.filt = (int8_t) (d.nfilter_expr[a] > 0);
		k.barg = (int8_t) cg_kind_is_bool(s.kind);
		switch (s.kind)
		{
			case CG_AGG_BIT_AND:
			case CG_AGG_BIT_OR:
			case CG_AGG_BOOL_AND:
			case CG_AGG_BOOL_OR:
				k.word0 = (int8_t) nw;
				push((s.kind == CG_AGG_BIT_AND || s.kind == CG_AGG_BOOL_AND) ? CG_WORD_AND : CG_WORD_OR);
				k.nullword = (int8_t) nw; push(CG_WORD_ADD);
				break;
			case CG_AGG_COUNT_STAR:
				k.word0 = 0;
				if (k.filt) { k.nullword = (int8_t) nw; push(CG_WORD_ADD); }
				break;
			case CG_AGG_COUNT:
				k.word0 = (int8_t) nw; k.nullword = (int8_t) nw; push(CG_WORD_ADD);
				break;
			case CG_AGG_VARIANCE:
			{
				/* sum(x): sum's words under sum's rule */
				k.word0 = (int8_t) nw;
				push(CG_WORD_ADD);
				const __int128 B = s.term_abs_bound, R = p->max_rows;
				if (B > 0 && R > 0 && B * R < ((__int128) 1 << 63)) { k.nlimbs = 1; k.bound = s.term_abs_bound; }
				else { k.nlimbs = 2; push(CG_WORD_ADD); if (B > 0) k.bound = s.term_abs_bound; }
				/* sum(x^2): every limb word grows by < 2^32 per row, so 2^32 rows per group never wrap one */
				k.qword = (int8_t) nw;
				if (B > 0 && R > 0 && B < ((__int128) 1 << 32) && (B * B) * R < ((__int128) 1 << 63)) k.qlimbs = 1;
				else if (B > 0 && B < ((__int128) 1 << 32)) k.qlimbs = 2;
				else k.qlimbs = 4;
				for (int l = 0; l < k.qlimbs; l++) push(CG_WORD_ADD);
				k.nullword = (int8_t) nw; push(CG_WORD_ADD);
				break;
			}
			case CG_AGG_SUM:
				k.word0 = (int8_t) nw;
				if (s.is_float) push(CG_WORD_FADD);
				else
				{
					push(CG_WORD_ADD);
					bool one = false;
					if (s.term_abs_bound > 0 && p->max_rows > 0)
					{
						__int128 worst = (__int128) s.term_abs_bound * (__int128) p->max_rows;
						one = worst < ((__int128) 1 << 63);
					}
					if (one) { k.nlimbs = 1; k.bound = s.term_abs_bound; }
					else { k.nlimbs = 2; push(CG_WORD_ADD); }
				}
				k.nullword = (int8_t) nw; push(CG_WORD_ADD);
				break;
			default:
				k.word0 = (int8_t) nw;
				if (s.kind == CG_AGG_MIN) push(s.is_float ? CG_WORD_FMIN : CG_WORD_MIN);
				else push(s.is_float ? CG_WORD_FMAX : CG_WORD_MAX);
				k.nullword = (int8_t) nw; push(CG_WORD_ADD);
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
	if (desc->composite_key)
	{
		/* a one-column key over the codes [0, D): key_min / key_max are not used */
		uint64_t radix[CG_MAX_GROUP_COLS];
		unsigned __int128 D;
		if ((rc = cg_key_codec(desc, radix, &D))) return rc;
		key_min = 0;
		key_max = (int64_t) (D - 1);
	}
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
	else if (desc->ngroup_cols == 2 && !desc->composite_key &&
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
	else if ((desc->ngroup_cols == 1 || desc->composite_key) && key_min <= key_max && ((uint64_t) key_max - (uint64_t) key_min) < kDenseLimit)
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
	p->sets.release();
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

/* aggregate a has the same CASE argument in both descriptors (both validated): the same arms in the same order, compared
 * field by field (the arms' positions in case_arms may differ) */
static bool same_case(const CgScanDesc *x, const CgScanDesc *y, int a)
{
	if (x->case_narms[a] != y->case_narms[a]) return false;
	for (int i = 0; i < x->case_narms[a]; i++)
	{
		const CgCaseArm &p = x->case_arms[x->case_first[a] + i], &q = y->case_arms[y->case_first[a] + i];
		if (p.nwhen != q.nwhen || memcmp(p.when, q.when, (size_t) p.nwhen) != 0 || p.form != q.form) return false;
		if (p.form == CG_CASE_CONST && p.a[0] != q.a[0]) return false;
		if (p.form != CG_CASE_PRODUCT) continue;
		if (p.nfactors != q.nfactors) return false;
		for (int f = 0; f < p.nfactors; f++)
			if (p.column[f] != q.column[f] || p.a[f] != q.a[f] || p.b[f] != q.b[f]) return false;
	}
	return true;
}

/*
 * Kernel plan: deduplicated projection (columnar_customscan.c:1813-1851 ColumnarAttrNeeded:
 * only the columns the quals, group keys and aggregate arguments reference are read).  Plan columns are numbered in first
 * use: the WHERE atoms' columns first, so the WHERE half (where()) is the same for an aggregate scan and a row scan.
 */
struct PlanBuilder
{
	const CgScanDesc *desc;
	const CgColumnDesc *columns;
	int natts;
	const std::vector<int32_t> *slot_of_att;
	KPlan *plan;
	int pcol_of_att[256];
	int ncols = 0;
	/* IN / NOT IN lists: every list's codes once per kind (integer / float), back to back */
	std::vector<uint64_t> codes;
	int list_at[CG_MAX_IN_LISTS][2];

	PlanBuilder(const CgScanDesc *d, const CgColumnDesc *c, int n, const std::vector<int32_t> *s, KPlan *p)
		: desc(d), columns(c), natts(n), slot_of_att(s), plan(p)
	{
		memset(plan, 0, sizeof *plan);
		for (int i = 0; i < 256; i++) pcol_of_att[i] = -1;
		for (int l = 0; l < CG_MAX_IN_LISTS; l++) list_at[l][0] = list_at[l][1] = -1;
	}

	/* the plan column of attribute att, added on first use */
	int use(int att, int *pc)
	{
		if (pcol_of_att[att] >= 0) { *pc = pcol_of_att[att]; return CG_OK; }
		if (ncols == CG_KMAX_COLS) return cg_set_error(CG_EUNSUPPORTED, "query reads more than %d columns", CG_KMAX_COLS);
		int slot = slot_of_att ? (*slot_of_att)[att] : att;
		if (slot < 0) return cg_set_error(CG_EINVAL, "column %d is not staged in this shard", att);
		plan->slot[ncols] = (uint8_t) slot;
		plan->len[ncols] = (uint8_t) cg_decoded_len(columns[att]);       /* a varlena column reaches the kernels decoded to a fixed width */
		plan->isfloat[ncols] = (uint8_t) (columns[att].type_class == CG_TYPE_FLOAT);
		pcol_of_att[att] = ncols;
		*pc = ncols++;
		return CG_OK;
	}

	/* integer atoms in range form: pass iff ((x >= lo && x <= hi) != neg); float atoms keep op + constant (a float4
	 * column's values are promoted to float8, the constant already is float8 bits) */
	static void atom_range(const CgQual &q, int64_t *lo_out, int64_t *hi_out, uint8_t *neg_out)
	{
		int64_t k = q.konst, lo = INT64_MIN, hi = INT64_MAX;
		bool neg = false;
		if (cg_op_is_column(q.op)) { *lo_out = *hi_out = 0; *neg_out = 0; return; }     /* no constant: KCmp instead */
		switch (q.op)
		{
			case CG_OP_LT: if (k == INT64_MIN) { lo = 1; hi = 0; } else hi = k - 1; break;
			case CG_OP_LE: hi = k; break;
			case CG_OP_EQ: lo = hi = k; break;
			case CG_OP_GE: lo = k; break;
			case CG_OP_GT: if (k == INT64_MAX) { lo = 1; hi = 0; } else lo = k + 1; break;
			default: lo = hi = k; neg = true; break;
		}
		*lo_out = lo; *hi_out = hi; *neg_out = neg;
	}

	/* IN / NOT IN lists: each atom's list as sorted, distinct codes in its column's order (cg_set_code); the atoms of one
	 * list on columns of one kind (integer / float) share them.  A list of NULLs only has no code (len 0): no row is found
	 * in it, and nnull decides. */
	void set_of(const CgQual &q, bool isfloat, KSet *ks)
	{
		memset(ks, 0, sizeof *ks);
		if (!op_is_list(q.op)) return;
		const CgInList &L = desc->in_lists[q.konst];
		int &at = list_at[q.konst][isfloat];
		std::vector<uint64_t> c;
		for (int i = 0; i < L.nvalues; i++) c.push_back(cg_set_code(desc->in_values[L.first + i], isfloat));
		std::sort(c.begin(), c.end());
		c.erase(std::unique(c.begin(), c.end()), c.end());
		if (at < 0)
		{
			at = (int) codes.size();
			codes.insert(codes.end(), c.begin(), c.end());
		}
		ks->off = (uint16_t) at;
		ks->len = (uint16_t) c.size();
		int steps = 0;
		while ((1u << steps) < c.size()) steps++;
		ks->steps = (uint8_t) steps;
		ks->nnull = (uint8_t) (L.nnulls > 0);
	}

	/* column atoms: the other column is a plan column too; integer-like sides of different scales align on the larger one */
	int cmp_of(const CgQual &q, KCmp *kc)
	{
		memset(kc, 0, sizeof *kc);
		kc->mul = 1;
		if (!cg_op_is_column(q.op)) return CG_OK;
		int pc = 0, rc;
		if ((rc = use((int) q.konst, &pc))) return rc;
		kc->col2 = (uint8_t) pc;
		const CgColumnDesc &x = columns[q.column], &y = columns[q.konst];
		if (cmp_class(x) != CMP_INTEGER) return CG_OK;
		const int sx = cg_type_class(x) == CG_TYPE_NUMERIC ? cg_type_scale(x) : 0;
		const int sy = cg_type_class(y) == CG_TYPE_NUMERIC ? cg_type_scale(y) : 0;
		kc->right = (uint8_t) (sx > sy);
		for (int i = 0; i < (sx > sy ? sx - sy : sy - sx); i++) kc->mul *= 10;      /* <= 10^18 */
		return CG_OK;
	}

	/* the WHERE half: atoms, lists, column atoms and the tree */
	int where()
	{
		int rc;
		plan->nquals = desc->nquals;
		for (int q = 0; q < desc->nquals; q++)
		{
			int pc = 0;
			if ((rc = use(desc->quals[q].column, &pc))) return rc;
			plan->qcol[q] = (uint8_t) pc;
			plan->qop[q] = (uint8_t) desc->quals[q].op;
			plan->qk[q] = desc->quals[q].konst;
			atom_range(desc->quals[q], &plan->qlo[q], &plan->qhi[q], &plan->qneg[q]);
			set_of(desc->quals[q], plan->isfloat[pc], &plan->qset[q]);
			if ((rc = cmp_of(desc->quals[q], &plan->qcc[q]))) return rc;
		}
		plan->slices = 1; plan->slice_rows = 1u << 30; plan->max_cg_rows = 0;
		plan->nqexpr = desc->nqual_expr;
		for (int i = 0; i < desc->nqual_expr; i++) plan->qexpr[i] = desc->qual_expr[i];
		return CG_OK;
	}

	/* the plan columns and the list codes (KPlan.sets is left NULL for the caller to point at their device copy) */
	void finish(std::vector<uint64_t> *set_codes, bool *all8)
	{
		plan->sets = nullptr;
		if (set_codes) set_codes->swap(codes);
		plan->ncols = ncols;
		bool a8 = true;
		for (int c = 0; c < ncols; c++) if (plan->len[c] != 8) a8 = false;
		*all8 = a8;
	}
};

int cg_build_where_plan(const CgScanDesc *desc, const CgColumnDesc *columns, int natts, const std::vector<int32_t> *slot_of_att,
						KPlan *plan, std::vector<uint64_t> *set_codes)
{
	if (desc->naggs != 0 || desc->ngroup_cols != 0 || desc->composite_key != 0 || cg_desc_uses_pool(desc) || desc->ncase_arms != 0)
		return cg_set_error(CG_EINVAL, "a row scan takes a WHERE tree only: no aggregates, group columns, FILTER, CASE or composite key");
	int rc = validate_desc(desc, columns, natts);
	if (rc) return rc;
	if (natts > 256) return cg_set_error(CG_EUNSUPPORTED, "more than 256 attributes");
	PlanBuilder b(desc, columns, natts, slot_of_att, plan);
	if ((rc = b.where())) return rc;
	bool all8;
	b.finish(set_codes, &all8);
	return CG_OK;
}

int cg_build_plan(const CgScanDesc *desc, const CgColumnDesc *columns, int natts,
				  const std::vector<int32_t> *slot_of_att, CgPartial *partial, KPlan *plan, bool *all8,
				  std::vector<uint64_t> *set_codes)
{
	int rc = validate_desc(desc, columns, natts);
	if (rc) return rc;
	/* the partial must have been created for the same aggregate list */
	if (partial->desc.naggs != desc->naggs || partial->desc.ngroup_cols != desc->ngroup_cols)
		return cg_set_error(CG_EINVAL, "partial aggregate was created for a different query shape");
	for (int a = 0; a < desc->naggs; a++)
		if (memcmp(&partial->desc.aggs[a], &desc->aggs[a], sizeof(CgAggSpec)) != 0 || partial->aggs[a].filt != (desc->nfilter_expr[a] > 0) ||
			partial->desc.narg_expr[a] != desc->narg_expr[a] ||
			memcmp(partial->desc.arg_expr[a], desc->arg_expr[a], (size_t) desc->narg_expr[a]) != 0 || !same_case(&partial->desc, desc, a))
			return cg_set_error(CG_EINVAL, "partial aggregate was created for a different aggregate list");
	/* a composite partial's codes mean something only under its own key columns and bounds */
	if (partial->desc.composite_key != desc->composite_key)
		return cg_set_error(CG_EINVAL, "partial aggregate was created for a different group key form");
	if (desc->composite_key)
		for (int g = 0; g < desc->ngroup_cols; g++)
			if (partial->desc.group_cols[g] != desc->group_cols[g] || partial->desc.key_col_min[g] != desc->key_col_min[g] ||
				partial->desc.key_col_max[g] != desc->key_col_max[g])
				return cg_set_error(CG_EINVAL, "partial aggregate was created for other composite key columns or bounds (column %d)", g);

	if (natts > 256) { memset(plan, 0, sizeof *plan); return cg_set_error(CG_EUNSUPPORTED, "more than 256 attributes"); }
	PlanBuilder b(desc, columns, natts, slot_of_att, plan);
	if ((rc = b.where())) return rc;
	plan->ngroup = desc->ngroup_cols;
	for (int g = 0; g < desc->ngroup_cols; g++)
	{
		int pc = 0;
		if ((rc = b.use(desc->group_cols[g], &pc))) return rc;
		plan->gcol[g] = (uint8_t) pc;
	}
	if (desc->composite_key)
	{
		unsigned __int128 D;
		if ((rc = cg_key_codec(desc, plan->kradix, &D))) return rc;
		plan->composite = 1;
		for (int g = 0; g < desc->ngroup_cols; g++) plan->kmin[g] = desc->key_col_min[g];
	}
	plan->naggs = desc->naggs;
	for (int a = 0; a < desc->naggs; a++)
	{
		plan->aggs[a] = partial->aggs[a];
		for (int f = 0; f < desc->aggs[a].nfactors; f++)
		{
			int pc = 0;
			if ((rc = b.use(desc->aggs[a].column[f], &pc))) return rc;
			plan->aggs[a].pcol[f] = (int8_t) pc;
		}
	}
	if (cg_desc_has_case(desc))
	{
		/* the arms the aggregates name (validate_case checked them), their factor columns as plan columns */
		bool done[CG_MAX_CASE_ARMS] = {false};
		plan->ncase = desc->ncase_arms;
		for (int a = 0; a < desc->naggs; a++)
		{
			plan->cfirst[a] = (int8_t) desc->case_first[a];
			plan->cnarms[a] = (int8_t) desc->case_narms[a];
			for (int i = desc->case_first[a]; i < desc->case_first[a] + desc->case_narms[a]; i++)
			{
				if (done[i]) continue;
				done[i] = true;
				const CgCaseArm &A = desc->case_arms[i];
				KArm &k = plan->arms[i];
				k.nwhen = (int8_t) A.nwhen;
				for (int t = 0; t < A.nwhen; t++) k.when[t] = A.when[t];
				k.form = (int8_t) A.form;
				k.a[0] = A.a[0];
				if (A.form != CG_CASE_PRODUCT) continue;
				k.nfactors = (int8_t) A.nfactors;
				for (int f = 0; f < A.nfactors; f++)
				{
					int pc = 0;
					if ((rc = b.use(A.column[f], &pc))) return rc;
					k.pcol[f] = (int8_t) pc;
					k.a[f] = A.a[f];
					k.b[f] = A.b[f];
				}
			}
		}
	}
	if (cg_desc_uses_pool(desc))
	{
		/* a column read only by a FILTER, a predicate argument or a CASE arm is a plan column like any other (projection,
		 * column limit) */
		plan->nfquals = desc->nfilter_quals;
		for (int q = 0; q < desc->nfilter_quals; q++)
		{
			int pc = 0;
			if ((rc = b.use(desc->filter_quals[q].column, &pc))) return rc;
			plan->fcol[q] = (uint8_t) pc;
			plan->fop[q] = (uint8_t) desc->filter_quals[q].op;
			plan->fk[q] = desc->filter_quals[q].konst;
			PlanBuilder::atom_range(desc->filter_quals[q], &plan->flo[q], &plan->fhi[q], &plan->fneg[q]);
			b.set_of(desc->filter_quals[q], plan->isfloat[pc], &plan->fset[q]);
			if ((rc = b.cmp_of(desc->filter_quals[q], &plan->fcc[q]))) return rc;
		}
		for (int a = 0; a < desc->naggs; a++)
		{
			plan->nfexpr[a] = desc->nfilter_expr[a];
			for (int i = 0; i < desc->nfilter_expr[a]; i++) plan->fexpr[a][i] = desc->filter_expr[a][i];
			plan->nargexpr[a] = desc->narg_expr[a];
			for (int i = 0; i < desc->narg_expr[a]; i++) plan->argexpr[a][i] = desc->arg_expr[a][i];
		}
	}
	b.finish(set_codes, all8);

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
 * point range); at most one group column, not a composite key; aggregates are count(*) and up to three
 * sum(column); every column plays exactly one role.  Anything else runs on the general
 * kernel.  NULLs are handled outside: the fast kernel only sees chunk groups whose plan
 * columns have none.
 */
bool cg_build_fast_plan(const CgScanDesc *desc, const KPlan &plan, bool all8, FPlan *fast)
{
	if (!all8 || plan.ngroup > 1 || plan.composite || plan.nqexpr != 0 || plan.nfquals != 0 || plan.ncase != 0) return false;
	for (int q = 0; q < plan.nquals; q++) if (plan.qop[q] > CG_OP_NE) return false;     /* IN lists, NULL tests, column atoms */
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
