/*
 * cg_device.cuh -- device helpers shared by the scan kernels (cg_scan.cu, cg_scan_small.cu) and the join-aggregate
 * kernel (cg_join.cu).
 */
#ifndef CG_DEVICE_CUH
#define CG_DEVICE_CUH

#include "cg_internal.h"

/* ------------------------------------------------------------------------------ *
 *  streaming loads: read-only path, no L1 allocation (each byte is used once)
 * ------------------------------------------------------------------------------ */
__device__ __forceinline__ void ldg_stream16(const void *p, uint64_t &a, uint64_t &b)
{
	asm("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p));
}
__device__ __forceinline__ uint64_t ldg_stream8(const void *p)
{
	uint64_t a;
	asm("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(a) : "l"(p));
	return a;
}
__device__ __forceinline__ uint32_t ldg_stream4(const void *p)
{
	uint32_t a;
	asm("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(a) : "l"(p));
	return a;
}
__device__ __forceinline__ uint32_t ldg_stream2(const void *p)
{
	uint16_t a;
	asm("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(a) : "l"(p));
	return a;
}
__device__ __forceinline__ uint32_t ldg_stream1(const void *p)
{
	uint32_t a;
	asm("ld.global.nc.L1::no_allocate.u8 %0, [%1];" : "=r"(a) : "l"(p));
	return a;
}

__device__ __forceinline__ int64_t f4_to_f8_bits(uint32_t u)
{
	return __double_as_longlong((double) __uint_as_float(u));
}

/* widen one stored datum (fetch_att for by-value types, columnar_reader.c:1557) */
__device__ __forceinline__ int64_t widen(uint64_t raw, int len, bool isfloat)
{
	switch (len)
	{
		case 8: return (int64_t) raw;
		case 4: return isfloat ? f4_to_f8_bits((uint32_t) raw) : (int64_t) (int32_t) (uint32_t) raw;
		case 2: return (int64_t) (int16_t) (uint16_t) raw;
		default: return (int64_t) (int8_t) (uint8_t) raw;
	}
}

__device__ __forceinline__ int64_t load_scalar(const uint8_t *p, int len, bool isfloat)
{
	switch (len)
	{
		case 8: return (int64_t) ldg_stream8(p);
		case 4: return widen(ldg_stream4(p), 4, isfloat);
		case 2: return widen(ldg_stream2(p), 2, isfloat);
		default: return widen(ldg_stream1(p), 1, isfloat);
	}
}

/* two consecutive rows (r even) of a NULL-free column */
__device__ __forceinline__ void load_pair(const uint8_t *vals, uint32_t r, int len, bool isfloat,
										  int64_t &v0, int64_t &v1)
{
	switch (len)
	{
		case 8:
		{
			uint64_t a, b;
			ldg_stream16(vals + (uint64_t) r * 8, a, b);
			v0 = (int64_t) a; v1 = (int64_t) b;
			break;
		}
		case 4:
		{
			uint64_t a = ldg_stream8(vals + (uint64_t) r * 4);
			v0 = widen(a & 0xffffffffu, 4, isfloat); v1 = widen(a >> 32, 4, isfloat);
			break;
		}
		case 2:
		{
			uint32_t a = ldg_stream4(vals + (uint64_t) r * 2);
			v0 = widen(a & 0xffffu, 2, false); v1 = widen(a >> 16, 2, false);
			break;
		}
		default:
		{
			uint32_t a = ldg_stream2(vals + r);
			v0 = widen(a & 0xffu, 1, false); v1 = widen(a >> 8, 1, false);
			break;
		}
	}
}

/* two consecutive rows (r even, r + 1 may be past `rows`) of column c, which has NULLs: row -> value index through
 * the exists bitmap and the rank directory (rank[b] = set exists bits before row 64 b; NULL rows occupy no bytes in
 * the value stream, columnar_reader.c:1550-1555).  A NULL row reads 0 and sets bit c of n0 / n1. */
__device__ __forceinline__ void load_pair_nullable(const uint8_t *vals, const uint64_t *exists, const uint32_t *rank, uint32_t r,
												   uint32_t rows, int len, bool isfloat, int c, int64_t &v0, int64_t &v1,
												   uint32_t &n0, uint32_t &n1)
{
	uint64_t w = ldg_stream8(exists + (r >> 6));
	uint32_t sh = r & 63u;
	uint32_t before = __ldg(rank + (r >> 6)) + __popcll(w & ((1ull << sh) - 1ull));
	uint32_t e0 = (uint32_t) (w >> sh) & 1u, e1 = (uint32_t) (w >> (sh + 1)) & 1u;
	v0 = e0 ? load_scalar(vals + (uint64_t) before * len, len, isfloat) : 0;
	v1 = (e1 && r + 1 < rows) ? load_scalar(vals + (uint64_t) (before + e0) * len, len, isfloat) : 0;
	n0 |= (e0 ^ 1u) << c;
	n1 |= (e1 ^ 1u) << c;
}

template <int N>
__device__ __forceinline__ int64_t pick(const int64_t (&v)[N], int idx)
{
	int64_t r = v[0];
#pragma unroll
	for (int c = 1; c < N; c++) r = (idx == c) ? v[c] : r;
	return r;
}

/* [PG] btree comparison result of "v <op> k" (int8 / float8 operators) */
__device__ __forceinline__ bool qual_true(int64_t v, int op, int64_t k, bool isfloat)
{
	if (isfloat)
	{
		double x = __longlong_as_double(v), y = __longlong_as_double(k);
		/* float8 btree order: NaN equals NaN and is greater than everything */
		bool xn = x != x, yn = y != y;
		int c = (xn || yn) ? ((int) xn - (int) yn) : ((x > y) - (x < y));
		switch (op)
		{
			case CG_OP_LT: return c < 0;
			case CG_OP_LE: return c <= 0;
			case CG_OP_EQ: return c == 0;
			case CG_OP_GE: return c >= 0;
			case CG_OP_GT: return c > 0;
			default: return c != 0;
		}
	}
	switch (op)
	{
		case CG_OP_LT: return v < k;
		case CG_OP_LE: return v <= k;
		case CG_OP_EQ: return v == k;
		case CG_OP_GE: return v >= k;
		case CG_OP_GT: return v > k;
		default: return v != k;
	}
}

/* is `key` one of the sorted codes s[0 .. len)?  A branch-free lower bound: exactly `steps` = ceil(log2(len)) halvings, the
 * same for every lane of the warp (the atom's list is uniform), so the search never diverges.  The codes are read through
 * the read-only path with L1 allocation: the column streams bypass L1, so a list of up to 8 KB stays there. */
__device__ __forceinline__ bool set_contains(const uint64_t *s, uint32_t len, uint32_t steps, uint64_t key)
{
	if (len == 0) return false;
	const uint64_t *b = s;
	uint32_t n = len;
#pragma unroll 1
	for (uint32_t i = 0; i < steps; i++)
	{
		const uint32_t h = n >> 1;
		b = (__ldg(b + h) <= key) ? b + h : b;
		n -= h;
	}
	return __ldg(b) == key;
}

/* sign of x * m - y, exact in 128 bits (m > 0) */
__device__ __forceinline__ int cmp_scaled(int64_t x, int64_t m, int64_t y)
{
	const int64_t h = __mul64hi(x, m), yh = y >> 63;
	const uint64_t l = (uint64_t) x * (uint64_t) m;
	return h != yh ? (h < yh ? -1 : 1) : ((l > (uint64_t) y) - (l < (uint64_t) y));
}

/* sign of x - y for a column atom's two sides: integer-like after scale alignment (KCmp), float in float8 btree order
 * (cg_set_code is that order as unsigned) */
__device__ __forceinline__ int col_cmp(int64_t x, int64_t y, bool isfloat, const KCmp &kc)
{
	if (isfloat)
	{
		const uint64_t a = cg_set_code(x, true), b = cg_set_code(y, true);
		return (a > b) - (a < b);
	}
	return kc.right ? -cmp_scaled(y, kc.mul, x) : cmp_scaled(x, kc.mul, y);
}

/*
 * K3: the WHERE tree ([PG] ExecQual under ExecScan, columnar_customscan.c:1907-1913) under three-valued
 * logic: an atom on a NULL input is not TRUE, AND/OR combine "is TRUE" bits (there is no NOT node: it is
 * folded into the comparison operators), the row passes iff the root is TRUE.  Without a tree the atoms
 * are an AND-list.  The list and NULL-test atoms have TRUE and FALSE of their own (include/citus_gpu.h, CgQual):
 * IS [NOT] NULL is never UNKNOWN, and a list with a NULL element makes "not found" UNKNOWN.  A column atom is UNKNOWN
 * when either of its columns is NULL.
 */
template <int NCC>
__device__ __forceinline__ uint32_t eval_atoms(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask, int n, const uint8_t *col,
											   const uint8_t *op, const int64_t *k, const int64_t *lo, const int64_t *hi, const uint8_t *neg,
											   const KSet *ks, const KCmp *kc, uint32_t *falsity = nullptr)
{
	uint32_t truth = 0, fals = 0;
#pragma unroll 1
	for (int q = 0; q < n; q++)
	{
		int c = col[q];
		bool isnull = (nullmask >> c) & 1u;
		int64_t x = pick<NCC>(v, c);
		bool t, f;
		if (op[q] <= CG_OP_NE)
		{
			const bool r = P.isfloat[c] ? qual_true(x, op[q], k[q], true) : (((x >= lo[q]) && (x <= hi[q])) != (bool) neg[q]);
			t = r && !isnull;
			f = !r && !isnull;
		}
		else if (op[q] >= CG_OP_COL_LT)
		{
			const KCmp cc = kc[q];
			const bool known = !isnull && !((nullmask >> cc.col2) & 1u);
			const int s = col_cmp(x, pick<NCC>(v, cc.col2), P.isfloat[c], cc);
			bool r;
			switch (op[q])
			{
				case CG_OP_COL_LT: r = s < 0; break;
				case CG_OP_COL_LE: r = s <= 0; break;
				case CG_OP_COL_EQ: r = s == 0; break;
				case CG_OP_COL_GE: r = s >= 0; break;
				case CG_OP_COL_GT: r = s > 0; break;
				default: r = s != 0; break;
			}
			t = r && known;
			f = !r && known;
		}
		else if (op[q] >= CG_OP_IS_NULL)
		{
			t = isnull == (op[q] == CG_OP_IS_NULL);
			f = !t;
		}
		else
		{
			const KSet s = ks[q];
			const bool found = set_contains(P.sets + s.off, s.len, s.steps, cg_set_code(x, P.isfloat[c]));
			const bool in = op[q] == CG_OP_IN;
			/* IN: found = TRUE, not found = FALSE without NULL elements; NOT IN the other way round; UNKNOWN otherwise */
			t = !isnull && (in ? found : (!found && !s.nnull));
			f = !isnull && (in ? (!found && !s.nnull) : found);
		}
		truth |= (uint32_t) t << q;
		fals |= (uint32_t) f << q;
	}
	if (falsity) *falsity = fals;
	return truth;
}

/* a postfix tree over "is TRUE" bits of atoms.  The second rail of three-valued logic: with `dual` and the "is FALSE"
 * bits, the same tree with AND and OR swapped is "the tree is FALSE" (De Morgan); neither = UNKNOWN */
__device__ __forceinline__ bool eval_postfix(uint32_t truth, int n, const int8_t *expr, bool dual = false)
{
	uint32_t st = 0;
#pragma unroll 1
	for (int i = 0; i < n; i++)
	{
		int t = expr[i];
		if (t >= 0) st = (st << 1) | ((truth >> t) & 1u);
		else
		{
			uint32_t b = st & 1u, a = (st >> 1) & 1u;
			st = ((st >> 2) << 1) | (((t == CG_QX_AND) != dual) ? (a & b) : (a | b));
		}
	}
	return st & 1u;
}

template <int NCC>
__device__ __forceinline__ bool eval_where(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask)
{
	uint32_t truth = eval_atoms<NCC>(P, v, nullmask, P.nquals, P.qcol, P.qop, P.qk, P.qlo, P.qhi, P.qneg, P.qset, P.qcc);
	if (P.nqexpr == 0) return truth == (1u << P.nquals) - 1u;
	return eval_postfix(truth, P.nqexpr, P.qexpr);
}

/* aggregate FILTERs of a row that passed WHERE, same three-valued logic: bit a set = aggregate a has a filter and
 * it is not TRUE, or (bool_and / bool_or) its predicate argument is UNKNOWN, so the row is no input of a.  Bit a of
 * *argtrue = the predicate argument of aggregate a is TRUE.  *pooltruth = the "is TRUE" bits of the pool's atoms (the
 * CASE arms' WHEN trees read them). */
template <int NCC>
__device__ __forceinline__ uint32_t eval_filters(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask, uint32_t *argtrue = nullptr,
												 uint32_t *pooltruth = nullptr)
{
	if (argtrue) *argtrue = 0u;
	if (pooltruth) *pooltruth = 0u;
	if (P.nfquals == 0) return 0u;
	uint32_t fals = 0;
	uint32_t truth = eval_atoms<NCC>(P, v, nullmask, P.nfquals, P.fcol, P.fop, P.fk, P.flo, P.fhi, P.fneg, P.fset, P.fcc, &fals);
	if (pooltruth) *pooltruth = truth;
	uint32_t rejected = 0, at = 0;
#pragma unroll 1
	for (int a = 0; a < P.naggs; a++)
	{
		if (P.nfexpr[a] > 0 && !eval_postfix(truth, P.nfexpr[a], P.fexpr[a])) rejected |= 1u << a;
		if (P.nargexpr[a] > 0)
		{
			const bool t = eval_postfix(truth, P.nargexpr[a], P.argexpr[a]);
			const bool f = eval_postfix(fals, P.nargexpr[a], P.argexpr[a], true);
			if (!t && !f) rejected |= 1u << a;
			at |= (uint32_t) t << a;
		}
	}
	if (argtrue) *argtrue = at;
	return rejected;
}

/* home slot of a key in the open-addressing table: Fibonacci (multiply-shift) hashing, one
 * 64-bit multiply; hash_shift = 64 - log2(capacity).  Every kernel that touches a hash table
 * must use this one function. */
__device__ __forceinline__ uint64_t cg_home_slot(int64_t key, int hash_shift)
{
	return ((uint64_t) key * 0x9E3779B97F4A7C15ull) >> hash_shift;
}

/* order-preserving map of float8 bits to unsigned (for min/max words), in [PG] float8 btree order: every NaN,
 * whatever its sign bit, is the one largest code (above +inf) */
__host__ __device__ __forceinline__ uint64_t f8_ordered(int64_t bits)
{
	uint64_t u = (uint64_t) bits;
	if ((u & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return ~0ull;
	return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

/* int64 multiply / add that set `ovf` when the exact result does not fit */
__device__ __forceinline__ int64_t mul_ovf(int64_t x, int64_t y, bool &ovf)
{
	int64_t lo = (int64_t) ((uint64_t) x * (uint64_t) y);
	ovf |= __mul64hi(x, y) != (lo >> 63);
	return lo;
}
__device__ __forceinline__ int64_t add_ovf(int64_t x, int64_t y, bool &ovf)
{
	int64_t s = (int64_t) ((uint64_t) x + (uint64_t) y);
	ovf |= ((x ^ s) & (y ^ s)) < 0;
	return s;
}

/* integer term prod (a + b*x) of one aggregate; factor f reads column value x[f].  Without a proven bound
 * (g.ovchk) a term that leaves int64 raises CG_ERRFLAG_TERM_OVERFLOW unless an input is NULL */
template <int NCC>
__device__ __forceinline__ int64_t int_term(const KAgg &g, const int64_t (&v)[NCC], bool isnull, unsigned long long *stats)
{
	int64_t it = 1;
	if (!g.ovchk)
	{
#pragma unroll
		for (int f = 0; f < 3; f++)
			if (f < g.nfactors) it *= g.a[f] + g.b[f] * pick<NCC>(v, g.pcol[f]);
		return it;
	}
	bool ovf = false;
#pragma unroll
	for (int f = 0; f < 3; f++)
		if (f < g.nfactors)
		{
			int64_t t = add_ovf(g.a[f], mul_ovf(g.b[f], pick<NCC>(v, g.pcol[f]), ovf), ovf);
			it = f ? mul_ovf(it, t, ovf) : t;
		}
	if (ovf && !isnull) atomicOr(stats + 2, CG_ERRFLAG_TERM_OVERFLOW);
	return it;
}

__device__ __forceinline__ void word_apply_global(uint64_t *p, int op, uint64_t val)
{
	switch (op)
	{
		case CG_WORD_ADD: atomicAdd((unsigned long long *) p, (unsigned long long) val); break;
		case CG_WORD_MIN: atomicMin((long long *) p, (long long) val); break;
		case CG_WORD_MAX: atomicMax((long long *) p, (long long) val); break;
		case CG_WORD_FADD: atomicAdd((double *) p, __longlong_as_double((long long) val)); break;
		case CG_WORD_FMIN: atomicMin((unsigned long long *) p, (unsigned long long) val); break;
		case CG_WORD_AND: atomicAnd((unsigned long long *) p, (unsigned long long) val); break;
		case CG_WORD_OR: atomicOr((unsigned long long *) p, (unsigned long long) val); break;
		default: atomicMax((unsigned long long *) p, (unsigned long long) val); break;
	}
}

__host__ __device__ __forceinline__ uint64_t word_identity(int op)
{
	switch (op)
	{
		case CG_WORD_MIN: return (uint64_t) INT64_MAX;
		case CG_WORD_MAX: return (uint64_t) INT64_MIN;
		case CG_WORD_FMIN: return ~0ull;
		case CG_WORD_AND: return ~0ull;
		case CG_WORD_OR: return 0ull;
		default: return 0ull;     /* ADD, FADD (+0.0), FMAX */
	}
}

__device__ __forceinline__ uint64_t word_combine(int op, uint64_t a, uint64_t b)
{
	switch (op)
	{
		case CG_WORD_ADD: return a + b;
		case CG_WORD_MIN: return (uint64_t) min((long long) a, (long long) b);
		case CG_WORD_MAX: return (uint64_t) max((long long) a, (long long) b);
		case CG_WORD_FADD: return (uint64_t) __double_as_longlong(__longlong_as_double((long long) a) + __longlong_as_double((long long) b));
		case CG_WORD_FMIN: return a < b ? a : b;
		case CG_WORD_AND: return a & b;
		case CG_WORD_OR: return a | b;
		default: return a > b ? a : b;
	}
}

__device__ __forceinline__ uint64_t warp_reduce_word(uint64_t x, int op)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
	{
		uint64_t y = __shfl_xor_sync(0xffffffffu, x, o);
		x = word_combine(op, x, y);
	}
	return x;
}

/* the group key of a row that passed WHERE: the composite code, one column, or two packed (low / high 32 bits).  false =
 * the row has no group here: a NULL in a packed two-column key (CG_ERRFLAG_NULL_MULTIKEY raised), or a composite key
 * value outside its column's bounds (CG_ERRFLAG_KEY_RANGE raised) */
template <int NCC>
__device__ __forceinline__ bool group_key(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask, int64_t &key, bool &key_null)
{
	if (P.composite)
	{
		uint64_t code = 0;
		bool ok = true;
#pragma unroll
		for (int g = 0; g < CG_MAX_GROUP_COLS; g++)
			if (g < P.ngroup)
			{
				const int c = P.gcol[g];
				const uint64_t d = (uint64_t) pick<NCC>(v, c) - (uint64_t) P.kmin[g];
				const bool isnull = (nullmask >> c) & 1u;
				ok = ok && (isnull || d < P.kradix[g] - 1u);
				const uint64_t digit = isnull ? 0u : d + 1u;
				code = g ? code * P.kradix[g] + digit : digit;
			}
		if (!ok)
		{
			atomicOr(P.stats + 2, CG_ERRFLAG_KEY_RANGE);
			return false;
		}
		key_null = false;
		key = (int64_t) code;
		return true;
	}
	if (P.ngroup == 1)
	{
		int c = P.gcol[0];
		key_null = (nullmask >> c) & 1u;
		key = pick<NCC>(v, c);
		return true;
	}
	int c0 = P.gcol[0], c1 = P.gcol[1];
	if (((nullmask >> c0) | (nullmask >> c1)) & 1u)
	{
		atomicOr(P.stats + 2, CG_ERRFLAG_NULL_MULTIKEY);
		return false;
	}
	key_null = false;
	key = (int64_t) ((uint64_t) (uint32_t) pick<NCC>(v, c0) | ((uint64_t) (uint32_t) pick<NCC>(v, c1) << 32));
	return true;
}

/* direct index of a group key (group_key's packing; a composite code is a one-column key with key_min 0); the NULL key
 * -> `capacity`; ~0 = outside the declared domain (CG_ERRFLAG_KEY_RANGE raised) */
__device__ __forceinline__ uint64_t dense_slot_of_packed(const KPlan &P, int64_t key, bool key_null)
{
	if (key_null) return P.capacity;
	uint64_t s;
	if (P.ngroup == 2 && !P.composite)
	{
		uint64_t a = (uint64_t) (int64_t) (int32_t) (uint32_t) key - (uint64_t) P.key_min;
		uint64_t b = (uint64_t) (int64_t) (int32_t) (uint32_t) ((uint64_t) key >> 32) - (uint64_t) P.key_min1;
		s = (b >= P.range1) ? ~0ull : a * P.range1 + b;
	}
	else
		s = (uint64_t) key - (uint64_t) P.key_min;
	if (s < P.capacity) return s;
	atomicOr(P.stats + 2, CG_ERRFLAG_KEY_RANGE);
	return ~0ull;
}

/*
 * The value of a CASE argument (KPlan.arms[first .. first + n)) for a row its FILTER accepted: the first arm whose WHEN tree
 * is TRUE over the pool atoms' "is TRUE" bits `truth` (UNKNOWN is not TRUE), else the ELSE arm, else NULL.  Only the chosen
 * arm's result is evaluated, so an arm that was not chosen raises nothing.  Sets isnull, or the integer term it / the float
 * term ft; a product arm is int_term's product over the arm's factors, with its overflow check when g.ovchk.
 */
template <int NCC>
__device__ __forceinline__ void case_term(const KPlan &P, const KAgg &g, int first, int n, uint32_t truth, const int64_t (&v)[NCC],
										  uint32_t nullmask, bool &isnull, int64_t &it, double &ft)
{
	int chosen = -1;
#pragma unroll 1
	for (int i = first; i < first + n; i++)
		if (P.arms[i].nwhen == 0 || eval_postfix(truth, P.arms[i].nwhen, P.arms[i].when))
		{
			chosen = i;
			break;
		}
	if (chosen < 0 || P.arms[chosen].form == CG_CASE_NULL)
	{
		isnull = true;
		return;
	}
	const KArm &A = P.arms[chosen];
	if (A.form == CG_CASE_CONST)
	{
		it = A.a[0];
		ft = __longlong_as_double(A.a[0]);
		return;
	}
	bool ovf = false;
#pragma unroll
	for (int f = 0; f < 3; f++)
		if (f < A.nfactors)
		{
			const int c = A.pcol[f];
			const int64_t x = pick<NCC>(v, c);
			isnull = isnull || ((nullmask >> c) & 1u);
			if (g.is_float) ft *= __longlong_as_double(A.a[f]) + __longlong_as_double(A.b[f]) * __longlong_as_double(x);
			else if (!g.ovchk) it *= A.a[f] + A.b[f] * x;
			else
			{
				const int64_t t = add_ovf(A.a[f], mul_ovf(A.b[f], x, ovf), ovf);
				it = f ? mul_ovf(it, t, ovf) : t;
			}
		}
	if (ovf && !isnull) atomicOr(P.stats + 2, CG_ERRFLAG_TERM_OVERFLOW);
}

/* the sum(x^2) callback of the kernels built without CG_AGG_VARIANCE (it is never called) */
struct NoSquares
{
	__device__ __forceinline__ void operator()(int, const KAgg &, uint64_t, uint64_t) const {}
};

/*
 * K4: the transition terms of a row that passed WHERE and has a group.  For each aggregate a < min(naggs, NA), in
 * order, term(a, g, noinput, w0, w1) is called when the row is no input of a -- an argument is NULL, its FILTER is
 * not TRUE or its bool_and / bool_or argument is UNKNOWN: a strict transition function skips the row, it is only
 * counted -- and otherwise when a has a value word: w0 = that word's operand, w1 = the high limb of a two-limb sum
 * (count(x) is rows - no-input rows).  A term goes to its accumulator before the next one is computed, so that the
 * 64-register general kernel never holds more than one.
 * VAR: the plan may hold CG_AGG_VARIANCE aggregates.  Their term is sum's (w0, w1 of x), and before it
 * sq(a, g, lo, hi) receives x^2 = hi:lo (unsigned 128 bits, from |x|).  Without VAR the kind is not compiled in, so the
 * kernels of the other plans are what they were.
 * CASE: the plan may hold CASE arguments (KPlan.arms); an aggregate with arms takes its term from case_term.  Without CASE
 * the arms are not compiled in, as VAR does for variance.
 */
template <int NCC, int NA, bool VAR = false, bool CASE = false, class Term, class Sq = NoSquares>
__device__ __forceinline__ void row_terms(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask, Term term, Sq sq = Sq())
{
	uint32_t argtrue, truth;
	const uint32_t rejected = eval_filters<NCC>(P, v, nullmask, &argtrue, CASE ? &truth : nullptr);
#pragma unroll
	for (int a = 0; a < NA; a++)
	{
		if (a < P.naggs)
		{
			const KAgg &g = P.aggs[a];
			bool isnull = (rejected >> a) & 1u;
			if (g.kind == CG_AGG_COUNT_STAR)
			{
				if (isnull) term(a, g, true, 0ull, 0ull);
				continue;
			}
			int64_t it = 1;
			double ft = 1.0;
			if (CASE && P.cnarms[a] > 0)
			{
				/* a row the FILTER rejected is no input: its CASE is not consulted */
				if (!isnull) case_term<NCC>(P, g, P.cfirst[a], P.cnarms[a], truth, v, nullmask, isnull, it, ft);
			}
			else
			{
#pragma unroll
				for (int f = 0; f < 3; f++)
					if (f < g.nfactors)
					{
						int c = g.pcol[f];
						isnull = isnull || ((nullmask >> c) & 1u);
						if (g.is_float) ft *= __longlong_as_double(g.a[f]) + __longlong_as_double(g.b[f]) * __longlong_as_double(pick<NCC>(v, c));
					}
				if (!g.is_float) it = int_term<NCC>(g, v, isnull, P.stats);
			}
			if (isnull) { term(a, g, true, 0ull, 0ull); continue; }
			if (g.kind == CG_AGG_COUNT) continue;
			uint64_t w0, w1 = 0;
			if (g.kind == CG_AGG_SUM)
			{
				if (g.is_float) w0 = (uint64_t) __double_as_longlong(ft);
				else if (g.nlimbs == 1)
				{
					if (it > g.bound || it < -g.bound) atomicOr(P.stats + 2, CG_ERRFLAG_SUM_BOUND);
					w0 = (uint64_t) it;
				}
				else { w0 = (uint64_t) (uint32_t) it; w1 = (uint64_t) (it >> 32); }
			}
			else if (VAR && g.kind == CG_AGG_VARIANCE)
			{
				if (g.bound > 0 && (it > g.bound || it < -g.bound)) atomicOr(P.stats + 2, CG_ERRFLAG_SUM_BOUND);
				if (g.nlimbs == 1) w0 = (uint64_t) it;
				else { w0 = (uint64_t) (uint32_t) it; w1 = (uint64_t) (it >> 32); }
				const uint64_t u = it < 0 ? 0ull - (uint64_t) it : (uint64_t) it;
				sq(a, g, u * u, __umul64hi(u, u));
			}
			else if (g.barg) /* BOOL_AND / BOOL_OR: TRUE = all ones */
				w0 = ((argtrue >> a) & 1u) ? ~0ull : 0ull;
			else /* MIN / MAX, BIT_AND / BIT_OR (the sign-extended column value) */
				w0 = g.is_float ? f8_ordered(__double_as_longlong(ft)) : (uint64_t) it;
			term(a, g, false, w0, w1);
		}
	}
}

/* an exact integer sum kept as two words (low 32 bits, high part) */
__host__ __device__ __forceinline__ bool two_limbs(const KAgg &g) { return g.kind == CG_AGG_SUM && !g.is_float && g.nlimbs == 2; }
/* the same, for kernels built with VAR: a variance aggregate's sum(x) may be two limbs too */
template <bool VAR>
__host__ __device__ __forceinline__ bool two_sum_limbs(const KAgg &g)
{
	return VAR ? (cg_kind_sums(g.kind) && !g.is_float && g.nlimbs == 2) : two_limbs(g);
}

/* the 32-bit limb l of x^2 = hi:lo */
__device__ __forceinline__ uint64_t square_limb(uint64_t lo, uint64_t hi, int l)
{
	const uint64_t w = l < 2 ? lo : hi;
	return (l & 1) ? (w >> 32) : (w & 0xffffffffull);
}

/* x^2 = hi:lo into the sum(x^2) words q[0 .. qlimbs) of a table entry (a zero limb adds nothing) */
__device__ __forceinline__ void squares_apply_global(uint64_t *q, int qlimbs, uint64_t lo, uint64_t hi)
{
	if (qlimbs == 1)
	{
		if (lo) atomicAdd((unsigned long long *) q, (unsigned long long) lo);
		return;
	}
#pragma unroll
	for (int l = 0; l < 4; l++)
		if (l < qlimbs)
		{
			const uint64_t x = square_limb(lo, hi, l);
			if (x) atomicAdd((unsigned long long *) q + l, (unsigned long long) x);
		}
}

/* one row into an entry of the global group table (word 0 = rows in the group) */
template <int NCC, int NA, bool VAR = false, bool CASE = false>
__device__ __forceinline__ void global_accumulate(const KPlan &P, uint64_t *entry, const int64_t (&v)[NCC], uint32_t nullmask)
{
	atomicAdd((unsigned long long *) entry, 1ull);
	auto term = [&](int, const KAgg &g, bool noinput, uint64_t w0, uint64_t w1) {
		if (noinput) atomicAdd((unsigned long long *) entry + g.nullword, 1ull);
		else
		{
			word_apply_global(entry + g.word0, P.wordop[g.word0], w0);
			if (two_sum_limbs<VAR>(g)) atomicAdd((unsigned long long *) entry + g.word0 + 1, (unsigned long long) w1);
		}
	};
	if constexpr (VAR)
		row_terms<NCC, NA, true, CASE>(P, v, nullmask, term,
									   [&](int, const KAgg &g, uint64_t lo, uint64_t hi) { squares_apply_global(entry + g.qword, g.qlimbs, lo, hi); });
	else
		row_terms<NCC, NA, false, CASE>(P, v, nullmask, term);
}

/* ------------------------------------------------------------------------------ *
 *  The row path of the interpretive kernels (cg_scan_kernel over staged chunk groups, cg_join_agg_kernel over joined
 *  rows): a row as v[] + NULL mask -> WHERE -> group table entry or per-thread accumulators.
 * ------------------------------------------------------------------------------ */
/*
 * Find (or claim) the table entry of a group key.  Returns the word pointer of the
 * entry (word 0 = rows in group) or NULL after raising an error flag.
 *   dense: entry = key - key_min, NULL key -> entry `capacity`
 *   hash : open addressing, linear probing over a separate key array (8 B per slot, so the
 *          probed working set is a quarter of an array-of-structs table), 64-bit CAS to claim
 *          a slot; the NULL group and the key equal to the EMPTY sentinel live in two extra
 *          entries behind the addressable ones
 */
template <int MODE>
__device__ __forceinline__ uint64_t *find_entry(const KPlan &P, int64_t key, bool key_null)
{
	if (MODE == CG_MODE_DENSE)
	{
		uint64_t slot = dense_slot_of_packed(P, key, key_null);
		return slot == ~0ull ? nullptr : P.table + slot * (uint64_t) P.stride;
	}
	else
	{
		if (key_null) return P.table + P.capacity * (uint64_t) P.stride;
		if (key == CG_HASH_EMPTY) return P.table + (P.capacity + 1) * (uint64_t) P.stride;
		uint64_t mask = P.capacity - 1;
		uint64_t h = cg_home_slot(key, P.hash_shift);
		for (uint32_t probes = 0; probes < 8192; probes++)
		{
			unsigned long long *kp = (unsigned long long *) (P.hkeys + h);
			long long cur = (long long) __ldcg(kp);     /* L2: keys only ever go EMPTY -> key */
			if (cur == key) return P.table + h * (uint64_t) P.stride;
			if (cur == CG_HASH_EMPTY)
			{
				long long old = (long long) atomicCAS(kp, (unsigned long long) CG_HASH_EMPTY, (unsigned long long) key);
				if (old == CG_HASH_EMPTY || old == key) return P.table + h * (uint64_t) P.stride;
			}
			h = (h + 1) & mask;
		}
		atomicOr(P.stats + 2, CG_ERRFLAG_TABLE_FULL);
		return nullptr;
	}
}

/* per-thread accumulators of the plain-aggregate mode */
template <int NAC, bool VAR>
struct ThreadAcc
{
	uint64_t w[NAC][3];     /* [agg][word0, word0+1, NULL-input count] */
	uint64_t rows;
	uint64_t q[NAC][VAR ? 4 : 1];   /* VAR: [agg][sum(x^2) word qword + l] */
};

/* every accumulator at its word's identity */
template <int NAC, bool VAR>
__device__ __forceinline__ void thread_acc_init(const KPlan &P, ThreadAcc<NAC, VAR> &acc)
{
	acc.rows = 0;
#pragma unroll
	for (int a = 0; a < NAC; a++)
	{
		acc.w[a][0] = (a < P.naggs && P.aggs[a].kind != CG_AGG_COUNT_STAR) ? word_identity(P.wordop[P.aggs[a].word0]) : 0;
		acc.w[a][1] = 0;
		acc.w[a][2] = 0;
		if constexpr (VAR)
		{
#pragma unroll
			for (int l = 0; l < 4; l++) acc.q[a][l] = 0;
		}
	}
}

template <int NCC, int NAC, int MODE, bool VAR, bool CASE = false>
__device__ __forceinline__ void process_row(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask,
											ThreadAcc<NAC, VAR> &acc, uint32_t &removed)
{
	/* K3: WHERE tree, three-valued: an atom on a NULL input is not TRUE */
	if (!eval_where<NCC>(P, v, nullmask))
	{
		removed++;
		return;
	}
	if (MODE != CG_MODE_GLOBAL)
	{
		int64_t key;
		bool key_null;
		if (!group_key<NCC>(P, v, nullmask, key, key_null)) return;
		uint64_t *entry = find_entry<MODE>(P, key, key_null);
		if (entry != nullptr) global_accumulate<NCC, NAC, VAR, CASE>(P, entry, v, nullmask);
		return;
	}
	acc.rows++;
	auto term = [&](int a, const KAgg &g, bool noinput, uint64_t w0, uint64_t w1) {
		if (noinput) acc.w[a][2]++;
		else
		{
			acc.w[a][0] = word_combine(P.wordop[g.word0], acc.w[a][0], w0);
			if (two_sum_limbs<VAR>(g)) acc.w[a][1] += w1;
		}
	};
	if constexpr (VAR)
		row_terms<NCC, NAC, true, CASE>(P, v, nullmask, term, [&](int a, const KAgg &g, uint64_t lo, uint64_t hi) {
			/* a thread's limb sums grow by < 2^32 per row; the one-word form is bounded by the table's own guarantee */
			if (g.qlimbs == 1) acc.q[a][0] += lo;
			else
			{
#pragma unroll
				for (int l = 0; l < 4; l++)
					if (l < g.qlimbs) acc.q[a][l] += square_limb(lo, hi, l);
			}
		});
	else
		row_terms<NCC, NAC, false, CASE>(P, v, nullmask, term);
}

/* the end of a kernel that ran process_row: the row counters into P.stats ([0] rows handed to WHERE, [1] rows removed)
 * and, in the plain-aggregate mode, the thread's accumulators into the table -- warp shuffle reduce, then one atomic per
 * warp and word.  Every thread of the block calls it. */
template <int NAC, int MODE, bool VAR>
__device__ __forceinline__ void flush_thread(const KPlan &P, const ThreadAcc<NAC, VAR> &acc, uint32_t removed, unsigned long long scanned)
{
	const uint32_t tid = threadIdx.x;
	unsigned long long rem = warp_reduce_word(removed, CG_WORD_ADD);
	unsigned long long scn = warp_reduce_word(scanned, CG_WORD_ADD);
	if ((tid & 31) == 0)
	{
		if (scn) atomicAdd(P.stats + 0, scn);
		if (rem) atomicAdd(P.stats + 1, rem);
	}
	if (MODE == CG_MODE_GLOBAL)
	{
		uint64_t rows_passed = warp_reduce_word(acc.rows, CG_WORD_ADD);
		if ((tid & 31) == 0 && rows_passed) atomicAdd((unsigned long long *) P.table, (unsigned long long) rows_passed);
#pragma unroll
		for (int a = 0; a < NAC; a++)
		{
			if (a < P.naggs && (P.aggs[a].kind != CG_AGG_COUNT_STAR || P.aggs[a].filt))
			{
				const KAgg &g = P.aggs[a];
				uint64_t nulls = warp_reduce_word(acc.w[a][2], CG_WORD_ADD);
				uint64_t x0 = warp_reduce_word(acc.w[a][0], P.wordop[g.word0]);
				uint64_t x1 = warp_reduce_word(acc.w[a][1], CG_WORD_ADD);
				if ((tid & 31) == 0)
				{
					if (nulls) atomicAdd((unsigned long long *) P.table + g.nullword, (unsigned long long) nulls);
					if (g.kind != CG_AGG_COUNT && g.kind != CG_AGG_COUNT_STAR)
					{
						if (x0 != word_identity(P.wordop[g.word0])) word_apply_global(P.table + g.word0, P.wordop[g.word0], x0);
						if (two_sum_limbs<VAR>(g) && x1)
							atomicAdd((unsigned long long *) P.table + g.word0 + 1, (unsigned long long) x1);
					}
				}
				if constexpr (VAR)
				{
					if (g.kind == CG_AGG_VARIANCE)
					{
#pragma unroll
						for (int l = 0; l < 4; l++)
						{
							const uint64_t x = warp_reduce_word(acc.q[a][l], CG_WORD_ADD);
							if ((tid & 31) == 0 && l < g.qlimbs && x) atomicAdd((unsigned long long *) P.table + g.qword + l, (unsigned long long) x);
						}
					}
				}
			}
		}
	}
}

#endif
