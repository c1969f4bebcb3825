/*
 * cg_device.cuh -- device helpers shared by the scan kernels (cg_scan.cu, cg_scan_small.cu).
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

/*
 * K3: the WHERE tree ([PG] ExecQual under ExecScan, columnar_customscan.c:1907-1913) under three-valued
 * logic: an atom on a NULL input is not TRUE, AND/OR combine "is TRUE" bits (there is no NOT node: it is
 * folded into the comparison operators), the row passes iff the root is TRUE.  Without a tree the atoms
 * are an AND-list.
 */
template <int NCC>
__device__ __forceinline__ bool eval_where(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask)
{
	uint32_t truth = 0;
#pragma unroll 1
	for (int q = 0; q < P.nquals; q++)
	{
		int c = P.qcol[q];
		bool isnull = (nullmask >> c) & 1u;
		int64_t x = pick<NCC>(v, c);
		bool t = P.isfloat[c] ? qual_true(x, P.qop[q], P.qk[q], true)
							  : (((x >= P.qlo[q]) && (x <= P.qhi[q])) != (bool) P.qneg[q]);
		truth |= (uint32_t) (t && !isnull) << q;
	}
	if (P.nqexpr == 0) return truth == (1u << P.nquals) - 1u;
	uint32_t st = 0;
#pragma unroll 1
	for (int i = 0; i < P.nqexpr; i++)
	{
		int t = P.qexpr[i];
		if (t >= 0) st = (st << 1) | ((truth >> t) & 1u);
		else
		{
			uint32_t b = st & 1u, a = (st >> 1) & 1u;
			st = ((st >> 2) << 1) | (t == CG_QX_AND ? (a & b) : (a | b));
		}
	}
	return st & 1u;
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
		default: atomicMax((unsigned long long *) p, (unsigned long long) val); break;
	}
}

__device__ __forceinline__ uint64_t word_identity(int op)
{
	switch (op)
	{
		case CG_WORD_MIN: return (uint64_t) INT64_MAX;
		case CG_WORD_MAX: return (uint64_t) INT64_MIN;
		case CG_WORD_FMIN: return ~0ull;
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
		default: return a > b ? a : b;
	}
}



/* direct index of a group key that arrives packed (two columns: low / high 32 bits);
 * ~0 = outside the declared domain */
__device__ __forceinline__ uint64_t dense_slot_of_packed(const KPlan &P, int64_t key, bool key_null)
{
	if (key_null) return P.capacity;
	if (P.ngroup == 2)
	{
		uint64_t a = (uint64_t) (int64_t) (int32_t) (uint32_t) key - (uint64_t) P.key_min;
		uint64_t b = (uint64_t) (int64_t) (int32_t) (uint32_t) ((uint64_t) key >> 32) - (uint64_t) P.key_min1;
		if (b >= P.range1 || a * P.range1 + b >= P.capacity) return ~0ull;
		return a * P.range1 + b;
	}
	uint64_t s = (uint64_t) key - (uint64_t) P.key_min;
	return s >= P.capacity ? ~0ull : s;
}

#endif
