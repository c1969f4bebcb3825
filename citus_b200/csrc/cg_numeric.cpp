/*
 * cg_numeric.cpp -- text of the coordinator-visible results.
 *
 * sum(int8) / sum(numeric) results are numeric in PostgreSQL; avg is the master-side
 * expression sum(sum) / sum(count) (planner/multi_logical_optimizer.c:1807-1830,
 * MasterAverageExpression :2302-2355) evaluated by [PG] numeric_div, whose result scale is
 * chosen by select_div_scale (numeric.c): at least NUMERIC_MIN_SIG_DIGITS = 16 significant
 * digits, counted in base-10000 digits, and never less than either input's display scale.
 * Pinned by the reference's expected/multi_tpch_query1.out (avg_qty, avg_price, avg_disc)
 * and expected/columnar_query.out:9-29 through tests/test_host_numeric.py.
 */
#include <string.h>

#include <stdlib.h>

#include <algorithm>
#include <string>
#include <vector>

#include "cg_internal.h"

typedef unsigned __int128 u128;
typedef __int128 i128;

static std::string u128_to_string(u128 v)
{
	if (v == 0) return "0";
	char buf[48];
	int i = 47;
	buf[i] = 0;
	while (v) { buf[--i] = (char) ('0' + (int) (v % 10)); v /= 10; }
	return std::string(buf + i);
}

static int put(const std::string &s, char *buf, size_t buflen)
{
	if (s.size() + 1 > buflen) return cg_set_error(CG_EINVAL, "numeric text needs %zu bytes", s.size() + 1);
	memcpy(buf, s.c_str(), s.size() + 1);
	return CG_OK;
}

static std::string scaled_text(bool neg, const std::string &digits_in, int scale)
{
	std::string digits = digits_in;
	if (scale > 0)
	{
		if ((int) digits.size() <= scale) digits = std::string(scale + 1 - digits.size(), '0') + digits;
		digits.insert(digits.size() - scale, ".");
	}
	bool zero = digits.find_first_not_of("0.") == std::string::npos;
	return (neg && !zero ? "-" : "") + digits;
}

extern "C" int cg_numeric_out(int64_t hi, uint64_t lo, int32_t scale, char *buf, size_t buflen)
{
	if (scale < 0 || scale > 30) return cg_set_error(CG_EINVAL, "scale %d", scale);
	i128 v = ((i128) hi << 64) | (i128) (u128) lo;
	bool neg = v < 0;
	u128 mag = neg ? (u128) (-(v + 1)) + 1 : (u128) v;
	return put(scaled_text(neg, u128_to_string(mag), scale), buf, buflen);
}

/* weight (base-10000 exponent) and value of the first non-zero base-10000 digit of
 * mag * 10^-scale, as the loop at the top of select_div_scale finds them */
static void weight_firstdigit(u128 mag, int scale, int *weight, int *first)
{
	if (mag == 0) { *weight = 0; *first = 0; return; }
	int pad = (4 - scale % 4) % 4;
	for (int i = 0; i < pad; i++) mag *= 10;      /* callers keep mag < 10^34, no overflow */
	int frac_digits = (scale + pad) / 4;
	int ndig = 0, f = 0;
	while (mag) { f = (int) (mag % 10000); mag /= 10000; ndig++; }
	*weight = ndig - 1 - frac_digits;
	*first = f;
}

extern "C" int cg_numeric_div_out(int64_t hi, uint64_t lo, int32_t scale, int64_t count, char *buf, size_t buflen)
{
	if (count <= 0) return cg_set_error(CG_EINVAL, "division by %lld", (long long) count);
	if (scale < 0 || scale > 30) return cg_set_error(CG_EINVAL, "scale %d", scale);
	i128 v = ((i128) hi << 64) | (i128) (u128) lo;
	bool neg = v < 0;
	u128 mag = neg ? (u128) (-(v + 1)) + 1 : (u128) v;
	u128 limit = 1;
	for (int i = 0; i < 34; i++) limit *= 10;
	if (mag >= limit) return cg_set_error(CG_EUNSUPPORTED, "sum too large for the numeric formatter");

	int w1, f1, w2, f2;
	weight_firstdigit(mag, scale, &w1, &f1);
	weight_firstdigit((u128) count, 0, &w2, &f2);
	int qweight = w1 - w2;
	if (f1 <= f2) qweight--;
	int rscale = 16 - qweight * 4;
	if (rscale < scale) rscale = scale;
	if (rscale < 0) rscale = 0;
	if (rscale > 1000) rscale = 1000;

	/* long division: integer part, then rscale + 1 fractional digits, round half away from zero */
	u128 d = (u128) count;
	u128 scale_pow = 1;
	for (int i = 0; i < scale; i++) scale_pow *= 10;
	/* quotient of mag / (count * 10^scale) */
	u128 denom = d * scale_pow;                /* count < 2^63, scale_pow <= 10^30: fits 2^127 only for small scale */
	if (scale > 18) return cg_set_error(CG_EUNSUPPORTED, "scale %d too large for the numeric formatter", scale);
	u128 ip = mag / denom;
	u128 rem = mag % denom;
	std::string frac;
	frac.reserve(rscale + 1);
	for (int i = 0; i < rscale + 1; i++)
	{
		/* rem < denom < 2^63 * 10^18 < 2^123; rem * 10 < 2^127 */
		rem *= 10;
		int digit = (int) (rem / denom);
		rem %= denom;
		frac.push_back((char) ('0' + digit));
	}
	/* round at rscale using the extra digit */
	bool up = frac[rscale] >= '5';
	frac.resize(rscale);
	std::string ips = u128_to_string(ip);
	if (up)
	{
		int i = rscale - 1;
		while (i >= 0 && frac[i] == '9') { frac[i] = '0'; i--; }
		if (i >= 0) frac[i]++;
		else
		{
			int j = (int) ips.size() - 1;
			while (j >= 0 && ips[j] == '9') { ips[j] = '0'; j--; }
			if (j >= 0) ips[j]++;
			else ips.insert(ips.begin(), '1');
		}
	}
	std::string s = ips;
	if (rscale > 0) s += "." + frac;
	bool zero = s.find_first_not_of("0.") == std::string::npos;
	if (neg && !zero) s = "-" + s;
	return put(s, buf, buflen);
}

/* ------------------------------------------------------------------------------ *
 *  var_pop / var_samp / stddev_pop / stddev_samp: [PG] numeric_stddev_internal over the exact state (N, S = sum(x),
 *  Q = sum(x^2)).  Its operands reach ~2^221 and its quotients carry up to 1000 fraction digits, so it runs on a small
 *  non-negative bignum: base-2^32 limbs, least significant first, no leading zero limbs.
 * ------------------------------------------------------------------------------ */
typedef std::vector<uint32_t> Big;

static void big_trim(Big &a) { while (!a.empty() && a.back() == 0) a.pop_back(); }
static Big big_of(u128 v)
{
	Big r;
	while (v) { r.push_back((uint32_t) v); v >>= 32; }
	return r;
}
static int big_cmp(const Big &a, const Big &b)
{
	if (a.size() != b.size()) return a.size() < b.size() ? -1 : 1;
	for (size_t i = a.size(); i-- > 0;)
		if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
	return 0;
}
static Big big_add(const Big &a, const Big &b)
{
	Big r(std::max(a.size(), b.size()) + 1, 0);
	uint64_t c = 0;
	for (size_t i = 0; i < r.size(); i++)
	{
		c += (i < a.size() ? a[i] : 0ull) + (i < b.size() ? b[i] : 0ull);
		r[i] = (uint32_t) c;
		c >>= 32;
	}
	big_trim(r);
	return r;
}
/* a - b, a >= b */
static Big big_sub(const Big &a, const Big &b)
{
	Big r(a.size(), 0);
	int64_t br = 0;
	for (size_t i = 0; i < a.size(); i++)
	{
		int64_t d = (int64_t) a[i] - (i < b.size() ? (int64_t) b[i] : 0) - br;
		br = d < 0;
		r[i] = (uint32_t) (d + (br << 32));
	}
	big_trim(r);
	return r;
}
static Big big_mul(const Big &a, const Big &b)
{
	if (a.empty() || b.empty()) return Big();
	Big r(a.size() + b.size(), 0);
	for (size_t i = 0; i < a.size(); i++)
	{
		uint64_t c = 0;
		for (size_t j = 0; j < b.size(); j++)
		{
			c += (uint64_t) a[i] * b[j] + r[i + j];
			r[i + j] = (uint32_t) c;
			c >>= 32;
		}
		for (size_t k = i + b.size(); c; k++) { c += r[k]; r[k] = (uint32_t) c; c >>= 32; }
	}
	big_trim(r);
	return r;
}
static Big big_pow10(int n)
{
	Big r = big_of(1);
	const Big ten9 = big_of(1000000000u);
	for (; n >= 9; n -= 9) r = big_mul(r, ten9);
	u128 t = 1;
	while (n-- > 0) t *= 10;
	return big_mul(r, big_of(t));
}
static size_t big_bits(const Big &a) { return a.empty() ? 0 : 32 * (a.size() - 1) + (32 - __builtin_clz(a.back())); }
/* q = a / d, returns a % d (d > 0) */
static uint32_t big_divmod_small(const Big &a, uint32_t d, Big &q)
{
	q.assign(a.size(), 0);
	uint64_t r = 0;
	for (size_t i = a.size(); i-- > 0;)
	{
		const uint64_t cur = (r << 32) | a[i];
		q[i] = (uint32_t) (cur / d);
		r = cur % d;
	}
	big_trim(q);
	return (uint32_t) r;
}
/* q = a / b, rem = a % b (b > 0): Knuth's algorithm D over base-2^32 digits (the form of Hacker's Delight's divmnu) */
static void big_divmod(const Big &a, const Big &b, Big &q, Big &rem)
{
	if (big_cmp(a, b) < 0) { q.clear(); rem = a; return; }
	if (b.size() == 1)
	{
		const uint32_t r = big_divmod_small(a, b[0], q);
		rem = big_of(r);
		return;
	}
	const size_t n = b.size(), m = a.size() - n;
	const int sh = __builtin_clz(b.back());
	/* normalise: the divisor's top digit gets its top bit set */
	Big vn(n), un(a.size() + 1);
	for (size_t i = n - 1; i > 0; i--) vn[i] = (b[i] << sh) | (sh ? (uint32_t) ((uint64_t) b[i - 1] >> (32 - sh)) : 0u);
	vn[0] = b[0] << sh;
	un[a.size()] = sh ? (uint32_t) ((uint64_t) a.back() >> (32 - sh)) : 0u;
	for (size_t i = a.size() - 1; i > 0; i--) un[i] = (a[i] << sh) | (sh ? (uint32_t) ((uint64_t) a[i - 1] >> (32 - sh)) : 0u);
	un[0] = a[0] << sh;
	q.assign(m + 1, 0);
	const uint64_t B = 1ull << 32;
	for (size_t j = m + 1; j-- > 0;)
	{
		/* estimate the quotient digit from the top two digits, correct it at most twice */
		const uint64_t num = ((uint64_t) un[j + n] << 32) | un[j + n - 1];
		uint64_t qhat = num / vn[n - 1], rhat = num % vn[n - 1];
		while (qhat >= B || qhat * vn[n - 2] > ((rhat << 32) | un[j + n - 2]))
		{
			qhat--;
			rhat += vn[n - 1];
			if (rhat >= B) break;
		}
		/* multiply and subtract */
		int64_t k = 0, t;
		for (size_t i = 0; i < n; i++)
		{
			const uint64_t p = qhat * vn[i];
			t = (int64_t) un[i + j] - k - (int64_t) (p & 0xffffffffull);
			un[i + j] = (uint32_t) t;
			k = (int64_t) (p >> 32) - (t >> 32);
		}
		t = (int64_t) un[j + n] - k;
		un[j + n] = (uint32_t) t;
		q[j] = (uint32_t) qhat;
		if (t < 0)
		{
			/* the estimate was one too large: add the divisor back */
			q[j]--;
			uint64_t c = 0;
			for (size_t i = 0; i < n; i++)
			{
				c += (uint64_t) un[i + j] + vn[i];
				un[i + j] = (uint32_t) c;
				c >>= 32;
			}
			un[j + n] += (uint32_t) c;
		}
	}
	big_trim(q);
	/* denormalise the remainder */
	rem.assign(n, 0);
	for (size_t i = 0; i < n; i++)
		rem[i] = (un[i] >> sh) | (sh ? (uint32_t) ((uint64_t) un[i + 1] << (32 - sh)) : 0u);
	big_trim(rem);
}
/* floor(sqrt(a)): Newton's iteration from above, x' = (x + a / x) / 2, until it stops decreasing */
static Big big_isqrt(const Big &a)
{
	if (a.empty()) return Big();
	Big x;
	const size_t half = (big_bits(a) + 1) / 2;           /* 2^half > sqrt(a) */
	x.assign(half / 32 + 1, 0);
	x[half / 32] = 1u << (half % 32);
	big_trim(x);
	for (;;)
	{
		Big q, r;
		big_divmod(a, x, q, r);
		Big y;
		big_divmod_small(big_add(x, q), 2, y);
		if (big_cmp(y, x) >= 0) return x;
		x = y;
	}
}
static std::string big_to_string(Big a)
{
	if (a.empty()) return "0";
	std::string s;
	while (!a.empty())
	{
		Big q;
		uint32_t d = big_divmod_small(a, 1000000000u, q);
		for (int i = 0; i < 9; i++) { s.push_back((char) ('0' + d % 10)); d /= 10; }
		a = q;
	}
	while (s.size() > 1 && s.back() == '0') s.pop_back();
	return std::string(s.rbegin(), s.rend());
}
/* weight and first base-10000 digit of a * 10^-scale (a > 0), as select_div_scale finds them */
static void big_weight_firstdigit(const Big &a, int scale, int *weight, int *first)
{
	const int pad = (4 - scale % 4) % 4;
	const std::string d = big_to_string(big_mul(a, big_pow10(pad)));
	const int ndig = ((int) d.size() + 3) / 4;
	*weight = ndig - 1 - (scale + pad) / 4;
	*first = atoi(d.substr(0, d.size() - 4 * (ndig - 1)).c_str());
}

extern "C" int cg_numeric_var_out(int32_t final, int64_t n, int64_t sum_hi, uint64_t sum_lo, const uint64_t *sumsq, int32_t scale,
								  char *buf, size_t buflen, int32_t *is_null)
{
	if (final < CG_VAR_POP || final > CG_STDDEV_SAMP) return cg_set_error(CG_EINVAL, "final function %d", final);
	if (scale < 0 || scale > 30) return cg_set_error(CG_EINVAL, "scale %d", scale);
	if (n < 0) return cg_set_error(CG_EINVAL, "negative count %lld", (long long) n);
	if (!sumsq || !buf || !is_null) return cg_set_error(CG_EINVAL, "NULL argument");
	const bool sample = final == CG_VAR_SAMP || final == CG_STDDEV_SAMP;
	*is_null = 0;
	if (n == 0 || (sample && n <= 1))
	{
		*is_null = 1;
		return put("", buf, buflen);
	}
	const i128 S = ((i128) sum_hi << 64) | (i128) (u128) sum_lo;
	const Big absS = big_of(S < 0 ? (u128) (-(S + 1)) + 1 : (u128) S);
	Big Q;
	for (int i = 2; i >= 0; i--) { Q.insert(Q.begin(), (uint32_t) (sumsq[i] >> 32)); Q.insert(Q.begin(), (uint32_t) sumsq[i]); }
	big_trim(Q);
	const Big N = big_of((u128) n);
	/* num = N Q - S^2 at dscale 2 scale; a result <= 0 is const_zero (no fraction digits) */
	const Big NQ = big_mul(N, Q), S2 = big_mul(absS, absS);
	if (big_cmp(NQ, S2) <= 0) return put("0", buf, buflen);
	const Big num = big_sub(NQ, S2);
	const Big den = big_mul(N, sample ? big_of((u128) (n - 1)) : N);
	/* select_div_scale(num, den): num has dscale 2 scale, den dscale 0 */
	int w1, f1, w2, f2;
	big_weight_firstdigit(num, 2 * scale, &w1, &f1);
	big_weight_firstdigit(den, 0, &w2, &f2);
	int qweight = w1 - w2;
	if (f1 <= f2) qweight--;
	int rscale = 16 - qweight * 4;
	rscale = std::max(rscale, 2 * scale);
	rscale = std::max(rscale, 0);
	rscale = std::min(rscale, 1000);
	/* variance V = round(num / 10^(2 scale) / den, rscale) as the integer v = V * 10^rscale, half away from zero
	 * (rscale >= 2 scale) */
	Big v, rem;
	big_divmod(big_mul(num, big_pow10(rscale - 2 * scale)), den, v, rem);
	if (big_cmp(big_add(rem, rem), den) >= 0) v = big_add(v, big_of(1));
	if (final == CG_STDDEV_POP || final == CG_STDDEV_SAMP)
	{
		/* sqrt_var: sqrt(V) at rscale, rounded half away from zero = floor(sqrt(v 10^rscale) + 1/2) */
		const Big M = big_mul(v, big_pow10(rscale));
		Big r = big_isqrt(M);
		/* sqrt(M) >= r + 1/2  <=>  M >= r^2 + r + 1/4  <=>  M > r^2 + r (integers) */
		if (big_cmp(M, big_add(big_mul(r, r), r)) > 0) r = big_add(r, big_of(1));
		v = r;
	}
	return put(scaled_text(false, big_to_string(v), rscale), buf, buflen);
}
