"""Exact reference of var_pop / var_samp / stddev_pop / stddev_samp over integer arguments, in Python integers.

    var_out(final, n, s, q, scale)                           ->  PostgreSQL's numeric text, or None for SQL NULL
    aggregate(cols, nulls, where, group_cols, aggs, ...)     ->  reference.Result; a variance aggregate's result has
                                                                 count = N, sum = sum(x), sumsq = sum(x^2)
    filtered(...)                                            ->  the same with every aggregate's FILTER applied

var_out restates numeric_stddev_internal (PostgreSQL's numeric.c) from its definition: with N, S = sum(x) and
Q = sum(x^2), all in units of 10^-scale,
    NULL                  when N = 0, or N <= 1 for the sample forms
    num = N * Q - S^2     at display scale 2 * scale; num <= 0 is the numeric zero, text "0"
    den = N * (N - 1) (sample) or N^2 (population), display scale 0
    rscale                select_div_scale(num, den): 16 significant digits counted in base-10000 digits, at least both
                          display scales, within [0, 1000]
    variance              num / den rounded half away from zero at rscale
    stddev                the square root of that rounded variance, rounded half away from zero at rscale
The kinds reference.aggregate knows are computed by it; sum(x^2) is summed here, one row at a time, over the same groups.
"""
from __future__ import annotations

import math
from dataclasses import replace

import reference as ref

VARIANCE = 9
VAR_POP, VAR_SAMP, STDDEV_POP, STDDEV_SAMP = range(4)
NUMERIC_MIN_SIG_DIGITS, DEC_DIGITS, MAX_DISPLAY_SCALE = 16, 4, 1000


def _weight_first(mag: int, dscale: int):
    """(weight, first base-10000 digit) of mag * 10^-dscale, mag > 0, as a NumericVar would hold it"""
    frac_groups = -(-dscale // DEC_DIGITS)                # fraction digits fill whole base-10000 digits
    digits = mag * 10 ** (frac_groups * DEC_DIGITS - dscale)
    groups = []
    while digits:
        digits, d = divmod(digits, 10000)
        groups.append(d)
    return len(groups) - 1 - frac_groups, groups[-1]


def select_div_scale(num: int, num_dscale: int, den: int, den_dscale: int) -> int:
    w1, f1 = _weight_first(num, num_dscale)
    w2, f2 = _weight_first(den, den_dscale)
    qweight = w1 - w2 - (1 if f1 <= f2 else 0)
    rscale = max(NUMERIC_MIN_SIG_DIGITS - qweight * DEC_DIGITS, num_dscale, den_dscale, 0)
    return min(rscale, MAX_DISPLAY_SCALE)


def _text(v: int, rscale: int) -> str:
    if rscale == 0:
        return str(v)
    ip, fp = divmod(v, 10 ** rscale)
    return f"{ip}.{fp:0{rscale}d}"


def var_out(final: int, n: int, s: int, q: int, scale: int):
    sample = final in (VAR_SAMP, STDDEV_SAMP)
    if n == 0 or (sample and n <= 1):
        return None
    num = n * q - s * s
    if num <= 0:
        return "0"
    den = n * (n - 1) if sample else n * n
    rscale = select_div_scale(num, 2 * scale, den, 0)
    # variance * 10^rscale = num * 10^rscale / (den * 10^(2 scale)), half away from zero (both are positive)
    top, bottom = num * 10 ** rscale, den * 10 ** (2 * scale)
    v = (2 * top + bottom) // (2 * bottom)
    if final in (STDDEV_POP, STDDEV_SAMP):
        m = v * 10 ** rscale                          # (sqrt(variance) * 10^rscale)^2
        r = math.isqrt(m)
        v = r + 1 if 4 * m >= (2 * r + 1) ** 2 else r  # sqrt(m) >= r + 1/2
    return _text(v, rscale)


def _as_sum(a):
    """a variance aggregate as reference.aggregate's sum over the same argument (count, sum, overflow)"""
    return replace(a, kind=ref.SUM) if a.kind == VARIANCE else a


def aggregate(cols, nulls, where, group_cols, aggs, float_cols=()) -> ref.Result:
    res = ref.aggregate(cols, nulls, where, group_cols, [_as_sum(a) for a in aggs], float_cols)
    var = [j for j, a in enumerate(aggs) if a.kind == VARIANCE]
    for per in res.groups.values():
        for j in var:
            per[j].sumsq = 0
    if not var:
        return res
    float_cols = set(float_cols)
    rows = lambda c: c.tolist() if hasattr(c, "tolist") else list(c)     # noqa: E731
    vals_of = [[float(v) if i in float_cols else int(v) for v in rows(c)] for i, c in enumerate(cols)]
    null_of = [None if n is None else [bool(v) for v in rows(n)] for n in (nulls or [])]
    null_of += [None] * (len(cols) - len(null_of))
    w = where if (isinstance(where, tuple) and where and where[0] in ("and", "or")) else ("and",) + tuple(where or ())
    for r in range(len(cols[0]) if cols else 0):
        vals = [c[r] for c in vals_of]
        isnull = [n[r] if n is not None else False for n in null_of]
        if len(w) > 1 and ref._where_value(w, vals, isnull, float_cols) is not True:
            continue
        key = tuple(None if isnull[c] else int(vals[c]) for c in group_cols)
        per = res.groups[key]
        for j in var:
            if any(isnull[c] for c, _, _ in aggs[j].factors):
                continue
            t, _ = ref._int_term(aggs[j].factors, vals)
            per[j].sumsq += t * t
    return res


def filtered(cols, nulls, where, group_cols, aggs, float_cols=()) -> ref.Result:
    """FILTER by composition: the groups are those of WHERE alone; aggregate j of a group is the aggregate over
    (WHERE AND FILTER_j), or no input where that has no row of the group"""
    res = aggregate(cols, nulls, where, group_cols, aggs, float_cols)
    w = where if (isinstance(where, tuple) and where and where[0] in ("and", "or")) else (("and",) + tuple(where) if where else None)
    for j, a in enumerate(aggs):
        if getattr(a, "filter", None) is None:
            continue
        f = a.filter if (isinstance(a.filter, tuple) and a.filter and a.filter[0] in ("and", "or")) else (
            ("and", a.filter) if isinstance(a.filter, tuple) else ("and",) + tuple(a.filter))
        sub = aggregate(cols, nulls, ("and", w, f) if w else f, group_cols, [replace(a, filter=None)], float_cols)
        for key, per in res.groups.items():
            if key in sub.groups:
                per[j] = sub.groups[key][0]
            else:
                per[j] = ref.AggResult()
                per[j].sumsq = 0
    return res
