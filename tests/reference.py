"""An exact, independent reference of the fused scan + partial aggregate, in plain Python.

It shares no code with oracle/oracle.c and nothing with the library's key packing: rows are evaluated one at a
time with Python integers (no overflow), math.fsum (correctly rounded float sums) and PostgreSQL's float8 btree
order.

    aggregate(cols, nulls, where, group_cols, aggs)  ->  Result
        cols        list of sequences, one per attribute (ints, or floats for float columns)
        nulls       list of per-row NULL flags per attribute, or None entries / None for no NULLs
        where       list of atoms (column, op, constant) -- their AND -- or a tree ("and" | "or", arm, arm, ...)
        group_cols  attribute indexes; groups are keyed by the tuple of key values (None = NULL)
        aggs        objects with .kind (0 count(*), 1 count, 2 sum, 3 min, 4 max), .factors [(column, a, b)] -- the
                    argument is prod (a + b * column) -- and .is_float

Per group and aggregate the result holds count (non-NULL inputs), the exact integer sum, the float terms (their
math.fsum is the correctly rounded float sum), and min / max.  `overflow` is set when an integer argument of a
passing row leaves int64 anywhere on the way (b * x, a + b * x or a partial product): PostgreSQL raises "bigint out
of range" there.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from fractions import Fraction

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
U = 2.0 ** -53                  # unit roundoff of float8
ETA = 2.0 ** -1074              # smallest subnormal: absolute error allowance of an underflowing operation

COUNT_STAR, COUNT, SUM, MIN, MAX = range(5)


def isnan(x) -> bool:
    return isinstance(x, float) and x != x


def float8_cmp(x: float, y: float) -> int:
    """[PG] float8_cmp_internal: every NaN equals every NaN and sorts above everything; -0.0 equals 0.0"""
    xn, yn = isnan(x), isnan(y)
    if xn or yn:
        return int(xn) - int(yn)
    return (x > y) - (x < y)


def float8_eq(x: float, y: float) -> bool:
    return float8_cmp(x, y) == 0


def _cmp(x, y, is_float: bool) -> int:
    return float8_cmp(float(x), float(y)) if is_float else (x > y) - (x < y)


_OPS = {"<": lambda c: c < 0, "<=": lambda c: c <= 0, "=": lambda c: c == 0,
        ">=": lambda c: c >= 0, ">": lambda c: c > 0, "<>": lambda c: c != 0}


def unpack_two_column_key(packed: int) -> tuple:
    """a packed two-column group key (low 32 bits: first column) -> (first, second), each half sign-extended"""
    u = packed & (2**64 - 1)
    lo, hi = u & 0xffffffff, u >> 32

    def sext(v):
        return v - 2**32 if v >= 2**31 else v
    return sext(lo), sext(hi)


@dataclass
class AggResult:
    count: int = 0
    sum: int = 0                       # integer sum (exact)
    terms: list = field(default_factory=list)     # finite float terms, each evaluated once in float8
    special: list = field(default_factory=list)   # non-finite float terms (NaN, +-inf)
    rounding: int = 0                  # roundings inside one float8 evaluation of a term (b*x, a+, products)
    min: object = None
    max: object = None
    overflow: bool = False

    def float_sum(self) -> float:
        """the correctly rounded sum of the terms; NaN / inf when a term is not finite"""
        if any(isnan(t) for t in self.special) or (math.inf in self.special and -math.inf in self.special):
            return math.nan
        if self.special:
            return self.special[0]
        return math.fsum(self.terms)

    def float_sum_ok(self, got: float) -> bool:
        """|got - fsum| <= ((n - 1) + 2m) * u * sum |term| + n * eta + 1/2 ulp(fsum): the worst case of any summation
        order of n terms, each of which the kernel and this reference evaluate with m roundings of their own.  The
        sign of a zero result is not compared (PostgreSQL's own answer depends on the order of the inputs there)."""
        want = self.float_sum()
        if isnan(want) or math.isinf(want):
            return float8_eq(got, want)
        if isnan(got) or math.isinf(got):
            return False
        n = len(self.terms)
        abs_sum = math.fsum(abs(t) for t in self.terms)
        tol = (max(n - 1, 0) + 2 * self.rounding) * U * abs_sum * 1.01 + ETA * n + math.ulp(want) / 2
        return abs(Fraction(got) - Fraction(want)) <= Fraction(tol)


@dataclass
class Result:
    groups: dict
    rows_passed: int
    rows_removed: int


def _where_value(node, row_vals, row_nulls, float_cols):
    """three-valued: True, False or None (unknown)"""
    if isinstance(node, tuple) and node and node[0] in ("and", "or"):
        vals = [_where_value(arm, row_vals, row_nulls, float_cols) for arm in node[1:]]
        if node[0] == "and":
            if any(v is False for v in vals):
                return False
            return None if any(v is None for v in vals) else True
        if any(v is True for v in vals):
            return True
        return None if any(v is None for v in vals) else False
    col, op, k = node
    if row_nulls[col]:
        return None
    return _OPS[op](_cmp(row_vals[col], k, col in float_cols))


def _int_term(factors, row_vals):
    """exact product and whether any step left int64"""
    prod, over = 1, False
    for f, (col, a, b) in enumerate(factors):
        m = b * int(row_vals[col])
        t = a + m
        over |= not (INT64_MIN <= m <= INT64_MAX and INT64_MIN <= t <= INT64_MAX)
        prod = t if f == 0 else prod * t
        over |= not (INT64_MIN <= prod <= INT64_MAX)
    return prod, over


def _float_term(factors, row_vals):
    """(the term evaluated in float8, left to right, and the roundings that evaluation makes)"""
    t, rounding = 1.0, 0
    for f, (col, a, b) in enumerate(factors):
        x = float(row_vals[col])
        if not (a == 0 and b == 1):
            x = a + b * x
            rounding += 2
        if f:
            t *= x
            rounding += 1
        else:
            t = x
    return t, rounding


def aggregate(cols, nulls, where, group_cols, aggs, float_cols=()) -> Result:
    nrows = len(cols[0]) if cols else 0
    float_cols = set(float_cols)
    cols = [[float(v) if i in float_cols else int(v) for v in (c.tolist() if hasattr(c, "tolist") else c)]
            for i, c in enumerate(cols)]
    nulls = [None if n is None else [bool(v) for v in (n.tolist() if hasattr(n, "tolist") else n)]
             for n in (nulls if nulls is not None else [])]
    nulls += [None] * (len(cols) - len(nulls))
    where = where if (isinstance(where, tuple) and where and where[0] in ("and", "or")) else ("and",) + tuple(where)
    groups = {}
    passed = removed = 0
    for r in range(nrows):
        vals = [c[r] for c in cols]
        isnull = [n[r] if n is not None else False for n in nulls]
        if len(where) > 1 and _where_value(where, vals, isnull, float_cols) is not True:
            removed += 1
            continue
        passed += 1
        key = tuple(None if isnull[c] else (float(vals[c]) if c in float_cols else int(vals[c])) for c in group_cols)
        per = groups.setdefault(key, [AggResult() for _ in aggs])
        for spec, st in zip(aggs, per):
            if spec.kind == COUNT_STAR:
                st.count += 1
                continue
            if any(isnull[c] for c, _, _ in spec.factors):
                continue
            st.count += 1
            if spec.kind == COUNT:
                continue
            if spec.is_float:
                v, st.rounding = _float_term(spec.factors, vals)
                (st.terms if math.isfinite(v) else st.special).append(v)
                if spec.kind == MIN and (st.min is None or float8_cmp(v, st.min) < 0):
                    st.min = v
                if spec.kind == MAX and (st.max is None or float8_cmp(v, st.max) > 0):
                    st.max = v
            else:
                t, over = _int_term(spec.factors, vals)
                st.overflow |= over and spec.kind in (SUM, MIN, MAX)
                st.sum += t
                if spec.kind == MIN and (st.min is None or t < st.min):
                    st.min = t
                if spec.kind == MAX and (st.max is None or t > st.max):
                    st.max = t
    return Result(groups, passed, removed)


def overflows(result: Result) -> bool:
    return any(st.overflow for per in result.groups.values() for st in per)
