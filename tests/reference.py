"""An exact, independent reference of the scan plan language -- the fused scan + partial aggregate -- in plain Python.

It shares no code with oracle/oracle.c and nothing with the library's key packing: rows are evaluated one at a
time with Python integers (no overflow), math.fsum (correctly rounded float sums) and PostgreSQL's float8 btree
order.  Chunk-group skipping is restated from the rows too: selected_chunk_mask computes every chunk's min / max from
the data and the writer's stripe / chunk row limits, never from the skip nodes a writer produced.

    aggregate(cols, nulls, where, group_cols, aggs, float_cols, scales)  ->  Result
    selected_chunk_mask(cols, nulls, where, stripe_row_limit, chunk_row_limit, float_cols)  ->  [[kept?] per chunk] per stripe
    atom_value(atom, vals, isnull, float_cols, scales)  ->  True / False / None (UNKNOWN)
    tree_value(tree, vals, isnull, float_cols, scales)  ->  True / False / None
    var_out(final, n, s, q, scale)                      ->  PostgreSQL's numeric text of a variance, or None for SQL NULL
        cols        list of sequences, one per attribute (ints, or floats for float columns)
        nulls       list of per-row NULL flags per attribute, or None entries / None for no NULLs
        where       a tree ("and" | "or", arm, arm, ...), a list of atoms (their AND), one atom, or None (TRUE)
        group_cols  attribute indexes; groups are keyed by the tuple of key values (None = NULL)
        aggs        objects with .kind (0 count(*), 1 count, 2 sum, 3 min, 4 max, 5 bit_and, 6 bit_or, 7 bool_and,
                    8 bool_or, 9 variance), .factors [(column, a, b)] -- the argument is prod (a + b * column) --,
                    .is_float, and optionally .filter (a tree: FILTER (WHERE ...)), .arg (the tree of bool_and /
                    bool_or) and .case (a columnar.Case argument in place of .factors)
        scales      {column: numeric scale} (0 for the others), for column-to-column atoms

Atoms:
    (column, op, constant)             op one of < <= = >= > <>; UNKNOWN if the column is NULL
    (column, "in" | "not in", (v, ...)) with None for a NULL element
    (column, "is null" | "is not null")
    (column, op, Col(other))           a column-to-column comparison

IN / NOT IN and IS [NOT] NULL follow PostgreSQL's ExecEvalScalarArrayOp and NullTest:

    x IN (...)       UNKNOWN if x is NULL; TRUE if x equals an element; else UNKNOWN if an element is NULL, else FALSE
    x NOT IN (...)   UNKNOWN if x is NULL; FALSE if x equals an element; else UNKNOWN if an element is NULL, else TRUE
    x IS NULL / x IS NOT NULL   never UNKNOWN

with equality in the column's btree order (float8_cmp for floats: NaN = NaN, -0.0 = 0.0).

Column atoms follow PostgreSQL's comparison of two Vars: UNKNOWN when either side is NULL, else the btree comparison.
Integer-like columns (int, bool, numeric(p, s) held as value * 10^s, char(1) as its unsigned byte) compare the
mathematical values, both sides brought to the larger scale with Python's exact integers; float columns compare in
float8 btree order (float8_cmp: NaN = NaN above everything, -0.0 = 0.0).

Aggregates.  A row WHERE does not find TRUE is removed; the others are grouped.  A row an aggregate's FILTER does not
find TRUE is no input of that aggregate (its group still exists: the groups are those of WHERE alone).  The argument's
value is the product of the factors, NULL when a factor column is NULL; or, for a CASE argument, PostgreSQL's CaseExpr
inside Aggref.args: the WHEN trees are evaluated in order under three-valued logic, the value is the result of the
first arm whose tree is TRUE (UNKNOWN is not TRUE), else the ELSE result, else NULL, and only that result is evaluated.
A row the aggregate's FILTER rejects is no input and its CASE is not consulted; a NULL value is no input, and so is a
bool_and / bool_or argument that is UNKNOWN.  Per group and aggregate the result holds
    count       inputs (count(*): rows); 0 is SQL NULL for every kind but count
    sum, min, max, sumsq    of integer inputs, exact; sumsq = sum(x^2) is what CG_AGG_VARIANCE keeps next to N = count
                            and sum(x) = sum
    terms, special, rounding    float inputs: finite terms (their math.fsum is the correctly rounded float sum),
                            non-finite ones, and the most roundings one float8 evaluation of a term makes
    value       bit_and / bit_or (AND / OR of the inputs as Python integers), bool_and (every input TRUE), bool_or
                (some input TRUE); None = no input
`overflow` is set when an integer term of sum / min / max / variance leaves int64 anywhere on the way (b * x, a + b * x
or a partial product), the chosen CASE arm's included: PostgreSQL raises "bigint out of range" there.

Chunk-group skipping restates predtest.c for weak = false: btree range atoms refute as in _atom_refutes_range; IN -- an
OR of "=" arms when the array has at most MAX_SAOP_ARRAY_SIZE = 100 elements, NULLs and duplicates counted -- is
refuted iff no element is NULL and every element lies outside [min, max]; a NullTest is never pushed down (it refutes
nothing), NOT IN (an AND of "<>") refutes nothing, and a Var op Var clause is never pushed down (ExtractPushdownClause
wants a constant side), so a column atom refutes nothing.

var_out restates numeric_stddev_internal (PostgreSQL's numeric.c) from its definition: with N, S = sum(x) and
Q = sum(x^2), all in units of 10^-scale,
    NULL                  when N = 0, or N <= 1 for the sample forms
    num = N * Q - S^2     at display scale 2 * scale; num <= 0 is the numeric zero, text "0"
    den = N * (N - 1) (sample) or N^2 (population), display scale 0
    rscale                select_div_scale(num, den): 16 significant digits counted in base-10000 digits, at least both
                          display scales, within [0, 1000]
    variance              num / den rounded half away from zero at rscale
    stddev                the square root of that rounded variance, rounded half away from zero at rscale
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from fractions import Fraction

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
U = 2.0 ** -53                  # unit roundoff of float8
ETA = 2.0 ** -1074              # smallest subnormal: absolute error allowance of an underflowing operation

COUNT_STAR, COUNT, SUM, MIN, MAX, BIT_AND, BIT_OR, BOOL_AND, BOOL_OR, VARIANCE = range(10)
MAX_SAOP_ARRAY_SIZE = 100


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
    value: object = None               # bit_* / bool_* result, None = no input
    sumsq: int = 0                     # sum(x^2) of the integer inputs (exact)

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


# --------------------------------------------------------------------------- predicates
def _is_tree(node) -> bool:
    return isinstance(node, tuple) and bool(node) and node[0] in ("and", "or")


def _is_column(k) -> bool:
    return type(k).__name__ == "Col"


def as_tree(where):
    """a WHERE / FILTER / WHEN condition in any accepted form -- a tree, a list of atoms (their AND), one atom -- as a
    tree; None when there is no condition"""
    if where is None or _is_tree(where):
        return where
    if not len(where):
        return None
    return ("and",) + tuple(where) if isinstance(where[0], (tuple, list)) else ("and", where)


def atom_value(atom, vals, isnull, float_cols=(), scales=None):
    """one atom on one row (vals / isnull indexed by column): True, False or None (UNKNOWN)"""
    c, op = atom[0], atom[1]
    if op == "is null":
        return bool(isnull[c])
    if op == "is not null":
        return not isnull[c]
    if isnull[c]:
        return None
    k, is_float = atom[2], c in float_cols
    if op in ("in", "not in"):
        if any(e is not None and _cmp(vals[c], e, is_float) == 0 for e in k):
            return op == "in"
        return None if any(e is None for e in k) else op == "not in"
    if _is_column(k):
        if isnull[k.index]:
            return None
        if is_float:
            return _OPS[op](_cmp(vals[c], vals[k.index], True))
        sx, sy = (scales or {}).get(c, 0), (scales or {}).get(k.index, 0)
        s = max(sx, sy)
        x, y = int(vals[c]) * 10 ** (s - sx), int(vals[k.index]) * 10 ** (s - sy)
        return _OPS[op]((x > y) - (x < y))
    return _OPS[op](_cmp(vals[c], k, is_float))


def tree_value(tree, vals, isnull, float_cols=(), scales=None):
    """a WHERE / FILTER / bool_* argument / WHEN condition in any form as_tree accepts, None being TRUE"""
    tree = as_tree(tree)
    if tree is None:
        return True
    v = [atom_value(arm, vals, isnull, float_cols, scales) if isinstance(arm, tuple) and not _is_tree(arm)
         else tree_value(arm, vals, isnull, float_cols, scales) for arm in tree[1:]]
    if tree[0] == "and":
        return False if any(x is False for x in v) else (None if any(x is None for x in v) else True)
    return True if any(x is True for x in v) else (None if any(x is None for x in v) else False)


# --------------------------------------------------------------------------- aggregates
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


def _product(factors, is_float, vals, isnull):
    """(value, overflow?, roundings) of prod (a + b * x) over the factors; value None when a factor column is NULL"""
    if any(isnull[c] for c, _, _ in factors):
        return None, False, 0
    if is_float:
        v, rounding = _float_term(factors, vals)
        return v, False, rounding
    v, over = _int_term(factors, vals)
    return v, over, 0


def _case_value(case, is_float, vals, isnull, float_cols, scales):
    """the result of the first arm whose WHEN tree is TRUE, else ELSE, else NULL; only the chosen result is evaluated"""
    from citus_b200 import columnar
    res = next((r for tree, r in case.arms if tree_value(tree, vals, isnull, float_cols, scales) is True),
               None if case.else_ is columnar._NO_ELSE else case.else_)
    if res is None:
        return None, False, 0
    if type(res).__name__ == "Const":
        return (float(res.value) if is_float else int(res.value)), False, 0
    return _product([(res, 0, 1)] if isinstance(res, int) else list(res), is_float, vals, isnull)


def _input(spec, vals, isnull, float_cols, scales):
    """(value, overflow?, roundings) of one aggregate's argument on one row that passed its FILTER; None = no input"""
    if spec.kind in (BOOL_AND, BOOL_OR):
        return tree_value(spec.arg, vals, isnull, float_cols, scales), False, 0
    if getattr(spec, "case", None) is not None:
        return _case_value(spec.case, spec.is_float, vals, isnull, float_cols, scales)
    if spec.kind == COUNT:                       # count(x) reads only the NULL flags: x may be a float column
        return (None if any(isnull[c] for c, _, _ in spec.factors) else 0), False, 0
    return _product(spec.factors, spec.is_float, vals, isnull)


def _accumulate(st: AggResult, kind, is_float, v, over, rounding):
    if kind == COUNT:
        return
    if kind in (BIT_AND, BIT_OR, BOOL_AND, BOOL_OR):
        if st.value is None:
            st.value = v
        elif kind == BIT_AND:
            st.value &= v
        elif kind == BIT_OR:
            st.value |= v
        else:
            st.value = (st.value and v) if kind == BOOL_AND else (st.value or v)
    elif is_float:
        st.rounding = max(st.rounding, rounding)
        (st.terms if math.isfinite(v) else st.special).append(v)
        if kind == MIN and (st.min is None or float8_cmp(v, st.min) < 0):
            st.min = v
        if kind == MAX and (st.max is None or float8_cmp(v, st.max) > 0):
            st.max = v
    else:
        st.overflow |= over
        st.sum += v
        st.sumsq += v * v
        if kind == MIN and (st.min is None or v < st.min):
            st.min = v
        if kind == MAX and (st.max is None or v > st.max):
            st.max = v


def _rows(col):
    return col.tolist() if hasattr(col, "tolist") else list(col)


def aggregate(cols, nulls, where, group_cols, aggs, float_cols=(), scales=None) -> Result:
    nrows = len(cols[0]) if len(cols) else 0
    float_cols = set(float_cols)
    cols = [[float(v) if i in float_cols else int(v) for v in _rows(c)] for i, c in enumerate(cols)]
    nulls = [None if n is None else [bool(v) for v in _rows(n)] for n in (nulls if nulls is not None else [])]
    nulls += [None] * (len(cols) - len(nulls))
    where = as_tree(where)
    groups = {}
    passed = removed = 0
    for r in range(nrows):
        vals = [c[r] for c in cols]
        isnull = [n[r] if n is not None else False for n in nulls]
        if tree_value(where, vals, isnull, float_cols, scales) is not True:
            removed += 1
            continue
        passed += 1
        key = tuple(None if isnull[c] else vals[c] for c in group_cols)
        per = groups.setdefault(key, [AggResult() for _ in aggs])
        for spec, st in zip(aggs, per):
            if tree_value(getattr(spec, "filter", None), vals, isnull, float_cols, scales) is not True:
                continue
            if spec.kind == COUNT_STAR:
                st.count += 1
                continue
            v, over, rounding = _input(spec, vals, isnull, float_cols, scales)
            if v is None:
                continue
            st.count += 1
            _accumulate(st, spec.kind, spec.is_float, v, over, rounding)
    return Result(groups, passed, removed)


def overflows(result: Result) -> bool:
    return any(st.overflow for per in result.groups.values() for st in per)


# --------------------------------------------------------------------------- variance final functions
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


# --------------------------------------------------------------------------- chunk-group skipping
def chunk_layout(nrows: int, stripe_row_limit: int, chunk_row_limit: int) -> list:
    """[(first row, rows) per chunk group] per stripe, as the writer cuts one INSERT: a stripe is closed after
    stripe_row_limit rows and a chunk group after chunk_row_limit rows of its stripe"""
    stripes = []
    for s0 in range(0, nrows, stripe_row_limit):
        s1 = min(nrows, s0 + stripe_row_limit)
        stripes.append([(c0, min(s1, c0 + chunk_row_limit) - c0) for c0 in range(s0, s1, chunk_row_limit)])
    return stripes


def chunk_minmax(values, isnull, first: int, rows: int, is_float: bool):
    """(min, max) of the non-NULL values of one column chunk in the type's btree order, None when all are NULL"""
    lo = hi = None
    for r in range(first, first + rows):
        if isnull is not None and isnull[r]:
            continue
        v = values[r]
        if lo is None or _cmp(v, lo, is_float) < 0:
            lo = v
        if hi is None or _cmp(v, hi, is_float) > 0:
            hi = v
    return None if lo is None else (lo, hi)


def _atom_refutes_range(op, k, lo, hi, is_float) -> bool:
    """[PG] btree refutation of the base constraint (col >= lo AND col <= hi) by one atom `col op k`: the atom
    refutes one half when no value of that half can satisfy it; `<>` refutes neither half"""
    if op == "<":
        return _cmp(lo, k, is_float) >= 0
    if op == "<=":
        return _cmp(lo, k, is_float) > 0
    if op == "=":
        return _cmp(k, lo, is_float) < 0 or _cmp(k, hi, is_float) > 0
    if op == ">=":
        return _cmp(hi, k, is_float) < 0
    if op == ">":
        return _cmp(hi, k, is_float) <= 0
    return False


def _atom_refutes(atom, lo, hi, is_float) -> bool:
    """IN as the OR of its "=" arms (at most MAX_SAOP_ARRAY_SIZE elements, none NULL); NOT IN, IS [NOT] NULL and
    column atoms refute nothing"""
    op = atom[1]
    if op == "in":
        elems = atom[2]
        return (len(elems) <= MAX_SAOP_ARRAY_SIZE and not any(e is None for e in elems)
                and all(_atom_refutes_range("=", e, lo, hi, is_float) for e in elems))
    if op not in _OPS or _is_column(atom[2]):
        return False
    return _atom_refutes_range(op, atom[2], lo, hi, is_float)


def _refuted(node, col, lo, hi, float_cols) -> bool:
    """[PG] predicate_refuted_by(one column's base constraint, WHERE tree): an AND node is refuted when any arm is,
    an OR node when every arm is; an atom on another column refutes nothing"""
    if _is_tree(node):
        arms = [_refuted(arm, col, lo, hi, float_cols) for arm in node[1:]]
        return any(arms) if node[0] == "and" else all(arms)
    return node[0] == col and _atom_refutes(node, lo, hi, col in float_cols)


def _atoms(node):
    if _is_tree(node):
        return [a for arm in node[1:] for a in _atoms(arm)]
    return [node]


def skip_minmax(cols, nulls, stripe_row_limit, chunk_row_limit, float_cols=()) -> list:
    """[column][stripe][chunk] -> (min, max) or None: what a faithful writer puts in the skip nodes"""
    float_cols = set(float_cols)
    nulls = list(nulls if nulls is not None else []) + [None] * (len(cols) - len(nulls or []))
    layout = chunk_layout(len(cols[0]) if len(cols) else 0, stripe_row_limit, chunk_row_limit)
    out = []
    for c, col in enumerate(cols):
        vals = [float(v) for v in _rows(col)] if c in float_cols else [int(v) for v in _rows(col)]
        isnull = None if nulls[c] is None else _rows(nulls[c])
        out.append([[chunk_minmax(vals, isnull, f, n, c in float_cols) for f, n in stripe] for stripe in layout])
    return out


def selected_chunk_mask(cols, nulls, where, stripe_row_limit, chunk_row_limit, float_cols=(), qual_pushdown=True,
                        minmax=None):
    """columnar_reader.c:1132-1187 SelectedChunkMask for every stripe of a relation written by one INSERT of these
    rows: [[kept?] per chunk group] per stripe.  Each column's per-chunk min / max come from the rows themselves (an
    all-NULL chunk has none and is never refuted; so is a column added after the stripe was written, whose rows
    read as NULL).  A chunk group is dropped when the base constraint of any WHERE column is refuted.  `minmax`:
    skip_minmax of the same arguments, when many WHERE trees run over one relation."""
    float_cols = set(float_cols)
    if minmax is None:
        minmax = skip_minmax(cols, nulls, stripe_row_limit, chunk_row_limit, float_cols)
    where = as_tree(where)
    qual_cols = sorted({a[0] for a in _atoms(where)}) if where is not None and qual_pushdown else []
    out = []
    for s, stripe in enumerate(chunk_layout(len(cols[0]) if len(cols) else 0, stripe_row_limit, chunk_row_limit)):
        mask = []
        for k in range(len(stripe)):
            mask.append(not any(minmax[c][s][k] is not None and _refuted(where, c, *minmax[c][s][k], float_cols)
                                for c in qual_cols))
        out.append(mask)
    return out


def chunks_filtered(mask) -> int:
    """"Columnar Chunk Groups Removed by Filter" of a selected_chunk_mask result"""
    return sum(not k for stripe in mask for k in stripe)


def rows_kept(mask, nrows, stripe_row_limit, chunk_row_limit) -> int:
    """rows of the chunk groups a selected_chunk_mask result keeps (the rows handed to the qual)"""
    layout = chunk_layout(nrows, stripe_row_limit, chunk_row_limit)
    return sum(rows for lay, stripe in zip(layout, mask) for (_, rows), k in zip(lay, stripe) if k)
