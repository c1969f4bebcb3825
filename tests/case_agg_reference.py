"""Exact reference of CASE aggregate arguments (columnar.Case), on the atom evaluation of tests/in_null_reference.py and
tests/column_compare_reference.py.

    atom_value(atom, vals, isnull, float_cols, scales)                        ->  True / False / None (UNKNOWN)
    tree_value(tree, vals, isnull, float_cols, scales)                        ->  True / False / None
    case_value(case, is_float, vals, isnull, float_cols, scales)              ->  (NULL?, value, overflow?, roundings)
    aggregate(cols, nulls, where, group_cols, aggs, float_cols, scales)       ->  reference.Result

Rows follow PostgreSQL's CaseExpr inside Aggref.args: the WHEN trees are evaluated in order under three-valued logic, the
value is the result of the first arm whose tree is TRUE (UNKNOWN is not TRUE), else the ELSE result, else NULL, and only
that result is evaluated.  A product result is NULL when a factor column is NULL; an integer product that leaves int64 at
any step is an overflow (PostgreSQL's "bigint out of range") only when its arm was chosen.  A row the aggregate's FILTER
rejects is no input and its CASE is not consulted; a NULL value is no input.  Per group the reference keeps exact Python
integers: count, sum, min, max, and for CG_AGG_VARIANCE also sumsq = sum(x^2) (N is count, sum(x) is sum).  Float values
follow reference.AggResult's terms (float sum tolerance) and float8 btree order for min / max.  Plain aggregates (no Case)
are evaluated the same way, so queries may mix both.
"""
from __future__ import annotations

import math

import column_compare_reference as ccref
import in_null_reference as iref
import reference as ref

COUNT_STAR, COUNT, SUM, MIN, MAX, VARIANCE = 0, 1, 2, 3, 4, 9
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


def atom_value(atom, vals, isnull, float_cols=(), scales=None):
    scales = scales or {}
    c = atom[0]
    if ccref.is_column_atom(atom):
        b = atom[2].index
        return ccref.atom_value(atom[1], vals[c], isnull[c], vals[b], isnull[b], c in float_cols, scales.get(c, 0), scales.get(b, 0))
    if iref.is_new(atom):
        return iref.atom_value(atom, vals[c], isnull[c], c in float_cols)
    if isnull[c]:
        return None
    return ref._OPS[atom[1]](ref._cmp(vals[c], atom[2], c in float_cols))


def tree_value(tree, vals, isnull, float_cols=(), scales=None):
    """a WHERE / FILTER / WHEN tree: ("and" | "or", arm, ...), a list of atoms (their AND), one atom, or None (TRUE)"""
    if tree is None:
        return True
    if isinstance(tree, list):
        tree = ("and", *tree) if len(tree) != 1 else tree[0]
        if tree == ("and",):
            return True
    if isinstance(tree, tuple) and tree and tree[0] in ("and", "or"):
        v = [tree_value(arm, vals, isnull, float_cols, scales) for arm in tree[1:]]
        if tree[0] == "and":
            return False if any(x is False for x in v) else (None if any(x is None for x in v) else True)
        return True if any(x is True for x in v) else (None if any(x is None for x in v) else False)
    return atom_value(tree, vals, isnull, float_cols, scales)


def _product(factors, is_float, vals, isnull):
    """(NULL?, value, overflow?, roundings) of prod (a + b * x) over the factors"""
    if any(isnull[c] for c, _, _ in factors):
        return True, None, False, 0
    if is_float:
        v, rounding = ref._float_term(factors, vals)
        return False, v, False, rounding
    v, over = ref._int_term(factors, vals)
    return False, v, over, 0


def _result(res, is_float, vals, isnull):
    if res is None:
        return True, None, False, 0
    if type(res).__name__ == "Const":
        return False, (float(res.value) if is_float else int(res.value)), False, 0
    factors = [(res, 0, 1)] if isinstance(res, int) else list(res)
    return _product(factors, is_float, vals, isnull)


def _has_else(case) -> bool:
    from citus_b200 import columnar
    return case.else_ is not columnar._NO_ELSE


def case_value(case, is_float, vals, isnull, float_cols=(), scales=None):
    """first arm whose WHEN tree is TRUE, else ELSE, else NULL; only the chosen result is evaluated"""
    for tree, res in case.arms:
        if tree_value(tree, vals, isnull, float_cols, scales) is True:
            return _result(res, is_float, vals, isnull)
    if not _has_else(case):
        return True, None, False, 0
    return _result(case.else_, is_float, vals, isnull)


def _value(spec, vals, isnull, float_cols, scales):
    case = getattr(spec, "case", None)
    if case is None:
        return _product(spec.factors, spec.is_float, vals, isnull)
    return case_value(case, spec.is_float, vals, isnull, float_cols, scales)


def _rows(c):
    return c.tolist() if hasattr(c, "tolist") else list(c)


def aggregate(cols, nulls, where, group_cols, aggs, float_cols=(), scales=None) -> ref.Result:
    float_cols = set(float_cols)
    n = len(cols[0]) if cols else 0
    cols = [[float(v) if i in float_cols else int(v) for v in _rows(c)] for i, c in enumerate(cols)]
    nulls = [None if x is None else [bool(v) for v in _rows(x)] for x in (nulls or [])] + [None] * (len(cols) - len(nulls or []))
    groups, passed, removed = {}, 0, 0
    for r in range(n):
        vals = [c[r] for c in cols]
        isnull = [z[r] if z is not None else False for z in nulls]
        if tree_value(list(where) if not isinstance(where, tuple) else where, vals, isnull, float_cols, scales) is not True:
            removed += 1
            continue
        passed += 1
        key = tuple(None if isnull[c] else vals[c] for c in group_cols)
        per = groups.get(key)
        if per is None:
            per = groups[key] = [ref.AggResult() for _ in aggs]
            for st in per:
                st.sumsq = 0
        for spec, st in zip(aggs, per):
            if getattr(spec, "filter", None) is not None and tree_value(spec.filter, vals, isnull, float_cols, scales) is not True:
                continue
            if spec.kind == COUNT_STAR:
                st.count += 1
                continue
            isn, v, over, rounding = _value(spec, vals, isnull, float_cols, scales)
            if isn:
                continue
            st.count += 1
            if spec.kind == COUNT:
                continue
            if spec.is_float:
                st.rounding = max(st.rounding, rounding)
                (st.terms if math.isfinite(v) else st.special).append(v)
                if spec.kind == MIN and (st.min is None or ref.float8_cmp(v, st.min) < 0):
                    st.min = v
                if spec.kind == MAX and (st.max is None or ref.float8_cmp(v, st.max) > 0):
                    st.max = v
                continue
            st.overflow |= over
            st.sum += v
            st.sumsq += v * v
            if spec.kind == MIN and (st.min is None or v < st.min):
                st.min = v
            if spec.kind == MAX and (st.max is None or v > st.max):
                st.max = v
    return ref.Result(groups, passed, removed)
