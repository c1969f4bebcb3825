"""Exact reference of bit_and / bit_or / bool_and / bool_or (every), on top of tests/reference.py.

    aggregate(cols, nulls, where, group_cols, aggs, float_cols)  ->  reference.Result
    filtered(cols, nulls, where, group_cols, aggs, float_cols)   ->  the same with every aggregate's FILTER applied

The kinds reference.aggregate knows (count(*), count, sum, min, max) are computed by it; the four new kinds are
computed here, one row at a time, over the same groups and with the same three-valued predicate evaluation:
        5 bit_and / 6 bit_or    .factors = [(column, 0, 1)]: AND / OR of the non-NULL values as Python integers
        7 bool_and / 8 bool_or  .arg = a WHERE-style predicate tree: a row whose predicate is UNKNOWN is no input;
                                bool_and = every input TRUE, bool_or = some input TRUE
Each new aggregate's result carries `count` (inputs; 0 = SQL NULL) and `value` (int or bool; None = no input).
"""
from __future__ import annotations

import reference as ref

BIT_AND, BIT_OR, BOOL_AND, BOOL_OR = range(5, 9)
NEW = (BIT_AND, BIT_OR, BOOL_AND, BOOL_OR)


def as_tree(where):
    """a WHERE-style condition in any accepted form -- tree, list of atoms (their AND), one atom -- as a tree (None =
    no condition)"""
    if isinstance(where, tuple) and where and where[0] in ("and", "or"):
        return where
    if isinstance(where, tuple):
        return ("and", where)
    return ("and",) + tuple(where) if where else None


class _CountStar:
    """stands in for a new aggregate in reference.aggregate (which then only keeps the groups and the counters)"""
    kind, factors, is_float = ref.COUNT_STAR, [], False


def _rows(c):
    return c.tolist() if hasattr(c, "tolist") else list(c)


def aggregate(cols, nulls, where, group_cols, aggs, float_cols=()) -> ref.Result:
    res = ref.aggregate(cols, nulls, where, group_cols, [_CountStar() if a.kind in NEW else a for a in aggs], float_cols)
    new = [j for j, a in enumerate(aggs) if a.kind in NEW]
    for per in res.groups.values():
        for j in new:
            per[j] = ref.AggResult()
            per[j].value = None
    if not new:
        return res
    float_cols = set(float_cols)
    vals_of = [[float(v) if i in float_cols else int(v) for v in _rows(c)] for i, c in enumerate(cols)]
    null_of = [None if n is None else [bool(v) for v in _rows(n)] for n in (nulls or [])]
    null_of += [None] * (len(cols) - len(null_of))
    w = as_tree(where)
    for r in range(len(cols[0]) if cols else 0):
        vals = [c[r] for c in vals_of]
        isnull = [n[r] if n is not None else False for n in null_of]
        if w is not None and ref._where_value(w, vals, isnull, float_cols) is not True:
            continue
        key = tuple(None if isnull[c] else (float(vals[c]) if c in float_cols else int(vals[c])) for c in group_cols)
        per = res.groups[key]
        for j in new:
            spec, st = aggs[j], per[j]
            if spec.kind in (BOOL_AND, BOOL_OR):
                v = ref._where_value(as_tree(spec.arg), vals, isnull, float_cols)
                if v is None:                                    # UNKNOWN: no input, like a NULL argument
                    continue
                st.value = v if st.value is None else (st.value and v) if spec.kind == BOOL_AND else (st.value or v)
            else:
                (col, a, b), = spec.factors
                assert (a, b) == (0, 1) and col not in float_cols, "bit_and / bit_or take one bare integer column"
                if isnull[col]:
                    continue
                v = int(vals[col])
                st.value = v if st.value is None else (st.value & v) if spec.kind == BIT_AND else (st.value | v)
            st.count += 1
    return res


def filtered(cols, nulls, where, group_cols, aggs, float_cols=()) -> ref.Result:
    """PostgreSQL's FILTER by composition: the groups are those of WHERE alone; aggregate j of a group is the aggregate
    over (WHERE AND FILTER_j), or no input (count 0, SQL NULL) where that has no row of the group"""
    res = aggregate(cols, nulls, where, group_cols, aggs, float_cols)
    w = as_tree(where)
    for j, a in enumerate(aggs):
        if getattr(a, "filter", None) is None:
            continue
        f = as_tree(a.filter)
        sub = aggregate(cols, nulls, ("and", w, f) if w else f, group_cols, [a], float_cols)
        for key, per in res.groups.items():
            if key in sub.groups:
                per[j] = sub.groups[key][0]
            else:
                per[j] = ref.AggResult()
                per[j].value = None
    return res
