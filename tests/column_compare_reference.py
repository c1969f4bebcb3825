"""Exact reference of the column-to-column atoms (column, op, Col(other)), on top of tests/in_null_reference.py (which
builds on tests/reference.py and tests/bool_bit_reference.py).

    atom_value(op, x, x_null, y, y_null, kind, sx, sy)                        ->  True / False / None (UNKNOWN)
    aggregate(cols, nulls, where, group_cols, aggs, float_cols, scales)       ->  reference.Result, every FILTER applied
    selected_chunk_mask(cols, nulls, where, stripe_row_limit, chunk_row_limit, float_cols, minmax)  ->  [[kept?]] per stripe

Rows follow PostgreSQL's comparison of two Vars: UNKNOWN when either side is NULL, else the btree comparison.  Integer-like
columns (int, bool, numeric(p, s) held as value * 10^s, char(1) as its unsigned byte) compare the mathematical values,
both sides brought to the larger scale with Python's exact integers; float columns compare in float8 btree order
(reference.float8_cmp: NaN = NaN above everything, -0.0 = 0.0).  aggregate() turns every column atom into a virtual column
holding its three-valued result (1 / 0 / NULL) and the atom into "virtual = 1", then hands the query to in_null_reference.

Chunk-group skipping: a Var op Var clause is never pushed down (ExtractPushdownClause wants a constant side), so a column
atom refutes nothing: it is replaced by "column IS NOT NULL", which refutes nothing either and names the same column.
"""
from __future__ import annotations

import in_null_reference as iref
import reference as ref

OPS = ("<", "<=", "=", ">=", ">", "<>")


def is_column_atom(atom) -> bool:
    return isinstance(atom, tuple) and len(atom) == 3 and type(atom[2]).__name__ == "Col" and atom[1] in OPS


def atom_value(op, x, x_null, y, y_null, is_float, sx=0, sy=0):
    if x_null or y_null:
        return None
    if is_float:
        c = ref._cmp(float(x), float(y), True)
    else:
        s = max(sx, sy)
        a, b = int(x) * 10 ** (s - sx), int(y) * 10 ** (s - sy)
        c = (a > b) - (a < b)
    return {"<": c < 0, "<=": c <= 0, "=": c == 0, ">=": c >= 0, ">": c > 0, "<>": c != 0}[op]


def _rows(c):
    return c.tolist() if hasattr(c, "tolist") else list(c)


class _Agg:
    def __init__(self, a, filt, arg):
        self.kind, self.factors, self.is_float = a.kind, list(getattr(a, "factors", [])), getattr(a, "is_float", False)
        self.filter, self.arg = filt, arg


def aggregate(cols, nulls, where, group_cols, aggs, float_cols=(), scales=None) -> ref.Result:
    """reference.Result of the query with column atoms anywhere: WHERE, FILTERs, bool_and / bool_or arguments.  scales:
    {column: numeric scale} (0 for the others)"""
    float_cols, scales = set(float_cols), dict(scales or {})
    n = len(cols[0]) if cols else 0
    cols = [_rows(c) for c in cols]
    nulls = [None if x is None else _rows(x) for x in (nulls or [])] + [None] * (len(cols) - len(nulls or []))
    extra_vals, extra_nulls, index = [], [], {}

    def virtual(atom):
        if not is_column_atom(atom):
            return atom
        key = (atom[0], atom[1], atom[2].index)
        if key not in index:
            a, op, b = key
            za, zb = nulls[a], nulls[b]
            res = [atom_value(op, cols[a][r], bool(za[r]) if za is not None else False, cols[b][r], bool(zb[r]) if zb is not None else False,
                              a in float_cols, scales.get(a, 0), scales.get(b, 0)) for r in range(n)]
            index[key] = len(cols) + len(extra_vals)
            extra_vals.append([1 if v else 0 for v in res])
            extra_nulls.append([v is None for v in res])
        return (index[key], "=", 1)

    w = iref._map_tree(where, virtual)
    new_aggs = [_Agg(a, iref._map_tree(getattr(a, "filter", None), virtual), iref._map_tree(getattr(a, "arg", None), virtual)) for a in aggs]
    return iref.aggregate(cols + extra_vals, nulls + extra_nulls, w, group_cols, new_aggs, float_cols)


def unpushed(where):
    """the WHERE tree as chunk-group skipping sees it: every column atom refutes nothing"""
    return iref._map_tree(where, lambda atom: (atom[0], "is not null") if is_column_atom(atom) else atom)


def selected_chunk_mask(cols, nulls, where, stripe_row_limit, chunk_row_limit, float_cols=(), qual_pushdown=True, minmax=None):
    """in_null_reference.selected_chunk_mask with column atoms refuting nothing"""
    return iref.selected_chunk_mask(cols, nulls, unpushed(where), stripe_row_limit, chunk_row_limit, float_cols=float_cols,
                                    qual_pushdown=qual_pushdown, minmax=minmax)
