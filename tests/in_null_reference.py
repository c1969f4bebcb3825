"""Exact reference of the IN / NOT IN list and IS [NOT] NULL atoms, on top of tests/reference.py and
tests/bool_bit_reference.py.

    atom_value(atom, value, isnull, is_float)                    ->  True / False / None (UNKNOWN)
    aggregate(cols, nulls, where, group_cols, aggs, float_cols)  ->  reference.Result, every FILTER applied
    selected_chunk_mask(cols, nulls, where, stripe_row_limit, chunk_row_limit, float_cols, minmax)  ->  [[kept?]] per stripe

Atoms: (column, "in" | "not in", (v, ...)) with None for a NULL element, and (column, "is null" | "is not null"), next to
the (column, op, constant) atoms reference.py knows.  Rows follow PostgreSQL's ExecEvalScalarArrayOp and NullTest:

    x IN (...)       UNKNOWN if x is NULL; TRUE if x equals an element; else UNKNOWN if an element is NULL, else FALSE
    x NOT IN (...)   UNKNOWN if x is NULL; FALSE if x equals an element; else UNKNOWN if an element is NULL, else TRUE
    x IS NULL / x IS NOT NULL   never UNKNOWN

with equality in the column's btree order (reference.float8_cmp for floats: NaN = NaN, -0.0 = 0.0).  aggregate() turns
every new atom into a virtual column holding its three-valued result (1 / 0 / NULL) and the atom into "virtual = 1", which
is TRUE, FALSE or UNKNOWN exactly when the atom is, then runs bool_bit_reference over the widened rows.

Chunk-group skipping restates predtest.c for weak = false: a NullTest is never pushed down (it refutes nothing), NOT IN
(an AND of "<>") refutes nothing, and IN -- an OR of "=" arms when the array has at most MAX_SAOP_ARRAY_SIZE = 100
elements, NULLs and duplicates counted -- is refuted iff no element is NULL and every element lies outside [min, max].
"""
from __future__ import annotations

import bool_bit_reference as bref
import reference as ref

MAX_SAOP_ARRAY_SIZE = 100
NEW_OPS = ("in", "not in", "is null", "is not null")


def is_new(atom) -> bool:
    return isinstance(atom, tuple) and len(atom) >= 2 and atom[1] in NEW_OPS


def atom_value(atom, value, isnull, is_float):
    op = atom[1]
    if op == "is null":
        return bool(isnull)
    if op == "is not null":
        return not isnull
    if isnull:
        return None
    elems = atom[2]
    found = any(e is not None and ref._cmp(value, e, is_float) == 0 for e in elems)
    has_null = any(e is None for e in elems)
    if op == "in":
        return True if found else (None if has_null else False)
    return False if found else (None if has_null else True)


def _map_tree(node, fn):
    if node is None:
        return None
    if isinstance(node, tuple) and node and node[0] in ("and", "or"):
        return (node[0],) + tuple(_map_tree(arm, fn) for arm in node[1:])
    if isinstance(node, list):
        return [_map_tree(a, fn) for a in node]
    return fn(node)


def _rows(c):
    return c.tolist() if hasattr(c, "tolist") else list(c)


class _Agg:
    def __init__(self, a, filt, arg):
        self.kind, self.factors, self.is_float = a.kind, list(getattr(a, "factors", [])), getattr(a, "is_float", False)
        self.filter, self.arg = filt, arg


def aggregate(cols, nulls, where, group_cols, aggs, float_cols=()) -> ref.Result:
    """reference.Result of the query with the new atoms anywhere: WHERE, FILTERs, bool_and / bool_or arguments"""
    float_cols = set(float_cols)
    n = len(cols[0]) if cols else 0
    cols = [_rows(c) for c in cols]
    nulls = [None if x is None else _rows(x) for x in (nulls or [])] + [None] * (len(cols) - len(nulls or []))
    extra_vals, extra_nulls, index = [], [], {}

    def virtual(atom):
        if not is_new(atom):
            return atom
        atom = (atom[0], atom[1]) + ((tuple(atom[2]),) if len(atom) > 2 else ())
        if atom not in index:
            c = atom[0]
            res = [atom_value(atom, cols[c][r], bool(nulls[c][r]) if nulls[c] is not None else False, c in float_cols)
                   for r in range(n)]
            index[atom] = len(cols) + len(extra_vals)
            extra_vals.append([1 if v else 0 for v in res])
            extra_nulls.append([v is None for v in res])
        return (index[atom], "=", 1)

    w = _map_tree(where, virtual)
    new_aggs = [_Agg(a, _map_tree(getattr(a, "filter", None), virtual), _map_tree(getattr(a, "arg", None), virtual)) for a in aggs]
    return bref.filtered(cols + extra_vals, nulls + extra_nulls, w, group_cols, new_aggs, float_cols)


def _atom_refutes(atom, lo, hi, is_float) -> bool:
    if not is_new(atom):
        return ref._atom_refutes_range(atom[1], atom[2], lo, hi, is_float)
    if atom[1] != "in":
        return False
    elems = atom[2]
    if len(elems) > MAX_SAOP_ARRAY_SIZE or any(e is None for e in elems):
        return False
    return all(ref._cmp(e, lo, is_float) < 0 or ref._cmp(e, hi, is_float) > 0 for e in elems)


def _refuted(node, col, lo, hi, float_cols) -> bool:
    if isinstance(node, tuple) and node and node[0] in ("and", "or"):
        arms = [_refuted(arm, col, lo, hi, float_cols) for arm in node[1:]]
        return any(arms) if node[0] == "and" else all(arms)
    return node[0] == col and _atom_refutes(node, lo, hi, col in float_cols)


def selected_chunk_mask(cols, nulls, where, stripe_row_limit, chunk_row_limit, float_cols=(), qual_pushdown=True, minmax=None):
    """reference.selected_chunk_mask with the new atoms' refutation rules"""
    float_cols = set(float_cols)
    if minmax is None:
        minmax = ref.skip_minmax(cols, nulls, stripe_row_limit, chunk_row_limit, float_cols)
    where = where if (isinstance(where, tuple) and where and where[0] in ("and", "or")) else ("and",) + tuple(where)
    qual_cols = sorted({a[0] for a in ref._atoms(where)}) if len(where) > 1 else []
    out = []
    for s, stripe in enumerate(ref.chunk_layout(len(cols[0]) if len(cols) else 0, stripe_row_limit, chunk_row_limit)):
        mask = []
        for k in range(len(stripe)):
            kept = True
            if qual_pushdown:
                for c in qual_cols:
                    mm = minmax[c][s][k]
                    if mm is not None and _refuted(where, c, mm[0], mm[1], float_cols):
                        kept = False
                        break
            mask.append(kept)
        out.append(mask)
    return out
