"""The rows a WHERE tree keeps, vectorised: a three-valued mask over decoded columns and the projected rows it selects,
for checking the row-emitting scan (cg_scan_shard_rows) on shards of millions of rows.

It restates tests/reference.py's atom_value / tree_value over whole columns with numpy (test_scan_rows_reference_host.py
checks the two against each other row by row), in the same atom and tree language:

    where_mask(where, vals, nulls, float_cols, scales)   -> bool array: the rows whose tree is TRUE
    tree_masks(tree, vals, nulls, float_cols, scales)    -> (is TRUE, is FALSE) bool arrays; neither = UNKNOWN
    expected_rows(vals, nulls, where, atts, float_cols, scales) -> (values, nulls) per output column

        vals    one array per attribute: int64 (the decoded integer-like value: bool 0 / 1, char(1) as its unsigned byte,
                numeric(p, s) as value * 10^s), or float64 for float columns
        nulls   one array of 0 / 1 per attribute, or None entries / None for no NULLs

Three-valued logic as PostgreSQL's ExecQual: an AND is FALSE when an arm is FALSE and TRUE when every arm is; an OR the
other way round; a row passes only when the tree is TRUE.  Float columns compare in float8 btree order (every NaN equals
every NaN and sorts above everything, -0.0 equals 0.0).  Column atoms of integer-like columns compare the mathematical
values, both sides brought to the larger numeric scale with exact Python integers.

The projected rows are in the form the library emits: int64 values, float columns as their float8 bits, 0 in the value
slot of a NULL, and one 0 / 1 byte per row and column for NULL.
"""
from __future__ import annotations

import numpy as np

_OPS = {"<": lambda c: c < 0, "<=": lambda c: c <= 0, "=": lambda c: c == 0,
        ">=": lambda c: c >= 0, ">": lambda c: c > 0, "<>": lambda c: c != 0}


def _is_tree(node) -> bool:
    return isinstance(node, tuple) and bool(node) and node[0] in ("and", "or")


def _as_tree(where):
    if where is None or _is_tree(where):
        return where
    if not len(where):
        return None
    return ("and",) + tuple(where) if isinstance(where[0], (tuple, list)) else ("and", where)


def _cmp(x, y, is_float):
    """sign of x - y element-wise (y an array or a scalar), in the column's btree order"""
    if not is_float:
        return (x > y).astype(np.int8) - (x < y).astype(np.int8)
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    xn, yn = np.isnan(x), np.isnan(y)
    plain = (x > y).astype(np.int8) - (x < y).astype(np.int8)
    return np.where(xn | yn, xn.astype(np.int8) - yn.astype(np.int8), plain)


def _null(nulls, c, n):
    if nulls is None or nulls[c] is None:
        return np.zeros(n, bool)
    return np.asarray(nulls[c]).astype(bool)


def atom_masks(atom, vals, nulls, float_cols=(), scales=None):
    """(is TRUE, is FALSE) of one atom over every row"""
    c, op = atom[0], atom[1]
    n = len(vals[c])
    isnull = _null(nulls, c, n)
    if op in ("is null", "is not null"):
        t = isnull if op == "is null" else ~isnull
        return t, ~t
    is_float = c in float_cols
    k = atom[2]
    x = vals[c]
    if op in ("in", "not in"):
        found = np.zeros(n, bool)
        for e in k:
            if e is not None:
                found |= _cmp(x, e, is_float) == 0
        has_null = any(e is None for e in k)
        if op == "in":
            t, f = found, ~found & (not has_null)
        else:
            t, f = ~found & (not has_null), found
        return t & ~isnull, f & ~isnull
    if type(k).__name__ == "Col":
        known = ~isnull & ~_null(nulls, k.index, n)
        y = vals[k.index]
        if is_float:
            r = _OPS[op](_cmp(x, y, True))
        else:
            sx, sy = (scales or {}).get(c, 0), (scales or {}).get(k.index, 0)
            s = max(sx, sy)
            if sx == sy:
                r = _OPS[op](_cmp(np.asarray(x, np.int64), np.asarray(y, np.int64), False))
            else:
                xs = np.array([int(v) * 10 ** (s - sx) for v in x], dtype=object)
                ys = np.array([int(v) * 10 ** (s - sy) for v in y], dtype=object)
                r = _OPS[op](np.array([(a > b) - (a < b) for a, b in zip(xs, ys)], np.int8))
        return r & known, ~r & known
    r = _OPS[op](_cmp(x, k, is_float))
    return r & ~isnull, ~r & ~isnull


def tree_masks(tree, vals, nulls, float_cols=(), scales=None):
    """(is TRUE, is FALSE) of a tree in any form the reference accepts; None is TRUE everywhere"""
    tree = _as_tree(tree)
    n = len(vals[0])
    if tree is None:
        return np.ones(n, bool), np.zeros(n, bool)
    arms = [atom_masks(arm, vals, nulls, float_cols, scales) if isinstance(arm, tuple) and not _is_tree(arm)
            else tree_masks(arm, vals, nulls, float_cols, scales) for arm in tree[1:]]
    if tree[0] == "and":
        return np.logical_and.reduce([t for t, _ in arms]), np.logical_or.reduce([f for _, f in arms])
    return np.logical_or.reduce([t for t, _ in arms]), np.logical_and.reduce([f for _, f in arms])


def where_mask(where, vals, nulls, float_cols=(), scales=None):
    return tree_masks(where, vals, nulls, float_cols, scales)[0]


def expected_rows(vals, nulls, where, atts, float_cols=(), scales=None):
    """the projected rows of SELECT atts FROM t WHERE where, in row order: ([int64 values], [uint8 nulls]) per output
    column"""
    keep = where_mask(where, vals, nulls, float_cols, scales)
    out_v, out_n = [], []
    for a in atts:
        v = np.asarray(vals[a])
        v = v.astype(np.float64).view(np.int64) if a in float_cols else v.astype(np.int64)
        isnull = _null(nulls, a, len(v))
        out_v.append(np.where(isnull, 0, v)[keep])
        out_n.append(isnull[keep].astype(np.uint8))
    return out_v, out_n
