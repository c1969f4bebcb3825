"""Exact reference of the equi-join that cg_join_aggregate aggregates over, in numpy.

    join(build_cols, build_nulls, build_key, probe_cols, probe_nulls, probe_key)  ->  (cols, nulls) of the joined rows
    nested_loop_join(...)                                                          ->  the same, one pair of rows at a time

A joined row is the build row's columns followed by the probe row's columns, so its attribute a < len(build_cols) is
build column a and attribute len(build_cols) + j is probe column j: the numbering the library's descriptor uses.  Keys
are equal when their int64 values are equal; a NULL key joins nothing, on either side.  INT64_MIN is a key like any
other.  The rows come out probe row by probe row, each probe row's matches in build-row order; a join has no order, so
callers compare multisets (or aggregates).

The joined columns feed the exact aggregate reference unchanged (reference.aggregate).
"""
from __future__ import annotations

import numpy as np


def _valid(nulls, key, n):
    k = None if nulls is None else nulls[key]
    return np.ones(n, bool) if k is None else ~np.asarray(k, bool)


def join_indexes(build_keys, build_valid, probe_keys, probe_valid):
    """(build row, probe row) index arrays of every joined pair: sort the build keys, searchsorted the probe keys"""
    bk, pk = np.asarray(build_keys, np.int64), np.asarray(probe_keys, np.int64)
    brows = np.flatnonzero(build_valid)
    order = brows[np.argsort(bk[brows], kind="stable")]
    sorted_keys = bk[order]
    prows = np.flatnonzero(probe_valid)
    lo = np.searchsorted(sorted_keys, pk[prows], "left")
    hi = np.searchsorted(sorted_keys, pk[prows], "right")
    m = hi - lo
    pi = np.repeat(prows, m)
    start = np.repeat(lo, m)
    within = np.arange(len(pi)) - np.repeat(np.cumsum(m) - m, m)
    bi = order[start + within] if len(pi) else np.zeros(0, np.int64)
    return bi.astype(np.int64), pi.astype(np.int64)


def _gather(cols, nulls, idx):
    out_c = [np.asarray(c)[idx] for c in cols]
    nulls = list(nulls or []) + [None] * (len(cols) - len(nulls or []))
    out_n = [None if x is None else np.asarray(x, np.uint8)[idx] for x in nulls]
    return out_c, out_n


def join(build_cols, build_nulls, build_key, probe_cols, probe_nulls, probe_key):
    """(cols, nulls) of the joined rows: build columns, then probe columns; nulls[i] None where that side had none"""
    nb, npr = len(build_cols[build_key]), len(probe_cols[probe_key])
    bi, pi = join_indexes(build_cols[build_key], _valid(build_nulls, build_key, nb),
                          probe_cols[probe_key], _valid(probe_nulls, probe_key, npr))
    bc, bn = _gather(build_cols, build_nulls, bi)
    pc, pn = _gather(probe_cols, probe_nulls, pi)
    return bc + pc, bn + pn


def nested_loop_join(build_cols, build_nulls, build_key, probe_cols, probe_nulls, probe_key):
    """the same join as plain Python loops over every pair of rows (for checking join())"""
    nb, npr = len(build_cols[build_key]), len(probe_cols[probe_key])
    bv, pv = _valid(build_nulls, build_key, nb), _valid(probe_nulls, probe_key, npr)
    bi, pi = [], []
    for p in range(npr):
        for b in range(nb):
            if bv[b] and pv[p] and int(build_cols[build_key][b]) == int(probe_cols[probe_key][p]):
                bi.append(b)
                pi.append(p)
    bc, bn = _gather(build_cols, build_nulls, np.array(bi, np.int64))
    pc, pn = _gather(probe_cols, probe_nulls, np.array(pi, np.int64))
    return bc + pc, bn + pn


def rows_of(cols, nulls):
    """the joined rows as a sorted list of tuples (None for NULL), for comparing two joins as multisets"""
    n = len(cols[0]) if cols else 0
    nulls = list(nulls) + [None] * (len(cols) - len(nulls))
    out = []
    for r in range(n):
        out.append(tuple(None if (x is not None and x[r]) else int(c[r]) for c, x in zip(cols, nulls)))
    return sorted(out, key=lambda t: tuple((v is None, v or 0) for v in t))


def exact_sum(a) -> int:
    """exact sum of an int64 array as a Python integer (two 32-bit halves, each summed in int64)"""
    a = np.asarray(a, np.int64)
    return int((a >> 32).sum()) * 2**32 + int((a & 0xffffffff).sum())
