"""cg_join_aggregate against the exact references: the numpy equi-join of tests/join_agg_reference.py, aggregated by
tests/reference.py (WHERE trees, IN lists, IS NULL, column atoms, FILTER, bit_* / bool_*, variance).  Covered: the plain aggregate against cg_join_count_sum on a C4-shaped input with a
3000 x 3000 key, INT64_MIN and NULL keys; every group key form on dense and hash tables; every aggregate kind; WHERE
trees with a cross-side column atom; accumulation over two calls and an export / merge round trip; the one-GPU
repartition exchange followed by one call per partition; the refusals."""
import ctypes as C
import types

import numpy as np
import pytest

import join_agg_reference as jref
import partition_reference as pr
import reference as ref
from test_gpu_bool_bit_agg import assert_exact
from gpu_harness import cg  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

INT64_MIN = -2**63
INT, FLOAT = 0, 1


def NUMERIC(s):
    return 2 | (s << 8)


# attributes of the joined row: build b(k, x, g, d, f) then probe p(k, y, h, d, f)
COLS = [(8, INT), (8, INT), (4, INT), (-1, NUMERIC(2)), (8, FLOAT),
        (8, INT), (8, INT), (4, INT), (-1, NUMERIC(3)), (8, FLOAT)]
FLOATS = (4, 9)
SCALES = {3: 2, 8: 3}


def _dev(a, dtype=np.int64):
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype == np.float64:
        a = a.view(np.int64)
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


class Side:
    """host columns (float columns as float64), their null arrays (None = no NULLs) and device copies"""

    def __init__(self, cols, nulls, key=0):
        import torch
        self.cols, self.nulls, self.key = cols, nulls, key
        self.d = [_dev(c) for c in cols]
        self.dn = [None if x is None else _dev(x, np.uint8) for x in nulls]
        torch.cuda.synchronize()          # the library's stream does not wait for torch's

    @property
    def n(self):
        return len(self.cols[0])

    def ptrs(self):
        return [t.data_ptr() for t in self.d]

    def null_ptrs(self):
        return [None if t is None else t.data_ptr() for t in self.dn]


def make_side(rng, n, nkeys, probe, null_rate=0.05, key_nulls=0.02, key_min=True):
    keys = rng.integers(0, nkeys, n)
    if key_min and n >= 40:
        keys[rng.choice(n, 7, replace=False)] = INT64_MIN          # the join table's EMPTY sentinel joins like any key
    x = rng.integers(-10**6, 10**6, n)
    g = rng.integers(0, 30 if probe else 50, n)
    d = rng.integers(-10**7, 10**7, n)
    f = np.round(rng.normal(0, 100, n), 3)
    cols = [keys, x, g, d, f]
    nulls = [(rng.random(n) < key_nulls).astype(np.uint8)] + [(rng.random(n) < null_rate).astype(np.uint8) for _ in range(3)] + [None]
    return Side(cols, nulls)


def joined(b, p):
    return jref.join(b.cols, b.nulls, b.key, p.cols, p.nulls, p.key)


def keyed(groups, group, composite):
    out = {}
    for k, per in groups.items():
        if composite or not group:
            out[k if group else ()] = per
        elif len(group) == 1:
            out[(k,)] = per
        else:
            out[ref.unpack_two_column_key(k)] = per
    return out


def run(cg, b, p, where, group, aggs, kmin=0, kmax=-1, composite=False, key_bounds=None, expected_groups=0, agg=None,
        want_stats=True):
    d = cg.make_desc(where, group, aggs, float_cols=FLOATS, composite=composite, key_bounds=key_bounds,
                     expected_groups=expected_groups)
    own = agg is None
    if own:
        agg = cg.GpuColumnarAgg(d, COLS, kmin, kmax, 0)
    st = agg.join_aggregate(b.ptrs(), b.key, b.n, p.ptrs(), p.key, p.n, b.null_ptrs(), p.null_ptrs(), want_stats=want_stats)
    return agg, st


def check(cg, b, p, where, group, aggs, **kw):
    jc, jn = joined(b, p)
    want = ref.aggregate(jc, jn, where, group, aggs, FLOATS, SCALES)
    agg, st = run(cg, b, p, where, group, aggs, **kw)
    try:
        got = keyed(agg.groups(), group, kw.get("composite", False))
    finally:
        agg.free()
    n = len(jc[0])
    assert st.rows_scanned == n
    assert st.rows_removed_by_filter == want.rows_removed
    assert st.chunk_groups_scanned == 0 and st.chunk_groups_filtered == 0 and st.h2d_bytes == 0
    assert_exact(st, got, want, aggs, n)
    return st, got, want


@pytest.fixture(scope="module")
def sides():
    rng = np.random.default_rng(20261019)
    return make_side(rng, 6000, 2000, False), make_side(rng, 6000, 2000, True)


# --------------------------------------------------------------------------- 1. against cg_join_count_sum
def test_plain_aggregate_equals_join_count_sum(cg):
    """C4 shape: 1 M rows per side, keys U[0, 2^20), one key with 3000 x 3000 matches, INT64_MIN and NULL keys"""
    rng = np.random.default_rng(4)
    n = 1 << 20
    bk, pk = rng.integers(0, 1 << 20, n), rng.integers(0, 1 << 20, n)
    bk[:3000] = pk[:3000] = 123456789
    bk[3000:3010] = INT64_MIN
    pk[3000:3004] = INT64_MIN
    bx, py = rng.integers(-2**40, 2**40, n), rng.integers(-2**40, 2**40, n)
    bx[:1000] = 2**63 - 1
    py[:1000] = INT64_MIN
    bnull = (rng.random(n) < 0.01).astype(np.uint8)
    pnull = (rng.random(n) < 0.01).astype(np.uint8)
    bnull[:3000] = pnull[:3000] = 0
    pb, pq = rng.permutation(n), rng.permutation(n)
    b = Side([bk[pb], bx[pb]], [bnull[pb], None])
    p = Side([pk[pq], py[pq]], [pnull[pq], None])
    bi, pi = jref.join_indexes(b.cols[0], b.nulls[0] == 0, p.cols[0], p.nulls[0] == 0)
    rows, sx, sy = len(bi), jref.exact_sum(b.cols[1][bi]), jref.exact_sum(p.cols[1][pi])
    assert rows > 9_000_000
    j_rows, j_sum = cg.join_count_sum(b.d[0].data_ptr(), b.d[1].data_ptr(), n, p.d[0].data_ptr(), p.d[1].data_ptr(), n,
                                      b.dn[0].data_ptr(), p.dn[0].data_ptr())
    assert (j_rows, j_sum) == (rows, sx + sy)
    aggs = [cg.count_star(), cg.sum_(1), cg.sum_(3)]
    d = cg.make_desc([], [], aggs)
    agg = cg.GpuColumnarAgg(d, [(8, INT), (8, INT), (8, INT), (8, INT)], 0, -1, 0)
    try:
        st = agg.join_aggregate(b.ptrs(), 0, n, p.ptrs(), 0, n, b.null_ptrs(), p.null_ptrs())
        (per,) = agg.groups().values()
    finally:
        agg.free()
    assert (per[0]["count"], per[1]["sum"], per[2]["sum"]) == (rows, sx, sy)
    assert per[1]["sum"] + per[2]["sum"] == j_sum and per[1]["count"] == per[2]["count"] == rows
    assert st.rows_scanned == st.rows_passed == rows and st.rows_removed_by_filter == 0
    assert st.bytes_scanned == 2 * (16 * n + n) and st.kernel_ms > 0


# --------------------------------------------------------------------------- 2. group key forms
def _bounds(jc, jn, cols):
    out = []
    for c in cols:
        v = jc[c][jn[c] == 0] if jn[c] is not None else jc[c]
        out.append((int(v.min()), int(v.max())))
    return out


@pytest.mark.parametrize("table", ["dense", "hash"])
@pytest.mark.parametrize("form", ["build", "probe", "key", "packed", "composite"])
def test_group_key_forms(cg, sides, form, table):
    b, p = sides
    aggs = [cg.count_star(), cg.sum_(1), cg.sum_(6), cg.min_(4, is_float=True), cg.max_(8), cg.count(3)]
    dense = table == "dense"
    kw, where = {}, []
    if form == "build":
        group = [2]
        kw = dict(kmin=0, kmax=49) if dense else {}
    elif form == "probe":
        group = [7]
        kw = dict(kmin=0, kmax=29) if dense else {}
    elif form == "key":
        group = [0]
        if dense:
            kw, where = dict(kmin=0, kmax=1999), [(0, ">=", 0)]
    elif form == "packed":
        group, where = [2, 7], [(2, "is not null"), (7, "is not null")]
        kw = dict(kmin=0, kmax=49 | (29 << 32)) if dense else {}
    else:
        group = [2, 7]
        jc, jn = joined(b, p)
        bounds = _bounds(jc, jn, group) if dense else [(-2**13, 2**13)] * 2
        kw = dict(composite=True, key_bounds=bounds)
    d = cg.make_desc(where, group, aggs, float_cols=FLOATS, composite=kw.get("composite", False), key_bounds=kw.get("key_bounds"))
    probe_partial = cg.GpuColumnarAgg(d, COLS, kw.get("kmin", 0), kw.get("kmax", -1), 0)
    assert probe_partial.layout()[2] == dense
    probe_partial.free()
    check(cg, b, p, where, group, aggs, **kw)


# --------------------------------------------------------------------------- 3. every aggregate kind
@pytest.mark.parametrize("group", [[], [2]])
def test_every_aggregate_kind(cg, sides, group):
    b, p = sides
    Col = cg.Col
    kw = dict(kmin=0, kmax=49) if group else {}
    cross = cg.Agg(2, [(1, 0, 1), (6, 1, 1)])                       # sum(b.x * (1 + p.y))
    first = [cg.count(1), cross, cg.min_(1), cg.max_(6), cg.min_(4, is_float=True), cg.max_(9, is_float=True),
             cg.bit_and(1), cg.bit_or(6)]
    check(cg, b, p, [], group, first, **kw)
    second = [cg.bool_and((3, "<", Col(8))), cg.bool_or(("or", (4, ">", 0.5), (7, "is null"))),
              cg.sum_(9, is_float=True, filter=("or", (2, "<", 10), (6, ">", 0))),
              cg.count_star(filter=("and", (1, ">", 0), (8, "is not null"))),
              cg.sum_(1, filter=(6, "in", (1, 2, 3, None)))]
    check(cg, b, p, [], group, second, **kw)


@pytest.mark.parametrize("group", [[], [2]])
def test_var_samp_over_numeric(cg, sides, group):
    b, p = sides
    aggs = [cg.count_star(), cg.variance(3), cg.variance(1, filter=(6, ">", 0))]
    jc, jn = joined(b, p)
    want = ref.aggregate(jc, jn, [], group, aggs, FLOATS)
    agg, st = run(cg, b, p, [], group, aggs, **(dict(kmin=0, kmax=49) if group else {}))
    try:
        got = keyed(agg.groups(), group, False)
    finally:
        agg.free()
    assert set(got) == set(want.groups)
    for key, per in want.groups.items():
        for a in (1, 2):
            g, w = got[key][a], per[a]
            assert (g["count"], g["sum"], g["sumsq"]) == (w.count, w.sum, w.sumsq), (key, a)
            if w.count > 1:
                assert cg.numeric_var_out(1, g["count"], g["sum"], g["sumsq"], 2 if a == 1 else 0) == \
                    ref.var_out(1, w.count, w.sum, w.sumsq, 2 if a == 1 else 0)


# --------------------------------------------------------------------------- 4. WHERE trees
@pytest.mark.parametrize("group", [[], [2], [7]])
@pytest.mark.parametrize("tree", range(4))
def test_where_trees(cg, sides, tree, group):
    b, p = sides
    Col = cg.Col
    where = [
        [(1, ">", -500000), (6, "<", 500000)],
        ("and", ("or", (2, "in", (1, 2, 3, None)), (7, "is null")), (3, "<", Col(8))),
        ("or", ("and", (3, "<", Col(8)), (6, "not in", (5, 7, 11))), (1, "is null"), (9, "<", -50.0)),
        ("and", (3, ">=", Col(8)), (8, "is not null"), ("or", (4, ">", 0.0), (7, "in", (0, 29)))),
    ][tree]
    aggs = [cg.count_star(), cg.sum_(1), cg.sum_(6), cg.max_(3)]
    kw = dict(kmin=0, kmax=49) if group == [2] else {}
    st, _, want = check(cg, b, p, where, group, aggs, **kw)
    assert 0 < st.rows_removed_by_filter < st.rows_scanned
    assert st.rows_passed == want.rows_passed


# --------------------------------------------------------------------------- 5. accumulation
def test_two_calls_and_export_merge(cg):
    import torch
    rng = np.random.default_rng(55)
    b1, p1 = make_side(rng, 4000, 1500, False), make_side(rng, 5000, 1500, True)
    b2, p2 = make_side(rng, 3000, 900, False), make_side(rng, 2000, 900, True)
    group = [2]
    aggs = [cg.count_star(), cg.sum_(1), cg.min_(6), cg.sum_(9, is_float=True)]
    j1, j2 = joined(b1, p1), joined(b2, p2)
    jc = [np.concatenate([a, c]) for a, c in zip(j1[0], j2[0])]
    jn = [None if a is None else np.concatenate([a, c]) for a, c in zip(j1[1], j2[1])]
    want = ref.aggregate(jc, jn, [], group, aggs, FLOATS, SCALES)
    agg, st1 = run(cg, b1, p1, [], group, aggs, expected_groups=64)
    other = None
    try:
        _, st2 = run(cg, b2, p2, [], group, aggs, agg=agg)
        st = types.SimpleNamespace(rows_passed=st1.rows_passed + st2.rows_passed,
                                   rows_removed_by_filter=st1.rows_removed_by_filter + st2.rows_removed_by_filter,
                                   rows_scanned=st1.rows_scanned + st2.rows_scanned)
        got = keyed(agg.groups(), group, False)
        assert_exact(st, got, want, aggs, len(jc[0]))
        nwords = agg.layout()[0]
        cap = agg.ngroups()
        keys = torch.empty(cap, dtype=torch.int64, device="cuda")
        nulls = torch.empty(cap, dtype=torch.uint8, device="cuda")
        words = torch.empty(cap * nwords, dtype=torch.int64, device="cuda")
        n = agg.export_device(keys.data_ptr(), nulls.data_ptr(), words.data_ptr(), cap)
        assert n == cap
        other = cg.GpuColumnarAgg(agg.desc, COLS, 0, 49, 0)
        other.merge_rows(keys.data_ptr(), nulls.data_ptr(), words.data_ptr(), n)
        assert keyed(other.groups(), group, False) == got
    finally:
        agg.free()
        if other is not None:
            other.free()


# --------------------------------------------------------------------------- 6. exchange -> one call per partition
@pytest.fixture(scope="module")
def comm(cg):
    from citus_b200 import distributed
    distributed.init(0, 1)
    yield distributed
    distributed.destroy()


def _exchange(cg, slot, cols, P):
    """received columns (device pointers), rows of every local partition"""
    import torch
    from citus_b200 import capi
    L = capi.lib()
    mins, maxs = (np.ascontiguousarray(x, np.int32) for x in pr.synthetic_intervals(P))
    dc = [_dev(c) for c in cols]
    cp = (C.c_void_p * len(cols))(*[c.data_ptr() for c in dc])
    got = C.c_int64(-1)
    torch.cuda.synchronize()
    capi.check(L.cg_comm_repartition_exchange(slot, cp, None, len(cols[0]), len(cols), 8, P, mins.ctypes.data, maxs.ctypes.data,
                                              C.byref(got)))
    capi.check(L.cg_comm_exchange_wait(slot))
    capi.check(L.cg_synchronize())
    ptrs = (C.c_void_p * 8)()
    nrows, nlocal = C.c_int64(), C.c_int32()
    counts = np.zeros(P, np.int64)
    capi.check(L.cg_comm_exchange_result(slot, ptrs, C.byref(nrows), counts.ctypes.data, C.byref(nlocal), None, None))
    assert nrows.value == len(cols[0]) and nlocal.value == P
    return [ptrs[c] for c in range(len(cols))], counts


def test_exchange_then_join_aggregate(cg, comm):
    rng = np.random.default_rng(606)
    P = 8
    nb, npr = 100_000, 80_000
    bk, pk = rng.integers(0, 50_000, nb), rng.integers(0, 50_000, npr)
    bk[:300] = pk[:300] = 77
    bk[300:310] = INT64_MIN
    pk[300:303] = INT64_MIN
    bx, bg = rng.integers(-10**9, 10**9, nb), rng.integers(0, 100, nb)
    py, ph = rng.integers(-10**9, 10**9, npr), rng.integers(0, 1000, npr)
    bptr, bcnt = _exchange(cg, 0, [bk, bx, bg], P)
    pptr, pcnt = _exchange(cg, 1, [pk, py, ph], P)
    cols = [(8, INT), (8, INT), (4, INT), (8, INT), (8, INT), (4, INT)]
    where = [(1, "<", cg.Col(4))]
    aggs = [cg.count_star(), cg.sum_(1), cg.sum_(4), cg.max_(5)]
    d = cg.make_desc(where, [2], aggs)
    agg = cg.GpuColumnarAgg(d, cols, 0, 99, 0)
    try:
        ob, op = np.concatenate([[0], np.cumsum(bcnt)]), np.concatenate([[0], np.cumsum(pcnt)])
        scanned = 0
        for q in range(P):
            st = agg.join_aggregate([x + 8 * int(ob[q]) for x in bptr], 0, int(bcnt[q]), [x + 8 * int(op[q]) for x in pptr], 0,
                                    int(pcnt[q]), want_stats=q % 2 == 0)
            scanned += st.rows_scanned
        got = keyed(agg.groups(), [2], False)
    finally:
        agg.free()
    jc, jn = jref.join([bk, bx, bg], None, 0, [pk, py, ph], None, 0)
    want = ref.aggregate(jc, jn, where, [2], aggs)
    assert set(got) == set(want.groups)
    for key, per in want.groups.items():
        for a, w in enumerate(per):
            g = got[key][a]
            assert g["count"] == w.count, (key, a)
            if a in (1, 2):
                assert g["sum"] == w.sum, (key, a)
            if a == 3:
                assert g["minmax"] == w.max, key


# --------------------------------------------------------------------------- 7. refusals
def test_refusals_leave_the_partial_untouched(cg, sides):
    from citus_b200 import capi
    b, p = sides
    group, aggs = [2], [cg.count_star(), cg.sum_(1), cg.sum_(6)]
    d = cg.make_desc([], group, aggs, float_cols=FLOATS)
    agg = cg.GpuColumnarAgg(d, COLS, 0, 49, 0)

    def refused(code, **kw):
        with pytest.raises(capi.CitusGpuError) as e:
            agg.join_aggregate(kw.get("bp", b.ptrs()), kw.get("bkey", 0), b.n, p.ptrs(), 0, p.n, b.null_ptrs(), p.null_ptrs(),
                               columns=kw.get("columns"))
        assert e.value.code == code, e.value

    try:
        float_key = list(COLS)
        float_key[0] = (8, FLOAT)
        refused(capi.CG_EUNSUPPORTED, columns=float_key)
        scales = list(COLS)
        scales[0] = (-1, NUMERIC(2))
        refused(capi.CG_EUNSUPPORTED, columns=scales)
        null_col = b.ptrs()
        null_col[1] = None
        refused(capi.CG_EINVAL, bp=null_col)
        refused(capi.CG_EINVAL, bkey=5)
        other = agg.desc
        agg.desc = cg.make_desc([], group, [cg.count_star(), cg.sum_(1)], float_cols=FLOATS)
        try:
            refused(capi.CG_EINVAL)
        finally:
            agg.desc = other
        # nothing of the above reached the partial: one valid call gives the reference
        jc, jn = joined(b, p)
        want = ref.aggregate(jc, jn, [], group, aggs, FLOATS, SCALES)
        st = agg.join_aggregate(b.ptrs(), 0, b.n, p.ptrs(), 0, p.n, b.null_ptrs(), p.null_ptrs())
        assert_exact(st, keyed(agg.groups(), group, False), want, aggs, len(jc[0]))
        # an empty side is a no-op
        st = agg.join_aggregate(b.ptrs(), 0, 0, p.ptrs(), 0, p.n, b.null_ptrs(), p.null_ptrs())
        assert st.rows_scanned == 0
        assert keyed(agg.groups(), group, False).keys() == want.groups.keys()
    finally:
        agg.free()


def test_term_abs_bound_is_refused(cg, sides):
    from citus_b200 import capi
    b, p = sides
    a = cg.sum_(1)
    a.term_abs_bound = 10**6
    d = cg.make_desc([], [], [cg.count_star(), a])
    agg = cg.GpuColumnarAgg(d, COLS, 0, -1, 0)
    try:
        with pytest.raises(capi.CitusGpuError) as e:
            agg.join_aggregate(b.ptrs(), 0, b.n, p.ptrs(), 0, p.n, b.null_ptrs(), p.null_ptrs())
        assert e.value.code == capi.CG_EINVAL
    finally:
        agg.free()


def test_errors_raised_by_the_kernel_surface_at_read(cg):
    from citus_b200 import capi
    rng = np.random.default_rng(9)
    n = 5000
    b = Side([rng.integers(0, 5000, n), np.full(n, 2**40)], [None, None])
    p = Side([rng.integers(0, 5000, n), np.full(n, 2**40)], [None, None])
    cols = [(8, INT)] * 4
    # b.x * p.y = 2^80 leaves int64
    d = cg.make_desc([], [], [cg.Agg(2, [(1, 0, 1), (3, 0, 1)])])
    agg = cg.GpuColumnarAgg(d, cols, 0, -1, 0)
    try:
        agg.join_aggregate(b.ptrs(), 0, n, p.ptrs(), 0, n, want_stats=False)
        with pytest.raises(capi.CitusGpuError) as e:
            agg.groups()
        assert e.value.code == capi.CG_EUNSUPPORTED
    finally:
        agg.free()
    # a hash table sized for one group: thousands of join keys fill it
    d = cg.make_desc([], [0], [cg.count_star()], expected_groups=1)
    agg = cg.GpuColumnarAgg(d, cols, 0, -1, 0)
    try:
        agg.join_aggregate(b.ptrs(), 0, n, p.ptrs(), 0, n, want_stats=False)
        with pytest.raises(capi.CitusGpuError) as e:
            agg.groups()
        assert e.value.code == capi.CG_ETABLEFULL
    finally:
        agg.free()
