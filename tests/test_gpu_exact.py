"""The fused scan's arithmetic against the exact reference (tests/reference.py) at the edges of the number types:
integer aggregate arguments near and beyond int64, NaN / inf / -0.0 / subnormal floats, cancellation in float sums,
negative group keys, and the combine paths.  Each case runs on every kernel family.  The expected answer is the exact
value; for an integer argument that leaves int64 it is CG_EUNSUPPORTED (the caller then runs the row-at-a-time
executor, which raises PostgreSQL's error or computes numeric exactly) -- never a different number."""
import ctypes as C
import dataclasses
import math
import struct

import numpy as np
import pytest

import reference as ref
from gpu_harness import cg, kernel_family, FAMILIES  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

NEG_NAN = struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000000))[0]
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


def gpu_run(cg, rel, where, group_cols, aggs, float_cols=(), use_bounds=True, force_hash=False, e2e=False,
            expected_groups=0, bounds=None):
    """one partial aggregate over `rel`; returns (stats, groups keyed like the reference, layout)"""
    aggs = [dataclasses.replace(a) for a in aggs]
    d = cg.make_desc(where, group_cols, aggs, float_cols=float_cols, expected_groups=expected_groups)
    kmin, kmax, proven, rows = cg.relation_bounds(rel, d)
    for i, a in enumerate(aggs):
        a.term_abs_bound = (bounds[i] if bounds else proven[i]) if use_bounds else 0
    d = cg.make_desc(where, group_cols, aggs, float_cols=float_cols, expected_groups=expected_groups)
    if force_hash:
        kmin, kmax = 0, -1
    agg = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, max(rows, 1))
    try:
        if e2e == "dma":
            rel.register()
            try:
                st = agg.scan_relation(rel)
            finally:
                rel.unregister()
        else:
            shard = cg.Shard(rel)
            st = agg.scan_shard(shard)
            shard.free()
        got = agg.groups()
        layout = agg.layout()
    finally:
        agg.free()
    keyed = {}
    for k, per in got.items():
        if not group_cols:
            key = ()
        elif len(group_cols) == 1:
            key = (k,)
        else:
            key = ref.unpack_two_column_key(k)
        keyed[key] = per
    return st, keyed, layout


def assert_matches_reference(st, got, want, aggs, nrows):
    assert st.rows_passed == want.rows_passed
    assert st.rows_removed_by_filter + (nrows - st.rows_scanned) == want.rows_removed
    if () in got and () not in want.groups:                     # a plain aggregate over no rows: one row of NULLs
        assert all(g["count"] == 0 for g in got[()])
        return
    assert set(got) == set(want.groups)
    for key, per in want.groups.items():
        for a, (spec, st_ref) in enumerate(zip(aggs, per)):
            g = got[key][a]
            assert g["count"] == st_ref.count, (key, a)
            if spec.kind in (0, 1) or st_ref.count == 0:
                continue
            if spec.kind == 2:
                if spec.is_float:
                    assert st_ref.float_sum_ok(g["fsum"]), (key, a, g["fsum"], st_ref.float_sum())
                else:
                    assert g["sum"] == st_ref.sum, (key, a)
            else:
                wantv = st_ref.min if spec.kind == 3 else st_ref.max
                if spec.is_float:
                    gotv = float(np.int64(g["minmax"]).view(np.float64))
                    assert ref.float8_eq(gotv, wantv), (key, a, gotv, wantv)
                else:
                    assert g["minmax"] == wantv, (key, a)


def check_exact_or_refused(cg, rel, cols, nulls, where, group_cols, aggs, nrows, want=None, **kw):
    """the exact answer, or CG_EUNSUPPORTED exactly when an integer argument leaves int64"""
    from citus_b200 import capi
    want = want or ref.aggregate(cols, nulls, where, group_cols, aggs, kw.get("float_cols", ()))
    if ref.overflows(want):
        with pytest.raises(capi.CitusGpuError) as e:
            gpu_run(cg, rel, where, group_cols, aggs, **kw)
        assert e.value.code == capi.CG_EUNSUPPORTED, str(e.value)
        return None
    st, got, layout = gpu_run(cg, rel, where, group_cols, aggs, **kw)
    assert_matches_reference(st, got, want, aggs, nrows)
    return layout


SHAPES = [dict(group_cols=[]), dict(group_cols=[0]), dict(group_cols=[1], expected_groups=5000),
          dict(group_cols=[1], expected_groups=5000, force_hash=True)]


# --------------------------------------------------------------------------- integer terms
@pytest.mark.parametrize("family", FAMILIES)
def test_integer_terms_exact_or_refused(cg, kernel_family, family):
    """sum / min / max(x*y) and sum((a + b*x)*(c + d*y)*z) with values near 2^31, 2^40 and 2^62, INT64_MIN / MAX in a
    bare column; each with the bounds cg_relation_bounds proves and with no bound; plain aggregate, shared-memory
    cells, a direct-indexed table and the hash table"""
    kernel_family(family)
    rng = np.random.default_rng(5)
    n = 20_000
    A = [cg.Agg(2, [(2, 0, 1), (3, 0, 1)]), cg.Agg(3, [(2, 0, 1), (3, 0, 1)]), cg.Agg(4, [(2, 0, 1), (3, 0, 1)]),
         cg.count_star(), cg.sum_(5), cg.min_(5), cg.max_(5)]
    B = [cg.Agg(2, [(2, 7, 1), (3, -5, 2), (4, 0, 1)]), cg.count_star()]
    refused = exact = 0
    for scale in (2**31, 2**40, 2**62):
        k = rng.integers(0, 4, n)
        k2 = rng.integers(0, 5000, n)
        x = rng.integers(-scale, scale, n)
        y = rng.integers(-scale, scale, n)
        z = rng.integers(-3, 4, n)
        m = rng.integers(INT64_MIN, INT64_MAX, n, endpoint=True)
        x[:2], y[:2] = [scale - 1, -scale], [-scale, -scale]
        m[:4] = [INT64_MAX, INT64_MIN, INT64_MAX, -1]
        cols = [k, k2, x, y, z, m]
        rel = cg.Relation.write([8] * 6, cols, stripe_row_limit=10_000, chunk_row_limit=5000)
        for aggs in (A, B):
            for shape in SHAPES:
                want = ref.aggregate(cols, None, [], shape["group_cols"], aggs)
                for use_bounds in (True, False):
                    r = check_exact_or_refused(cg, rel, cols, None, [], aggs=aggs, nrows=n, want=want, use_bounds=use_bounds, **shape)
                    refused += r is None
                    exact += r is not None
        # rows that would overflow, filtered out by WHERE: the check stays armed but never fires
        where = [(2, ">", -2**31), (2, "<", 2**31), (3, ">", -2**31), (3, "<", 2**31)]
        check_exact_or_refused(cg, rel, cols, None, where, [0], A, n)
    assert refused and exact


@pytest.mark.parametrize("family", FAMILIES)
def test_q1_shape_over_decimal_prices_near_the_type_limit(cg, oracle, kernel_family, family):
    """sum(l_extendedprice*(1-l_discount)*(1+l_tax)) over decimal(15,2) varlena columns: with prices near 9.99e12 the
    scaled term (price*100 * (100-d) * (100+t)) leaves int64 and the scan is refused; below ~8.5e12 it is exact"""
    kernel_family(family)
    NUM2 = 2 | (2 << 8)
    rng = np.random.default_rng(17)
    n = 6000
    aggs = [cg.sum_(0), cg.sum_(1), cg.Agg(2, [(1, 0, 1), (2, 100, -1)]), cg.Agg(2, [(1, 0, 1), (2, 100, -1), (3, 100, 1)]),
            cg.count_star()]
    for lo, hi in ((9 * 10**14, 10**15), (10**5, 8 * 10**14)):           # scaled by 10^2: decimal(15,2) ends at 10^15 - 1
        q = rng.integers(1, 51, n) * 100
        p = rng.integers(lo, hi, n)
        p[0] = hi - 1
        d = rng.integers(0, 11, n)
        t = rng.integers(0, 9, n)
        t[0], d[0] = 8, 0
        rf = rng.choice([65, 78, 82], n)
        ls = rng.choice([70, 79], n)
        cols = [q, p, d, t, rf, ls]
        tab = oracle.Table([-1, -1, -1, -1, -1, -1], [NUM2, NUM2, NUM2, NUM2, 3, 3], stripe_row_limit=3000, chunk_row_limit=1000)
        tab.insert(cols)
        rel = cg.Relation.from_image(tab.pages(), tab.stripes_array(), tab.nodes_array(), [-1] * 6, [NUM2] * 4 + [3, 3])
        want = ref.aggregate(cols, None, [], [4, 5], aggs)
        assert ref.overflows(want) == (lo > 10**14)
        for e2e in (False, "dma"):
            check_exact_or_refused(cg, rel, cols, None, [], [4, 5], aggs, n, want=want, expected_groups=16, e2e=e2e)
        # without the tax factor the same prices fit
        check_exact_or_refused(cg, rel, cols, None, [], [4, 5], aggs[:3] + aggs[4:], n, expected_groups=16)


@pytest.mark.parametrize("family", FAMILIES)
def test_bound_violated_by_the_data_is_an_error(cg, kernel_family, family):
    """a term_abs_bound the data does not respect fails the scan with CG_EINVAL (CG_ERRFLAG_SUM_BOUND)"""
    from citus_b200 import capi
    kernel_family(family)
    rng = np.random.default_rng(2)
    n = 30_000
    cols = [rng.integers(0, 100, n), rng.integers(-1000, 1000, n)]
    rel = cg.Relation.write([8, 8], cols)
    for group in ([], [0]):
        with pytest.raises(capi.CitusGpuError) as e:
            gpu_run(cg, rel, [], group, [cg.sum_(1), cg.count_star()], bounds=[10, 0])
        assert e.value.code == capi.CG_EINVAL


# --------------------------------------------------------------------------- floats
def _specials(rng, n, frac=0.02):
    sp = np.array([math.nan, NEG_NAN, math.inf, -math.inf, -0.0, 0.0, 5e-324, -5e-324, 2.2250738585072014e-308 / 3, 1.5])
    f = rng.normal(size=n) * 1e3
    pick = rng.random(n) < frac
    f[pick] = sp[rng.integers(0, len(sp), int(pick.sum()))]
    return f


@pytest.mark.parametrize("family", FAMILIES)
def test_float_specials_min_max_sum_count(cg, kernel_family, family):
    """float8 and float4 columns holding +NaN, -NaN (0xFFF8...), +-inf, -0.0 and subnormals: min / max in PostgreSQL's
    float8 order (every NaN above +inf), sums that are NaN / inf exactly when the exact sum is"""
    kernel_family(family)
    rng = np.random.default_rng(23)
    n = 40_000
    k = rng.integers(-3, 4, n)
    k2 = rng.integers(0, 3000, n)
    f8 = _specials(rng, n, 0.0005)
    f4 = _specials(rng, n, 0.0005).astype(np.float32).astype(np.float64)
    f8[k == 2] = np.abs(f8[k == 2])
    f8[np.flatnonzero(k == 2)[::5000]] = NEG_NAN                          # group 2: -NaN is its max, never its min
    f4[k == -3] = -7.5
    f4[np.flatnonzero(k == -3)[-1]] = NEG_NAN
    nf8 = (rng.random(n) < 0.05).astype(np.uint8)
    cols = [k, k2, f8, f4]
    nulls = [None, None, nf8, None]
    rel = cg.Relation.write([8, 8, 8, 4], cols, nulls, type_classes=[0, 0, 1, 1], stripe_row_limit=20_000, chunk_row_limit=4000)
    aggs = [cg.min_(2, True), cg.max_(2, True), cg.min_(3, True), cg.max_(3, True), cg.sum_(2, True), cg.sum_(3, True),
            cg.count(2), cg.count_star()]
    fc = (2, 3)
    for shape in SHAPES:
        check_exact_or_refused(cg, rel, cols, nulls, [], aggs=aggs, nrows=n, float_cols=fc, **shape)
    check_exact_or_refused(cg, rel, cols, nulls, [(1, "<", 2000)], [0], aggs, n, float_cols=fc, e2e="dma")
    g = ref.aggregate(cols, nulls, [], [0], aggs, fc).groups
    assert ref.isnan(g[(2,)][1].max) and not ref.isnan(g[(2,)][0].min) and ref.isnan(g[(-3,)][3].max)


@pytest.mark.parametrize("family", FAMILIES)
def test_float_quals_against_nan_inf_and_zero(cg, oracle, kernel_family, family):
    """<, <=, =, >=, >, <> against NaN, +-inf, 0.0 and -0.0 constants and OR trees; chunk groups whose max is NaN
    (sorted data): rows and chunk-group counters as the oracle counts them, values as the reference computes them"""
    kernel_family(family)
    rng = np.random.default_rng(29)
    n = 30_000
    f = np.sort(_specials(rng, n, 0.01))                                 # NaNs sort last: the last chunks' max is NaN
    f[-7:] = NEG_NAN
    v = rng.integers(-100, 100, n)
    k = rng.integers(0, 5, n)
    cols = [f, v, k]
    rel = cg.Relation.write([8, 8, 8], cols, type_classes=[1, 0, 0], stripe_row_limit=10_000, chunk_row_limit=2000)
    t = oracle.Table.attach(rel.pages(), rel.stripes_bytes(), rel.nodes_bytes(), [8, 8, 8], [1, 0, 0], chunk_row_limit=2000)
    aggs = [cg.count_star(), cg.sum_(1), cg.min_(0, True), cg.max_(0, True)]
    oaggs = [oracle.Agg(a.kind, list(a.factors), a.is_float) for a in aggs]
    trees = [[(0, op, c)] for c in (math.nan, math.inf, -math.inf, 0.0, -0.0) for op in ("<", "<=", "=", ">=", ">", "<>")]
    trees += [("or", (0, ">", math.inf), ("and", (0, "<", 0.0), (1, ">", 50))),
              ("or", (0, "=", math.nan), (0, "<=", -math.inf)),
              ("and", (0, "<>", math.nan), ("or", (0, ">=", 0.0), (2, "=", 3)))]
    for where in trees:
        for group in ([], [2]):
            st, got, _ = gpu_run(cg, rel, where, group, aggs, float_cols=(0,))
            r = t.scan(where, group, oaggs)
            assert (st.rows_scanned, st.rows_removed_by_filter, st.chunk_groups_filtered) == \
                (r.rows_scanned, r.rows_removed_by_filter, r.chunk_groups_filtered), where
            assert_matches_reference(st, got, ref.aggregate(cols, None, where, group, aggs, (0,)), aggs, n)
    st, _, _ = gpu_run(cg, rel, [(0, ">", 1e300)], [], aggs, float_cols=(0,))
    assert st.chunk_groups_filtered > 0 and st.rows_passed == int((f > 1e300).sum() + np.isnan(f).sum())


def test_float_sum_accuracy_under_cancellation_and_hot_groups(cg, kernel_family):
    """cancellation-heavy data (large +- pairs and small values), one group of ~10^6 rows and product terms: every
    float sum within the order-independent error bound of the exact sum"""
    rng = np.random.default_rng(31)
    n = 1_100_000
    big = rng.choice([1e16, -1e16, 3e15, -3e15], n)
    small = rng.normal(size=n)
    x = np.where(rng.random(n) < 0.5, big, small)
    y = rng.normal(size=n) * 1e-3 + 1.0
    k = np.where(rng.random(n) < 0.92, 0, rng.integers(1, 40, n))         # group 0: ~10^6 rows
    k2 = rng.integers(0, 3000, n)
    cols = [k, k2, x, y]
    rel = cg.Relation.write([8, 8, 8, 8], cols, type_classes=[0, 0, 1, 1], stripe_row_limit=200_000, chunk_row_limit=50_000)
    aggs = [cg.sum_(2, True), cg.Agg(2, [(2, 0.0, 1.0), (3, 0.0, 1.0)], True), cg.Agg(2, [(3, 2.5, -1.0), (2, 0.0, 1.0)], True),
            cg.count_star()]
    wants = {tuple(s["group_cols"]): ref.aggregate(cols, None, [], s["group_cols"], aggs, (2, 3)) for s in SHAPES[:3]}
    for family in FAMILIES:
        kernel_family(family)
        for shape in SHAPES:
            check_exact_or_refused(cg, rel, cols, None, [], aggs=aggs, nrows=n, float_cols=(2, 3),
                                   want=wants[tuple(shape["group_cols"])], **shape)


# --------------------------------------------------------------------------- group keys
@pytest.mark.parametrize("family", FAMILIES)
def test_negative_narrow_group_keys(cg, kernel_family, family):
    """int1 / int2 / int4 group keys with negative values, one and two columns, compared as tuples; small per-column
    ranges get a direct-indexed table even when the packed 64-bit bounds are out of order"""
    kernel_family(family)
    rng = np.random.default_rng(37)
    n = 50_000
    k1 = rng.integers(-128, 128, n)
    k2 = rng.integers(-300, 300, n)
    k4 = rng.integers(-2**31, 2**31, n)
    k4[:1000] = rng.integers(-5, 6, 1000)
    c = np.full(n, 3)
    v = rng.integers(-10**12, 10**12, n)
    cols = [k1, k2, k4, c, v, rng.integers(-5, 6, n)]
    rel = cg.Relation.write([1, 2, 4, 2, 8, 1], cols)
    aggs = [cg.sum_(4), cg.count_star(), cg.min_(4), cg.max_(0)]
    for group, dense in (([0], True), ([1], True), ([2], False), ([0, 1], True), ([1, 0], True), ([5, 3], True),
                         ([3, 5], True), ([2, 0], False)):
        layout = check_exact_or_refused(cg, rel, cols, None, [], group, aggs, n, expected_groups=70_000)
        assert layout[2] == dense, group
        check_exact_or_refused(cg, rel, cols, None, [(4, ">", 0)], group, aggs, n, expected_groups=70_000, force_hash=True)


# --------------------------------------------------------------------------- combine and host column paths
def test_merge_values_export_merge_and_agg_column_at_the_edges(cg):
    """cg_partial_merge_values, export_device -> merge_rows and cg_agg_column with NaN / inf floats and integer sums
    beyond int64: the merged answer equals the reference over all rows"""
    import torch
    from citus_b200 import capi
    L = capi.lib()
    rng = np.random.default_rng(41)
    n = 40_000
    k = rng.integers(0, 6, n)
    m = rng.integers(INT64_MIN, INT64_MAX, n, endpoint=True)
    m[:3] = [INT64_MAX, INT64_MAX, INT64_MIN]
    f = _specials(rng, n, 0.001)
    f[k == 4] = 2.0
    f[np.flatnonzero(k == 4)[0]] = NEG_NAN
    cols = [k, m, f]
    aggs = [cg.sum_(1), cg.min_(1), cg.max_(1), cg.min_(2, True), cg.max_(2, True), cg.sum_(2, True), cg.count_star()]
    halves = [slice(0, n // 2), slice(n // 2, n)]
    rels = [cg.Relation.write([8, 8, 8], [c[h] for c in cols], type_classes=[0, 0, 1]) for h in halves]
    want = ref.aggregate(cols, None, [], [0], aggs, (2,))
    for force_hash in (False, True):
        d = cg.make_desc([], [0], aggs, float_cols=(2,), expected_groups=16)
        kmin, kmax = (0, 5) if not force_hash else (0, -1)
        final = cg.GpuColumnarAgg(d, rels[0].column_descs(), kmin, kmax, n)
        via_values = cg.GpuColumnarAgg(d, rels[0].column_descs(), kmin, kmax, n)
        for rel in rels:
            part = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, n)
            part.scan_shard(cg.Shard(rel))
            nw = part.layout()[0]
            g = part.ngroups()
            keys = torch.empty(g, dtype=torch.int64, device="cuda")
            kn = torch.empty(g, dtype=torch.uint8, device="cuda")
            words = torch.empty(g * nw, dtype=torch.int64, device="cuda")
            assert part.export_device(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), g) == g
            final.merge_rows(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), g)
            fr = part.fetch()
            capi.check(L.cg_partial_merge_values(via_values.h, fr["n"], fr["keys"].ctypes.data, fr["key_nulls"].ctypes.data,
                                                 np.ascontiguousarray(fr["sum_hi"]).ctypes.data, np.ascontiguousarray(fr["sum_lo"]).ctypes.data,
                                                 np.ascontiguousarray(fr["count"]).ctypes.data, np.ascontiguousarray(fr["minmax"]).ctypes.data,
                                                 np.ascontiguousarray(fr["fsum"]).ctypes.data))
            part.free()
        for combined in (final, via_values):
            got = {(kk,): per for kk, per in combined.groups().items()}
            st = type("S", (), dict(rows_passed=n, rows_removed_by_filter=0, rows_scanned=n))
            assert_matches_reference(st, got, want, aggs, n)
            combined.free()
    # one host column at a time
    for attlen, vals, is_float in ((8, m, 0), (8, f, 1), (4, f.astype(np.float32), 1)):
        nulls = (rng.random(n) < 0.1).astype(np.uint8)
        cnt, hi, mn, mx = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
        lo = C.c_uint64()
        arr = np.ascontiguousarray(vals)
        capi.check(L.cg_agg_column(attlen, is_float, arr.ctypes.data, nulls.ctypes.data, n, C.byref(cnt), C.byref(hi),
                                   C.byref(lo), C.byref(mn), C.byref(mx)))
        w = ref.aggregate([np.asarray(vals, np.float64) if is_float else vals], [nulls], [], [],
                          [cg.count(0), cg.sum_(0, bool(is_float)), cg.min_(0, bool(is_float)), cg.max_(0, bool(is_float))],
                          (0,) if is_float else ()).groups[()]
        assert cnt.value == w[0].count
        if is_float:
            as_f = lambda b: float(np.int64(b).view(np.float64))
            assert ref.float8_eq(as_f(mn.value), w[2].min) and ref.float8_eq(as_f(mx.value), w[3].max)
        else:
            assert (hi.value << 64) + lo.value == w[1].sum and (mn.value, mx.value) == (w[2].min, w[3].max)


def test_merge_rows_low_words_that_add_past_2_64(cg):
    """two-limb sums keep the low 32 bits of every term in one unsigned word: merged rows whose low words add past
    2^64 give the exact sum (the carry moves to the high word), and a group that reaches 2^32 rows is refused"""
    import torch
    from citus_b200 import capi
    rel = cg.Relation.write([8, 8], [np.zeros(1, np.int64), np.zeros(1, np.int64)])
    aggs = [cg.sum_(1), cg.count_star()]
    for group in ([], [0]):
        d = cg.make_desc([], group, aggs)
        p = cg.GpuColumnarAgg(d, rel.column_descs(), 0, 3 if group else -1, 0)
        nw, ops, _, _ = p.layout()
        assert nw == 4                                           # rows, low word, high word, NULL inputs: the two-limb form
        rows = [[1, 2**64 - 5, 7, 0], [1, 2**63 + 9, -3, 0], [2, 2**64 - 1, 2**40, 0]]
        words = torch.tensor([[w - 2**64 if w >= 2**63 else w for w in r] for r in rows], dtype=torch.int64, device="cuda")
        keys = torch.full((3,), 2, dtype=torch.int64, device="cuda")
        kn = torch.zeros(3, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()                                 # the fills run on torch's stream, the merge on the library's
        p.merge_rows(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), 3)
        g = list(p.groups().values())[0]
        assert g[0]["sum"] == sum(r[1] + (r[2] << 32) for r in rows) and g[1]["count"] == 4
        big = torch.tensor([[2**32, 5, 0, 0]], dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        p.merge_rows(keys.data_ptr(), kn.data_ptr(), big.data_ptr(), 1)
        with pytest.raises(capi.CitusGpuError) as e:
            p.groups()
        assert e.value.code == capi.CG_EUNSUPPORTED
        p.free()
