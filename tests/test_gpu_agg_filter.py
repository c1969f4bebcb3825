"""Aggregate FILTER (WHERE ...) in the fused scan against the exact reference (tests/reference.py), on every kernel
family: the groups come from WHERE alone, a row its FILTER does not find TRUE is no input of that aggregate, and a group
without such rows has count 0 / SQL NULL."""
import dataclasses
import math

import numpy as np
import pytest

import reference as ref
from test_gpu_exact import NEG_NAN, assert_matches_reference, gpu_run
from test_where_reference import constant_pools, random_tree
from gpu_harness import cg, kernel_family, FAMILIES  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

OPS = ("<", "<=", "=", ">=", ">", "<>")
SHAPES = [dict(group_cols=[]), dict(group_cols=[0]), dict(group_cols=[0, 1]), dict(group_cols=[2], expected_groups=4096, force_hash=True)]


def check(cg, rel, cols, nulls, where, group_cols, aggs, n, float_cols=(), **kw):
    """the scan equals the reference; the WHERE counters equal those of the same query without filters"""
    from citus_b200 import capi
    want = ref.aggregate(cols, nulls, where, group_cols, aggs, float_cols)
    if ref.overflows(want):
        with pytest.raises(capi.CitusGpuError) as e:
            gpu_run(cg, rel, where, group_cols, aggs, float_cols=float_cols, **kw)
        assert e.value.code == capi.CG_EUNSUPPORTED, str(e.value)
        return None
    st, got, layout = gpu_run(cg, rel, where, group_cols, aggs, float_cols=float_cols, **kw)
    assert_matches_reference(st, got, want, aggs, n)
    # the counters depend on WHERE alone (count(*) only: dropping a filter may expose an argument error)
    st0, _, _ = gpu_run(cg, rel, where, group_cols, [cg.count_star()], float_cols=float_cols, **kw)
    assert (st.rows_scanned, st.rows_removed_by_filter, st.chunk_groups_filtered) == \
        (st0.rows_scanned, st0.rows_removed_by_filter, st0.chunk_groups_filtered)
    return got


def mixed_relation(cg, rng, n=12_000, stripe_rows=4000, chunk_rows=1000):
    """k1 int2 0..4, k2 int4 0..2 (no NULLs: group keys), x int2 / y int4 / z int8 / f float8 at their types' edges, with
    NULL-bearing chunk groups (an all-NULL chunk in z and f)"""
    k1 = rng.integers(0, 5, n)
    k2 = rng.integers(0, 3, n)
    x = rng.integers(-2**15, 2**15, n)
    y = rng.integers(-2**31, 2**31, n)
    z = rng.integers(-2**62, 2**62, n)
    f = rng.normal(size=n) * 1e3
    sp = np.array([math.nan, NEG_NAN, math.inf, -math.inf, -0.0, 0.0])
    pick = rng.random(n) < 0.01
    f[pick] = sp[rng.integers(0, len(sp), int(pick.sum()))]
    x[:2], y[:2], z[:2] = [-2**15, 2**15 - 1], [-2**31, 2**31 - 1], [-2**62, 2**62 - 1]
    cols = [k1, k2, x, y, z, f]
    nulls = [None, None] + [(rng.random(n) < rate).astype(np.uint8) for rate in (0.05, 0.0, 0.1, 0.05)]
    nulls[4][chunk_rows:2 * chunk_rows] = 1
    nulls[5][chunk_rows:2 * chunk_rows] = 1
    rel = cg.Relation.write([2, 4, 2, 4, 8, 8], cols, nulls, type_classes=[0, 0, 0, 0, 0, 1], stripe_row_limit=stripe_rows,
                            chunk_row_limit=chunk_rows)
    return rel, cols, nulls, stripe_rows, chunk_rows


@pytest.mark.parametrize("family", FAMILIES)
def test_random_where_and_filter_trees(cg, kernel_family, family):
    """random WHERE trees x random per-aggregate FILTER trees over int2 / int4 / int8 / float8 columns (NaN, +-inf, NULL
    chunks) with constants at chunk min / max and the types' edges: plain aggregate, one- and two-column direct-indexed
    tables and the hash table"""
    kernel_family(family)
    rng = np.random.default_rng(20261017)
    rel, cols, nulls, sr, cr = mixed_relation(cg, rng)
    fc = (5,)
    minmax = ref.skip_minmax(cols, nulls, sr, cr, fc)
    pools = constant_pools(minmax, [2, 4, 2, 4, 8, 8], fc)

    def atom():
        c = int(rng.integers(0, 6))
        return (c, OPS[int(rng.integers(0, 6))], pools[c][int(rng.integers(0, len(pools[c])))])

    def small_atom():                                            # atoms that keep some rows and reject others
        c = int(rng.integers(0, 6))
        return (c, OPS[int(rng.integers(0, 6))], [2, 1, 0, 0, 0, 0.0][c])
    base = [cg.count_star(), cg.count(4), cg.sum_(3), cg.min_(2), cg.max_(5, True), cg.sum_(5, True), cg.sum_(4), cg.count_star()]
    for trial in range(6):
        aggs = [dataclasses.replace(a) for a in base]
        budget = 8
        for j in rng.permutation(len(aggs))[:int(rng.integers(2, 7))]:
            if budget < 1:
                break
            tree = random_tree(rng, small_atom if rng.random() < 0.6 else atom, min(3, budget))
            aggs[j] = dataclasses.replace(aggs[j], filter=tree)
            budget -= len(cg.flatten_where(tree)[0]) if isinstance(tree, tuple) else len(tree)
        where = random_tree(rng, small_atom, 3) if trial % 2 else []
        for shape in SHAPES:
            check(cg, rel, cols, nulls, where, aggs=aggs, n=len(cols[0]), float_cols=fc, **shape)


@pytest.mark.parametrize("family", FAMILIES)
def test_groups_without_accepted_rows(cg, kernel_family, family):
    """a group whose every row a FILTER rejects: count(*) / count(x) 0, sum / min / max NULL; a FILTER that matches
    nothing while its groups exist; the plain aggregate over zero accepted rows and over zero WHERE rows"""
    kernel_family(family)
    rng = np.random.default_rng(3)
    n = 20_000
    k = rng.integers(0, 6, n)
    v = rng.integers(-1000, 1000, n)
    f = rng.normal(size=n)
    cols = [k, rng.integers(0, 2, n), v, f]
    rel = cg.Relation.write([8, 8, 8, 8], cols, type_classes=[0, 0, 0, 1], chunk_row_limit=2500)
    rej = ("or", (0, "=", 1), (0, "=", 4))                       # groups 0, 2, 3, 5 reject every row
    aggs = [cg.count_star(filter=rej), cg.count(2, filter=rej), cg.sum_(2, filter=rej), cg.min_(2, filter=rej),
            cg.max_(3, True, filter=rej), cg.sum_(3, True, filter=(2, ">", 5000)), cg.count_star(), cg.sum_(2)]
    for shape in SHAPES[:2] + SHAPES[3:]:
        got = check(cg, rel, cols, None, [], aggs=aggs, n=n, float_cols=(3,), **dict(shape, group_cols=[0] if shape["group_cols"] else []))
        if shape["group_cols"]:
            assert len(got) == 6 and all(got[(g,)][a]["count"] == 0 for g in (0, 2, 3, 5) for a in range(6))
    nothing = [cg.count_star(filter=(2, ">", 5000)), cg.sum_(2, filter=(2, ">", 5000)), cg.max_(3, True, filter=(2, "<", -5000))]
    got = check(cg, rel, cols, None, [], [], nothing, n, float_cols=(3,))
    assert [g["count"] for g in got[()]] == [0, 0, 0]
    got = check(cg, rel, cols, None, [(2, ">", 5000)], [], nothing, n, float_cols=(3,))
    assert [g["count"] for g in got[()]] == [0, 0, 0]


@pytest.mark.parametrize("family", FAMILIES)
def test_argument_errors_only_on_accepted_rows(cg, kernel_family, family):
    """an integer argument that leaves int64 only on rejected rows is exact; on one accepted row it is CG_EUNSUPPORTED.
    A term_abs_bound violated only by rejected rows is no error; violated by an accepted row it is CG_EINVAL"""
    from citus_b200 import capi
    kernel_family(family)
    rng = np.random.default_rng(9)
    n = 16_000
    k = rng.integers(0, 4, n)
    x = rng.integers(-1000, 1000, n)
    big = np.flatnonzero(rng.random(n) < 0.01)
    x[big] = 2**40 + 7
    cols = [k, x, rng.integers(0, 100, n)]
    rel = cg.Relation.write([8, 8, 8], cols, chunk_row_limit=2000)
    sq = lambda flt: cg.Agg(2, [(1, 0, 1), (1, 0, 1)], filter=flt)
    for group, hash_ in (([], False), ([0], False), ([0], True)):
        kw = dict(use_bounds=False, force_hash=hash_, expected_groups=16)
        check(cg, rel, cols, None, [], group, [sq((1, "<", 2**20)), cg.count_star(filter=(1, ">", 0))], n, **kw)
        with pytest.raises(capi.CitusGpuError) as e:
            gpu_run(cg, rel, [], group, [sq(("or", (1, "<", 2**20), (2, "=", int(cols[2][big[0]])))), cg.count_star()], **kw)
        assert e.value.code == capi.CG_EUNSUPPORTED
        # bound 1000: only the rows the filter rejects break it
        agg = [cg.sum_(1, filter=("and", (1, ">=", -1000), (1, "<=", 1000))), cg.count_star()]
        st, got, _ = gpu_run(cg, rel, [], group, agg, bounds=[1000, 0], force_hash=hash_, expected_groups=16)
        assert_matches_reference(st, got, ref.aggregate(cols, None, [], group, agg), agg, n)
        with pytest.raises(capi.CitusGpuError) as e:
            gpu_run(cg, rel, [], group, [cg.sum_(1, filter=(1, ">", -5000)), cg.count_star()], bounds=[1000, 0], force_hash=hash_,
                    expected_groups=16)
        assert e.value.code == capi.CG_EINVAL


def scan_relation(cg, rel, where, group, aggs, dma):
    """cg_scan_relation from the pages (pageable, or registered: DMA); groups keyed like the reference"""
    d = cg.make_desc(where, group, aggs)
    kmin, kmax, _, rows = cg.relation_bounds(rel, d)
    part = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, max(rows, 1))
    try:
        if dma:
            rel.register()
        try:
            st = part.scan_relation(rel)
        finally:
            rel.unregister()
        got = {((k,) if group else ()): per for k, per in part.groups().items()}
    finally:
        part.free()
    return st, got


@pytest.mark.parametrize("family", FAMILIES)
def test_filter_only_column_is_staged(cg, kernel_family, family):
    """a column read only by a FILTER is staged by cg_scan_relation, pageable and registered (DMA): the h2d bytes are
    those of a query that reads the same columns, and the removal counters those of the query without the filter"""
    kernel_family(family)
    rng = np.random.default_rng(11)
    n = 30_000
    cols = [rng.integers(0, 4, n), np.sort(rng.integers(0, 10**6, n)), rng.integers(-50, 50, n), rng.integers(0, 10**9, n)]
    rel = cg.Relation.write([8, 8, 8, 8], cols, chunk_row_limit=5000)
    where = [(1, "<", 400_000)]
    aggs = [cg.count_star(filter=(2, ">", 10)), cg.sum_(1)]
    same_cols = [cg.count_star(), cg.sum_(1), cg.max_(2)]
    for dma in (False, True):
        for group in ([], [0]):
            st, got = scan_relation(cg, rel, where, group, aggs, dma)
            assert_matches_reference(st, got, ref.aggregate(cols, None, where, group, aggs), aggs, n)
            st2, _ = scan_relation(cg, rel, where, group, same_cols, dma)
            assert st.h2d_bytes == st2.h2d_bytes and st.h2d_bytes > 0
            assert (st.chunk_groups_filtered, st.rows_removed_by_filter, st.rows_scanned) == \
                (st2.chunk_groups_filtered, st2.rows_removed_by_filter, st2.rows_scanned)
            assert st.chunk_groups_filtered > 0


@pytest.mark.parametrize("family", FAMILIES)
def test_q1_shape_with_filters_packing_on_and_off(cg, oracle, kernel_family, family):
    """Q1 over decimal(15,2) / char(1) columns (the shared-memory kind: 6 groups) plus count(*) FILTER (discount > 5),
    sum(price) FILTER (shipdate >= -1000) and sum(quantity) FILTER (returnflag = 'A' OR tax < 3), with the packed
    count+sum word on and off"""
    kernel_family(family)
    NUM2 = 2 | (2 << 8)
    rng = np.random.default_rng(19)
    n = 8000
    q = rng.integers(1, 51, n) * 100
    p = rng.integers(10**5, 10**8, n)
    d = rng.integers(0, 11, n)
    t = rng.integers(0, 9, n)
    rf = rng.choice([65, 78, 82], n)
    ls = rng.choice([70, 79], n)
    sd = rng.integers(-2000, 2000, n)
    cols = [q, p, d, t, rf, ls, sd]
    tab = oracle.Table([-1, -1, -1, -1, -1, -1, 4], [NUM2, NUM2, NUM2, NUM2, 3, 3, 0], stripe_row_limit=3000, chunk_row_limit=1000)
    tab.insert(cols)
    rel = cg.Relation.from_image(tab.pages(), tab.stripes_array(), tab.nodes_array(), [-1] * 6 + [4], [NUM2] * 4 + [3, 3, 0])
    aggs = [cg.sum_(0), cg.sum_(1), cg.Agg(2, [(1, 0, 1), (2, 100, -1)]), cg.count_star(),
            cg.count_star(filter=(2, ">", 5)), cg.sum_(1, filter=(6, ">=", -1000)), cg.sum_(0, filter=("or", (4, "=", 65), (3, "<", 3)))]
    want = ref.aggregate(cols, None, [(6, "<=", 1500)], [4, 5], aggs)
    for packing in (True, False):
        a = [dataclasses.replace(x) for x in aggs]
        dsc = cg.make_desc([(6, "<=", 1500)], [4, 5], a, expected_groups=16)
        kmin, kmax, bounds, rows = cg.relation_bounds(rel, dsc)
        for i, x in enumerate(a):
            x.term_abs_bound = bounds[i]
        dsc = cg.make_desc([(6, "<=", 1500)], [4, 5], a, expected_groups=16)
        part = cg.GpuColumnarAgg(dsc, rel.column_descs(), kmin, kmax, rows)
        part.set_packing(packing)
        for e2e in ("shard", "relation"):
            part.reset()
            st = part.scan_shard(cg.Shard(rel)) if e2e == "shard" else part.scan_relation(rel)
            got = {ref.unpack_two_column_key(k): per for k, per in part.groups().items()}
            assert_matches_reference(st, got, want, a, n)
        part.free()


def test_export_merge_and_fetch_merge_values_round_trips(cg):
    """a filtered partial through export_device -> merge_rows and fetch -> merge_values equals the reference over all
    rows; also with a filtered count(*) and no unfiltered one"""
    import torch
    from citus_b200 import capi
    L = capi.lib()
    rng = np.random.default_rng(41)
    n = 30_000
    k = rng.integers(0, 6, n)
    v = rng.integers(-10**12, 10**12, n)
    f = rng.normal(size=n)
    cols = [k, v, f]
    halves = [slice(0, n // 2), slice(n // 2, n)]
    rels = [cg.Relation.write([8, 8, 8], [c[h] for c in cols], type_classes=[0, 0, 1]) for h in halves]
    F = ("or", (0, "=", 2), (1, ">", 0))
    lists = [[cg.sum_(1, filter=F), cg.min_(1, filter=(0, "=", 5)), cg.max_(2, True, filter=F), cg.count_star(filter=(0, "<", 3)),
              cg.count(1, filter=(2, ">", 0.0)), cg.count_star()],
             [cg.count_star(filter=(0, "<", 3)), cg.sum_(1, filter=(0, ">=", 3))]]
    for aggs in lists:
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
