"""CASE aggregate arguments in the fused scan and the join aggregate, exact against tests/reference.py on every
kernel family: random CASE trees with NULLs in WHEN and THEN columns, every ELSE form, groups where every row chose NULL
next to groups that chose ELSE 0, overflow and bound violations in chosen and unchosen arms, CASE with FILTER, every table
kind with packing on and off, the three staging paths, float sums, min and max with NaN, variance, an export / merge /
fetch round trip, and arms mixing build and probe attributes of a join."""
import dataclasses
import json
import math
import os

import numpy as np
import pytest

import join_agg_reference as jref
import reference as ref
from test_gpu_exact import NEG_NAN
from gpu_harness import cg, kernel_family, FAMILIES  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def run(cg, rel, where, group_cols, aggs, float_cols=(), use_bounds=True, force_hash=False, e2e=False, packing=True,
        expected_groups=0):
    """one partial aggregate over `rel` (bounds from cg_relation_bounds); (stats, {key tuple: per-aggregate dicts})"""
    aggs = [dataclasses.replace(a) for a in aggs]
    d = cg.make_desc(where, group_cols, aggs, float_cols=float_cols, expected_groups=expected_groups)
    kmin, kmax, proven, rows = cg.relation_bounds(rel, d)
    for i, a in enumerate(aggs):
        a.term_abs_bound = proven[i] if use_bounds else 0
    d = cg.make_desc(where, group_cols, aggs, float_cols=float_cols, expected_groups=expected_groups)
    if force_hash:
        kmin, kmax = 0, -1
    agg = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, max(rows, 1))
    try:
        agg.set_packing(packing)
        if e2e:
            if e2e == "dma":
                rel.register()
            try:
                st = agg.scan_relation(rel)
            finally:
                if e2e == "dma":
                    rel.unregister()
        else:
            shard = cg.Shard(rel)
            st = agg.scan_shard(shard)
            shard.free()
        got = agg.groups()
    finally:
        agg.free()
    keyed = {}
    for k, per in got.items():
        keyed[() if not group_cols else (k,) if len(group_cols) == 1 else ref.unpack_two_column_key(k)] = per
    return st, keyed


def assert_exact(st, got, want, aggs, nrows):
    assert st.rows_passed == want.rows_passed
    assert st.rows_removed_by_filter + (nrows - st.rows_scanned) == want.rows_removed
    if () in got and () not in want.groups:
        assert all(g["count"] == 0 for g in got[()])
        return
    assert set(got) == set(want.groups)
    for key, per in want.groups.items():
        for a, (spec, w) in enumerate(zip(aggs, per)):
            g = got[key][a]
            assert g["count"] == w.count, (key, a)
            if spec.kind in (0, 1) or w.count == 0:
                continue
            if spec.kind == 2 and spec.is_float:
                assert w.float_sum_ok(g["fsum"]), (key, a, g["fsum"], w.float_sum())
            elif spec.kind in (2, 9):
                assert g["sum"] == w.sum, (key, a)
                if spec.kind == 9:
                    assert g["sumsq"] == w.sumsq, (key, a)
            else:
                wantv = w.min if spec.kind == 3 else w.max
                if spec.is_float:
                    assert ref.float8_eq(float(np.int64(g["minmax"]).view(np.float64)), wantv), (key, a)
                else:
                    assert g["minmax"] == wantv, (key, a)


def check(cg, rel, cols, nulls, where, group_cols, aggs, n, float_cols=(), **kw):
    from citus_b200 import capi
    want = ref.aggregate(cols, nulls, where, group_cols, aggs, float_cols)
    if ref.overflows(want):
        with pytest.raises(capi.CitusGpuError) as e:
            run(cg, rel, where, group_cols, aggs, float_cols=float_cols, **kw)
        assert e.value.code == capi.CG_EUNSUPPORTED, str(e.value)
        return None
    st, got = run(cg, rel, where, group_cols, aggs, float_cols=float_cols, **kw)
    assert_exact(st, got, want, aggs, n)
    return got


def relation(cg, rng, n=12_000, stripe_rows=4000, chunk_rows=1000):
    """k int2 0..4, m int4 0..7 (no NULLs: group keys), x int2, y int4, z int8 near 2^62, w int8 small, f float8 with NaN
    / inf / -0.0; NULL-bearing chunk groups, one all-NULL chunk in z and f, and NULL-free chunk groups"""
    k = rng.integers(0, 5, n)
    m = rng.integers(0, 8, n)
    x = rng.integers(-2**15, 2**15, n)
    y = rng.integers(-2**31, 2**31, n)
    z = rng.integers(-2**62, 2**62, n)
    w = rng.integers(-1000, 1000, n)
    f = rng.normal(size=n) * 1e3
    sp = np.array([math.nan, NEG_NAN, math.inf, -math.inf, -0.0, 0.0])
    pick = rng.random(n) < 0.01
    f[pick] = sp[rng.integers(0, len(sp), int(pick.sum()))]
    cols = [k, m, x, y, z, w, f]
    nulls = [None, None] + [(rng.random(n) < rate).astype(np.uint8) for rate in (0.05, 0.05, 0.1, 0.1, 0.05)]
    for c in range(2, 7):
        nulls[c][3 * chunk_rows:5 * chunk_rows] = 0         # NULL-free chunk groups: the generated kernel's plain form
    nulls[4][chunk_rows:2 * chunk_rows] = 1
    nulls[6][chunk_rows:2 * chunk_rows] = 1
    rel = cg.Relation.write([2, 4, 2, 4, 8, 8, 8], cols, nulls, type_classes=[0, 0, 0, 0, 0, 0, 1], stripe_row_limit=stripe_rows,
                            chunk_row_limit=chunk_rows)
    return rel, cols, nulls


def random_case(cg, rng, is_float=False):
    """a CASE of 1..3 arms over comparison, IN, IS NULL and column atoms, with product, constant and NULL results and
    every ELSE form"""
    Case, Const, Col = cg.Case, cg.Const, cg.Col

    def atom():
        r = rng.random()
        if r < 0.15:
            return (int(rng.choice([2, 3, 5])), "is null" if rng.random() < 0.5 else "is not null")
        if r < 0.3:
            return (1, "in", tuple(int(v) for v in rng.integers(0, 8, 3)) + ((None,) if rng.random() < 0.3 else ()))
        if r < 0.45:
            return (2, "<", Col(5))
        c = int(rng.choice([0, 1, 2, 5]))
        return (c, ["<", "<=", "=", ">=", ">", "<>"][int(rng.integers(0, 6))], int(rng.integers(-3, 8)) * (100 if c in (2, 5) else 1))

    def tree():
        if rng.random() < 0.4:
            return atom()
        return (["and", "or"][int(rng.integers(0, 2))], atom(), atom())

    def result():
        r = rng.random()
        if is_float:
            return None if r < 0.15 else Const(float(rng.integers(-5, 5)) / 4) if r < 0.4 else 6
        if r < 0.15:
            return None
        if r < 0.4:
            return Const(int(rng.integers(-10**6, 10**6)))
        if r < 0.7:
            return int(rng.choice([2, 3, 5]))
        return [(int(rng.choice([2, 5])), int(rng.integers(-3, 4)), int(rng.integers(-3, 4))), (5, 1, int(rng.integers(-2, 3)))]
    arms = [(tree(), result()) for _ in range(int(rng.integers(1, 4)))]
    e = rng.random()
    return Case(arms) if e < 0.25 else Case(arms, else_=None) if e < 0.4 else Case(arms, else_=(Const(0.0) if is_float else Const(0))) \
        if e < 0.7 else Case(arms, else_=result())


SHAPES = [dict(group_cols=[]), dict(group_cols=[0]), dict(group_cols=[1]), dict(group_cols=[0, 1]),
          dict(group_cols=[1], expected_groups=4096, force_hash=True)]


@pytest.mark.parametrize("family", FAMILIES)
def test_random_case_trees_on_every_table_kind(cg, kernel_family, family):
    from citus_b200 import capi
    kernel_family(family)
    rng = np.random.default_rng(20261019)
    rel, cols, nulls = relation(cg, rng)
    n = len(cols[0])
    for trial in range(12):
        shape = SHAPES[trial % len(SHAPES)]
        while True:
            c1, c2 = random_case(cg, rng), random_case(cg, rng)
            aggs = [cg.sum_(c1), cg.count(c1), cg.min_(c2), cg.max_(c2, filter=(0, "<>", 2)), cg.count_star(), cg.sum_(5)]
            try:
                cg.make_desc([], [], aggs)       # the WHEN atoms of both CASEs and the FILTER fit the pool
                break
            except capi.CitusGpuError as e:
                assert e.code == capi.CG_EUNSUPPORTED
        where = [(3, ">", -2**31 + 1000)] if trial % 2 else []
        check(cg, rel, cols, nulls, where, shape["group_cols"], aggs, n, float_cols=(6,), use_bounds=trial % 3 != 0,
              force_hash=shape.get("force_hash", False), expected_groups=shape.get("expected_groups", 0), packing=trial % 4 < 2)


@pytest.mark.parametrize("family", FAMILIES)
def test_pivot_else_zero_against_filter_and_null_groups(cg, kernel_family, family):
    """sum(CASE WHEN m = i THEN w ELSE 0 END) is 0 where sum(w) FILTER (WHERE m = i) is NULL; count(CASE WHEN m = i THEN
    1 END) counts the rows of m = i; a CASE whose every chosen arm is NULL gives NULL and count 0 in every group"""
    kernel_family(family)
    Case, Const = cg.Case, cg.Const
    rng = np.random.default_rng(5)
    n = 8000
    k = rng.integers(0, 6, n)
    m = np.where(k == 5, 7, rng.integers(0, 4, n))          # group 5 never has m < 4
    w = rng.integers(-100, 100, n)
    cols, nulls = [k, m, w], [None, None, (rng.random(n) < 0.05).astype(np.uint8)]
    rel = cg.Relation.write([8, 8, 8], cols, nulls, stripe_row_limit=3000, chunk_row_limit=1000)
    aggs = []
    for i in range(4):
        aggs.append(cg.sum_(Case([((1, "=", i), 2)], else_=Const(0))))
    aggs += [cg.sum_(2, filter=(1, "=", 0)), cg.count(Case([((1, "=", 1), Const(1))])),
             cg.sum_(Case([((1, "=", 1), None)], else_=None))]
    for packing in (True, False):
        got = check(cg, rel, cols, nulls, [], [0], aggs, n, packing=packing)
        assert got[(5,)][0]["count"] > 0 and got[(5,)][0]["sum"] == 0
        assert got[(5,)][4]["count"] == 0
        assert all(per[6]["count"] == 0 for per in got.values())


@pytest.mark.parametrize("family", FAMILIES)
def test_overflow_and_bound_only_in_the_chosen_arm(cg, kernel_family, family):
    from citus_b200 import capi
    kernel_family(family)
    Case, Const = cg.Case, cg.Const
    n = 4000
    x = np.full(n, 2**40, dtype=np.int64)
    sel = np.zeros(n, dtype=np.int64)
    rel = cg.Relation.write([8, 8], [x, sel], None, stripe_row_limit=2000, chunk_row_limit=1000)
    big = Case([((1, "=", 1), [(0, 0, 2**30)])], else_=Const(5))        # 2^70 in the arm never chosen
    st, got = run(cg, rel, [], [], [cg.sum_(big), cg.max_(big)], use_bounds=False)
    assert (got[()][0]["sum"], got[()][1]["minmax"]) == (5 * n, 5)
    sel2 = sel.copy()
    sel2[1234] = 1
    rel2 = cg.Relation.write([8, 8], [x, sel2], None, stripe_row_limit=2000, chunk_row_limit=1000)
    with pytest.raises(capi.CitusGpuError) as e:
        run(cg, rel2, [], [], [cg.sum_(big)], use_bounds=False)
    assert e.value.code == capi.CG_EUNSUPPORTED
    # a term bound that only an unchosen arm would violate raises nothing; the chosen arm's violation is CG_EINVAL
    small = Case([((1, "=", 1), 0)], else_=Const(3))
    aggs = [dataclasses.replace(cg.sum_(small), term_abs_bound=3)]
    d = cg.make_desc([], [], aggs)
    for r, want in ((rel, 3 * n), (rel2, None)):
        agg = cg.GpuColumnarAgg(d, r.column_descs(), 0, -1, n)
        try:
            shard = cg.Shard(r)
            try:
                if want is None:
                    with pytest.raises(capi.CitusGpuError) as e:
                        agg.scan_shard(shard)
                        agg.groups()
                    assert e.value.code == capi.CG_EINVAL
                else:
                    agg.scan_shard(shard)
                    assert list(agg.groups().values())[0][0]["sum"] == want
            finally:
                shard.free()
        finally:
            agg.free()


@pytest.mark.parametrize("family", FAMILIES)
def test_staging_paths_and_float_cases(cg, kernel_family, family):
    """float CASE sums within the float tolerance, min / max exact with NaN and -0.0, over host pages, registered pages
    and a staged shard"""
    kernel_family(family)
    rng = np.random.default_rng(99)
    rel, cols, nulls = relation(cg, rng)
    n = len(cols[0])
    Case, Const = cg.Case, cg.Const
    fcase = Case([((6, ">", 0.0), 6), ((1, "<", 3), Const(-0.0)), ((2, "is null"), Const(math.nan))], else_=None)
    icase = random_case(cg, rng)
    aggs = [cg.sum_(fcase, is_float=True), cg.min_(fcase, is_float=True), cg.max_(fcase, is_float=True), cg.count(fcase, is_float=True),
            cg.sum_(icase)]
    for e2e in (False, True, "dma"):
        for shape in SHAPES[:3]:
            check(cg, rel, cols, nulls, [], shape["group_cols"], aggs, n, float_cols=(6,), e2e=e2e)


@pytest.mark.parametrize("family", FAMILIES)
def test_variance_over_case_to_exact_text(cg, kernel_family, family):
    from citus_b200 import capi
    kernel_family(family)
    Case, Const = cg.Case, cg.Const
    rng = np.random.default_rng(3)
    n = 6000
    g = rng.integers(0, 4, n)
    v = rng.integers(-10**6, 10**6, n)
    nv = (rng.random(n) < 0.1).astype(np.uint8)
    cols, nulls = [g, v], [None, nv]
    rel = cg.Relation.write([8, 8], cols, nulls, stripe_row_limit=3000, chunk_row_limit=1000)
    case = Case([((0, "=", 0), None), ((0, "=", 1), Const(250))], else_=[(1, 0, 1)])
    aggs = [cg.variance(case)]
    for use_bounds in (True, False):
        got = check(cg, rel, cols, nulls, [], [0], aggs, n, use_bounds=use_bounds)
        want = ref.aggregate(cols, nulls, [], [0], aggs)
        for key, per in want.groups.items():
            w, gg = per[0], got[key][0]
            for final in (capi.CG_VAR_POP, capi.CG_VAR_SAMP, capi.CG_STDDEV_POP, capi.CG_STDDEV_SAMP):
                assert cg.numeric_var_out(final, gg["count"], gg["sum"], gg["sumsq"], 0) == ref.var_out(final, w.count, w.sum, w.sumsq, 0), \
                    (key, final)


def test_export_merge_fetch_round_trip(cg):
    import torch
    Case, Const = cg.Case, cg.Const
    rng = np.random.default_rng(8)
    rel, cols, nulls = relation(cg, rng)
    n = len(cols[0])
    case = Case([((1, "<", 4), 5), ((2, "is null"), Const(-1))], else_=Const(0))
    aggs = [cg.sum_(case), cg.count(case), cg.min_(case), cg.max_(case)]
    d = cg.make_desc([], [0], aggs)
    kmin, kmax, _, rows = cg.relation_bounds(rel, d)
    a = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, rows)
    b = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, 2 * rows)
    try:
        shard = cg.Shard(rel)
        a.scan_shard(shard)
        b.scan_shard(shard)
        shard.free()
        nwords = a.layout()[0]
        keys = torch.zeros(64, dtype=torch.int64, device="cuda")
        knull = torch.zeros(64, dtype=torch.uint8, device="cuda")
        words = torch.zeros(64 * nwords, dtype=torch.int64, device="cuda")
        nrows = a.export_device(keys.data_ptr(), knull.data_ptr(), words.data_ptr(), 64)
        b.merge_rows(keys.data_ptr(), knull.data_ptr(), words.data_ptr(), nrows)
        got = b.groups()
    finally:
        a.free()
        b.free()
    # b holds its own scan plus a's exported rows: counts and sums twice, min and max once
    want = ref.aggregate(cols, nulls, [], [0], aggs, float_cols=(6,))
    for (key,), (s, c, lo, hi) in want.groups.items():
        g = got[key]
        assert [g[j]["count"] for j in range(4)] == [2 * s.count, 2 * c.count, 2 * lo.count, 2 * hi.count]
        assert (g[0]["sum"], g[2]["minmax"], g[3]["minmax"]) == (2 * s.sum, lo.min, hi.max)


@pytest.mark.parametrize("mode", ["plain", "dense", "hash"])
def test_join_aggregate_arms_mix_build_and_probe(cg, mode):
    """arms whose WHEN trees and products read both sides of the join, against join_agg_reference + the CASE reference"""
    import torch
    Case, Const, Col = cg.Case, cg.Const, cg.Col
    rng = np.random.default_rng(21)
    nb, npr = 3000, 5000
    bk = rng.integers(0, 800, nb)
    bx = rng.integers(-50, 50, nb)
    bn = (rng.random(nb) < 0.1).astype(np.uint8)
    pk = rng.integers(0, 900, npr)
    py = rng.integers(-50, 50, npr)
    pg = rng.integers(0, 5, npr)
    pn = (rng.random(npr) < 0.1).astype(np.uint8)
    bcols, bnulls, pcols, pnulls = [bk, bx], [None, bn], [pk, py, pg], [None, pn, None]
    jcols, jnulls = jref.join(bcols, bnulls, 0, pcols, pnulls, 0)
    # attributes: 0 b.key, 1 b.x, 2 p.key, 3 p.y, 4 p.g
    case = Case([((1, "<", Col(3)), [(1, 0, 1), (3, 1, 1)]), (("or", (4, "in", (1, 2)), (1, "is null")), Const(7))], else_=3)
    aggs = [cg.sum_(case), cg.count(case), cg.min_(case, filter=(4, "<>", 0)), cg.max_(case), cg.variance(case)]
    group = [] if mode == "plain" else [4]
    where = [(3, ">", -40)]
    want = ref.aggregate(jcols, jnulls, where, group, aggs)
    d = cg.make_desc(where, group, aggs, expected_groups=16 if mode == "hash" else 0)
    colspec = [(8, 0)] * 5
    kmin, kmax = (0, 4) if mode == "dense" else (0, -1)
    agg = cg.GpuColumnarAgg(d, colspec, kmin, kmax, len(jcols[0]) + 1)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    bt, pt = [dev(c.astype(np.int64)) for c in bcols], [dev(c.astype(np.int64)) for c in pcols]
    bnt, pnt = [None, dev(bn)], [None, dev(pn), None]
    try:
        st = agg.join_aggregate([t.data_ptr() for t in bt], 0, nb, [t.data_ptr() for t in pt], 0, npr,
                           build_null_ptrs=[t.data_ptr() if t is not None else None for t in bnt],
                           probe_null_ptrs=[t.data_ptr() if t is not None else None for t in pnt], columns=colspec)
        torch.cuda.synchronize()
        got = agg.groups()
    finally:
        agg.free()
    keyed = {(() if not group else (k,)): per for k, per in got.items()}
    assert st.rows_scanned == len(jcols[0])              # the joined rows handed to WHERE
    assert_exact(st, keyed, want, aggs, len(jcols[0]))


# --------------------------------------------------------------------------- TPC-H goldens through the join aggregate
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _case_golden():
    z = np.load(os.path.join(GOLDEN, "case_golden.npz"))
    with open(os.path.join(GOLDEN, "case_golden.json")) as f:
        return {k: z[k] for k in z.files}, json.load(f)


def _join(cg, build_cols, probe_cols, desc_where, group, aggs, kmin, kmax):
    """cg_join_aggregate of int64 host columns (key = column 0 of each side) into a fresh partial; groups()"""
    import torch
    d = cg.make_desc(desc_where, group, aggs)
    colspec = [(8, 0)] * (len(build_cols) + len(probe_cols))
    agg = cg.GpuColumnarAgg(d, colspec, kmin, kmax, len(probe_cols[0]) * 4)
    dev = [torch.from_numpy(np.ascontiguousarray(c, dtype=np.int64)).cuda() for c in list(build_cols) + list(probe_cols)]
    nb = len(build_cols)
    try:
        agg.join_aggregate([t.data_ptr() for t in dev[:nb]], 0, len(build_cols[0]), [t.data_ptr() for t in dev[nb:]], 0,
                           len(probe_cols[0]), columns=colspec)
        return agg.groups()
    finally:
        agg.free()


def _pgdate(s):
    import datetime
    return (datetime.date(*map(int, s.split("-"))) - datetime.date(2000, 1, 1)).days


def test_tpch_q12_through_the_join_aggregate(cg, lineitem):
    """multi_tpch_query12: orders (build) JOIN lineitem (probe), l_shipmode IN ('MAIL', 'SHIP'), two column atoms and the
    receipt-date range, GROUP BY l_shipmode; high / low line counts as sum(CASE ... THEN 1 ELSE 0 END)"""
    Case, Const, Col = cg.Case, cg.Const, cg.Col
    fx, want = _case_golden()
    modes = want["shipmodes"]
    # attributes: 0 o_orderkey, 1 o_orderpriority | 2 l_orderkey, 3 l_shipmode, 4 l_shipdate, 5 l_commitdate, 6 l_receiptdate
    build = [fx["o_orderkey"], fx["o_orderpriority"]]
    probe = [lineitem["l_orderkey"], fx["l_shipmode"], lineitem["l_shipdate"], lineitem["l_commitdate"], lineitem["l_receiptdate"]]
    where = [(3, "in", (modes.index("MAIL"), modes.index("SHIP"))), (5, "<", Col(6)), (4, "<", Col(5)),
             (6, ">=", _pgdate("1994-01-01")), (6, "<", _pgdate("1995-01-01"))]
    high = Case([(("or", (1, "=", 1), (1, "=", 2)), Const(1))], else_=Const(0))
    low = Case([(("and", (1, "<>", 1), (1, "<>", 2)), Const(1))], else_=Const(0))
    got = _join(cg, build, probe, where, [3], [cg.sum_(high), cg.sum_(low)], 0, len(modes) - 1)
    rows = sorted([modes[k], str(per[0]["sum"]), str(per[1]["sum"])] for k, per in got.items())
    assert rows == want["q12"]


def test_tpch_q14_through_the_join_aggregate(cg, oracle, lineitem):
    """multi_tpch_query14: part (build) JOIN lineitem (probe) over a year of l_shipdate; 100.00 * sum(CASE WHEN p_type LIKE
    'PROMO%' THEN l_extendedprice * (1 - l_discount) ELSE 0 END) / sum(l_extendedprice * (1 - l_discount)), both sums at
    scale 4"""
    Case, Const = cg.Case, cg.Const
    fx, want = _case_golden()
    # attributes: 0 p_partkey, 1 p_promo | 2 l_partkey, 3 l_extendedprice, 4 l_discount, 5 l_shipdate
    build = [fx["p_partkey"], fx["p_promo"]]
    probe = [lineitem["l_partkey"], lineitem["l_extendedprice"], lineitem["l_discount"], lineitem["l_shipdate"]]
    where = [(5, ">=", _pgdate("1995-09-01")), (5, "<", _pgdate("1996-09-01"))]
    revenue = [(3, 0, 1), (4, 100, -1)]
    aggs = [cg.sum_(Case([((1, "=", 1), revenue)], else_=Const(0))), cg.Agg(2, revenue), cg.count_star()]
    got = _join(cg, build, probe, where, [], aggs, 0, -1)
    (per,) = got.values()
    num, den = per[0]["sum"], per[1]["sum"]
    assert per[2]["count"] == 10
    assert oracle.numeric_div_str(10000 * num, 6, den, 4) == want["q14"][0][0]
