"""Column-to-column atoms (column, op, Col(other)) in the fused scan against the exact reference
(tests/reference.py), on every kernel family: groups and aggregates, rows scanned, rows removed by the
filter and chunk groups removed by the filter, in WHERE, in FILTERs and in bool_and / bool_or arguments, over every
same-class pair of column types, NULLs on either side, NaN / +-0.0 / +-inf, numeric scale alignment beyond 64 bits, and
the TPC-H Q12 predicates over the lineitem fixture."""
import dataclasses
import datetime
import math

import numpy as np
import pytest

import reference as ref
from test_gpu_agg_filter import mixed_relation
from test_gpu_bool_bit_agg import assert_exact
from test_gpu_in_null_atoms import OPS, keyed, small_tree, typed_relation
from test_where_reference import constant_pools
from gpu_harness import cg, kernel_family, FAMILIES  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
BPCHAR1 = 3


def NUMERIC(s):
    return 2 | (s << 8)


def run(cg, rel, where, group, aggs, float_cols=(), stage="shard", expected_groups=0, force_hash=False, packing=True):
    """a partial with the skip lists' key range and term bounds, as a caller plans one, scanned through one staging path"""
    aggs = [dataclasses.replace(a) for a in aggs]
    d = cg.make_desc(where, group, aggs, float_cols=float_cols, expected_groups=expected_groups)
    kmin, kmax, proven, rows = cg.relation_bounds(rel, d)
    for a, b in zip(aggs, proven):
        a.term_abs_bound = b
    d = cg.make_desc(where, group, aggs, float_cols=float_cols, expected_groups=expected_groups)
    if force_hash:
        kmin, kmax = 0, -1
    agg = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, max(rows, 1))
    if not packing:
        agg.set_packing(False)
    try:
        if stage == "shard":
            shard = cg.Shard(rel)
            st = agg.scan_shard(shard)
            shard.free()
        elif stage == "pageable":
            st = agg.scan_relation(rel)
        else:
            rel.register()
            try:
                st = agg.scan_relation(rel)
            finally:
                rel.unregister()
        got = keyed(agg.groups(), group)
    finally:
        agg.free()
    return st, got


_WANT = {}


def check(cg, rel, cols, nulls, where, group, aggs, stripe_rows, chunk_rows, float_cols=(), scales=None, key=None, **kw):
    """groups, aggregates and the three counters equal the reference's"""
    n = len(cols[0])
    ck = (key, repr(where), tuple(group), repr(aggs))
    if key is None or ck not in _WANT:
        want = ref.aggregate(cols, nulls, where, group, aggs, float_cols, scales)
        mask = ref.selected_chunk_mask(cols, nulls, where, stripe_rows, chunk_rows, float_cols=float_cols)
        _WANT[ck] = (want, mask)
    want, mask = _WANT[ck]
    st, got = run(cg, rel, where, group, aggs, float_cols, **kw)
    assert st.chunk_groups_filtered == ref.chunks_filtered(mask), where
    assert st.rows_scanned == ref.rows_kept(mask, n, stripe_rows, chunk_rows), where
    assert_exact(st, got, want, aggs, n)
    return st, got


def jit_launches():
    from citus_b200 import capi
    return capi.lib().cg_jit_launches()


# --------------------------------------------------------------------------- random trees
SHAPES = [dict(group=[]), dict(group=[0]), dict(group=[0, 1]), dict(group=[2], expected_groups=4096, force_hash=True)]


@pytest.mark.parametrize("family", FAMILIES)
def test_random_trees_mixing_column_atoms(cg, kernel_family, family):
    """random WHERE trees, FILTERs and bool_and / bool_or arguments mixing column atoms (int2 / int4 / int8 in any pairing,
    float8 with itself, x op x) with comparisons, IN lists and IS tests, over NULL-bearing and all-NULL chunk groups, NaN,
    +-inf and +-0.0: plain aggregate, one- and two-column direct-indexed tables and the hash table"""
    kernel_family(family)
    Col = cg.Col
    rng = np.random.default_rng(20261018)
    rel, cols, nulls, stripe_rows, chunk_rows = mixed_relation(cg, rng)
    fc = (5,)
    minmax = ref.skip_minmax(cols, nulls, stripe_rows, chunk_rows, fc)
    pools = constant_pools(minmax, [2, 4, 2, 4, 8, 8], fc)

    def atom():
        r = rng.random()
        if r < 0.45:
            if rng.random() < 0.2:
                return (5, OPS[int(rng.integers(0, 6))], Col(5))
            a, b = (int(x) for x in rng.integers(0, 5, 2))
            return (a, OPS[int(rng.integers(0, 6))], Col(b))
        c = int(rng.integers(0, 6))
        if r < 0.55:
            return (c, "is null" if rng.random() < 0.5 else "is not null")
        if r < 0.65:
            return (c, "in" if rng.random() < 0.5 else "not in", tuple(pools[c][int(rng.integers(0, len(pools[c])))] for _ in range(3)))
        return (c, OPS[int(rng.integers(0, 6))], pools[c][int(rng.integers(0, len(pools[c])))])
    before = jit_launches()
    for i in range(12):
        shape = SHAPES[i % len(SHAPES)]
        where = small_tree(rng, atom)
        aggs = [cg.count_star(), cg.sum_(4, filter=small_tree(rng, atom, 2)), cg.bool_or(small_tree(rng, atom)),
                cg.bool_and(small_tree(rng, atom, 2)), cg.count(5, filter=small_tree(rng, atom, 1))]
        try:
            cg.make_desc(where, shape["group"], aggs, float_cols=fc)
        except Exception:                                         # more than 8 pool atoms: drawn again next time
            continue
        check(cg, rel, cols, nulls, where, shape["group"], aggs, stripe_rows, chunk_rows, fc, key=("random", i),
              expected_groups=shape.get("expected_groups", 0), force_hash=shape.get("force_hash", False))
    if family in ("jit", "jit_always"):
        assert jit_launches() > before                            # the generated kernels ran
    elif family == "general":
        assert jit_launches() == before


# --------------------------------------------------------------------------- every same-class type pair
INT_LIKE = [0, 1, 2, 3, 4, 6, 7, 9]          # bool, int1, int2, int4, int8, numeric(12, 2), int8, int8 added afterwards


def typed_queries(cg):
    Col = cg.Col
    qs = []
    pairs = [(a, b) for a in INT_LIKE for b in INT_LIKE if a < b] + [(5, 5), (8, 8), (4, 4), (6, 6)]
    for i, (a, b) in enumerate(pairs):
        op = OPS[i % 6]
        aggs = [cg.count_star(), cg.count_star(filter=(b, OPS[(i + 1) % 6], Col(a))), cg.sum_(7, filter=(a, "<>", Col(b))),
                cg.bool_or((a, OPS[(i + 2) % 6], Col(b))), cg.bool_and(("or", (b, ">=", Col(a)), (a, "is null")))]
        qs.append(([(a, op, Col(b))], [], aggs))
        qs.append((("or", (a, op, Col(b)), (3, "<", 0)), [3], aggs[:3]))
    return qs


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("stage", ["shard", "pageable", "dma"])
def test_every_column_type_pair_and_staging_path(cg, oracle, kernel_family, family, stage):
    """every pair of integer-like columns (bool, int1, int2, int4, int8, numeric(12, 2) -- scale alignment by 100 --, a
    column added after writing, which is all NULL), char(1) with its high bytes against itself, float8 against itself;
    NULLs in the second half of the rows, so the NULL-free and the nullable forms both run; packing on and off"""
    kernel_family(family)
    rel, cols, nulls, n = typed_relation(cg, oracle)
    scales = {6: 2}
    for i, (where, group, aggs) in enumerate(typed_queries(cg)):
        for packing in ((True, False) if group and i % 4 == 1 else (True,)):
            check(cg, rel, cols, nulls, where, group, aggs, 4000, 1000, (8,), scales, key=("typed", i), stage=stage, packing=packing)


@pytest.mark.parametrize("family", FAMILIES)
def test_float4_float8_and_int2_int8(cg, kernel_family, family):
    """float4 against float8 (float4 widened exactly) with NaN, -NaN, +-inf and +-0.0 on both sides, equal values across the
    widths; int2 against int8 at the int2 edges; NULLs on either side"""
    kernel_family(family)
    Col = cg.Col
    rng = np.random.default_rng(44)
    n = 8000
    sp = [math.nan, -math.nan, math.inf, -math.inf, 0.0, -0.0, 1.5, -1.5]
    f4 = np.asarray(rng.choice(sp, n), np.float32)
    f8 = rng.choice(sp, n).astype(np.float64)
    f8[::7] = f4[::7]                                              # the same value at both widths
    f4 = f4.astype(np.float64)                                     # as the reference sees it: widened
    i2 = rng.integers(-2**15, 2**15, n)
    i8 = rng.integers(-2**15 - 2, 2**15 + 2, n)
    i8[::5] = i2[::5]
    g = rng.integers(0, 5, n)
    cols = [g, f4, f8, i2, i8]
    nulls = [None] + [(rng.random(n) < 0.05).astype(np.uint8) for _ in range(4)]
    for z in nulls[1:]:
        z[:2000] = 0                                               # two NULL-free chunk groups
    rel = cg.Relation.write([8, 4, 8, 2, 8], cols, nulls, type_classes=[0, 1, 1, 0, 0], stripe_row_limit=4000, chunk_row_limit=1000)
    fc = (1, 2)
    for op in OPS:
        for where in ([(1, op, Col(2))], [(2, op, Col(1))], [(3, op, Col(4))], [(4, op, Col(3))], [(1, op, Col(1))]):
            aggs = [cg.count_star(), cg.sum_(3), cg.max_(2, True), cg.bool_and((4, op, Col(3))), cg.count_star(filter=(2, op, Col(1)))]
            check(cg, rel, cols, nulls, where, [0], aggs, 4000, 1000, fc, key=("f48", op, repr(where)))


def numeric_relation(cg, oracle):
    """numeric(18, 0), numeric(18, 18) and int8 at their extremes, where scale alignment leaves 64 bits: x * 10^18 against
    y.  Values as stored: value * 10^scale"""
    rng = np.random.default_rng(18)
    n = 6000
    big = 10**18 - 1
    a = rng.integers(-big, big, n, endpoint=True)                   # numeric(18, 0)
    b = rng.integers(-big, big, n, endpoint=True)                   # numeric(18, 18): |value| < 1
    c = rng.integers(INT64_MIN, INT64_MAX, n, endpoint=True)        # int8
    edges = [(0, 0, 0), (1, big, INT64_MAX), (-1, -big, INT64_MIN), (big, big, 1), (-big, -big, -1), (0, 1, 0), (0, -1, 0),
             (1, 10**18 - 1, 1), (9, big, 9), (-9, -big, -9)]
    for i, (x, y, z) in enumerate(edges):
        a[i], b[i], c[i] = x, y, z
    a[20:40] = 0
    b[20:40] = 0
    c[40:60] = 0
    b[60:80] = rng.integers(-5, 6, 20)
    g = rng.integers(0, 4, n)
    cols = [g, a, b, c]
    nulls = [None] + [np.zeros(n, np.uint8) for _ in range(3)]
    for z in nulls[1:]:
        z[n // 2:] = rng.random(n - n // 2) < 0.1
    attlens, types = [8, -1, -1, 8], [0, NUMERIC(0), NUMERIC(18), 0]
    t = oracle.Table(attlens, types, stripe_row_limit=3000, chunk_row_limit=1000)
    t.insert(cols, nulls)
    rel = cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), attlens, types)
    return rel, cols, nulls


@pytest.mark.parametrize("family", FAMILIES)
def test_numeric_scale_alignment_beyond_64_bits(cg, oracle, kernel_family, family):
    """numeric(18, 0) against numeric(18, 18) and int8 against numeric(18, 18) at the int64 extremes: x * 10^18 is exact in
    128 bits, on either side of the operator"""
    kernel_family(family)
    Col = cg.Col
    rel, cols, nulls = numeric_relation(cg, oracle)
    scales = {1: 0, 2: 18}
    for op in OPS:
        for where in ([(1, op, Col(2))], [(2, op, Col(1))], [(3, op, Col(2))], [(2, op, Col(3))], [(3, op, Col(1))]):
            aggs = [cg.count_star(), cg.count_star(filter=(2, op, Col(3))), cg.bool_or((1, op, Col(2)))]
            check(cg, rel, cols, nulls, where, [0], aggs, 3000, 1000, (), scales, key=("numeric", op, repr(where)))


# --------------------------------------------------------------------------- TPC-H Q12's predicates
def days(y, m, d):
    return (datetime.date(y, m, d) - datetime.date(2000, 1, 1)).days


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("stage", ["shard", "pageable", "dma"])
def test_q12_predicates_over_lineitem(cg, lineitem, kernel_family, family, stage):
    """l_commitdate < l_receiptdate AND l_shipdate < l_commitdate AND l_receiptdate >= date '1994-01-01' AND l_receiptdate <
    date '1995-01-01', count(*) and sum(l_extendedprice) grouped by l_returnflag, over the 12 000-row fixture (dates as int4
    days since 2000-01-01), equal to numpy over the same rows"""
    kernel_family(family)
    Col = cg.Col
    li = lineitem
    names = ["l_returnflag", "l_extendedprice", "l_shipdate", "l_commitdate", "l_receiptdate"]
    cols = [np.asarray(li[k], np.int64) for k in names]
    rel = cg.Relation.write([1, 8, 4, 4, 4], cols, None, stripe_row_limit=6000, chunk_row_limit=1000)
    lo, hi = days(1994, 1, 1), days(1995, 1, 1)
    where = [(3, "<", Col(4)), (2, "<", Col(3)), (4, ">=", lo), (4, "<", hi)]
    before = jit_launches()
    st, got = run(cg, rel, where, [0], [cg.count_star(), cg.sum_(1)], stage=stage)
    flag, price, ship, commit, receipt = cols
    keep = (commit < receipt) & (ship < commit) & (receipt >= lo) & (receipt < hi)
    want = {(int(f),): (int((keep & (flag == f)).sum()), int(price[keep & (flag == f)].sum())) for f in np.unique(flag[keep])}
    assert {k: (v[0]["count"], v[1]["sum"]) for k, v in got.items()} == want
    assert st.rows_passed == int(keep.sum())
    assert st.rows_scanned == len(flag) - 1000 * st.chunk_groups_filtered
    if family in ("jit", "jit_always"):
        assert jit_launches() > before
    # and against the reference, counters included
    check(cg, rel, cols, None, where, [0], [cg.count_star(), cg.sum_(1)], 6000, 1000, key=("q12",), stage=stage)
