"""Aggregate FILTER (WHERE ...) on the host side, without a GPU: the descriptor make_desc builds, the checks of the new
CgScanDesc fields, the generated kernels of every kind with filters, chunk-group skipping and bounds that ignore
filters, and the composition the GPU tests take their expected answers from."""
import ctypes as C

import numpy as np
import pytest

import reference as ref
from test_where_reference import constant_pools, edge_relation, random_tree

OPS = ("<", "<=", "=", ">=", ">", "<>")


@pytest.fixture(scope="module")
def cg():
    from citus_b200 import build
    build.build()
    from citus_b200 import capi, columnar
    capi.lib()
    return columnar


def as_tree(where):
    """a WHERE / FILTER in any accepted form -> a tree the reference evaluates (None = no condition)"""
    if isinstance(where, tuple) and where and where[0] in ("and", "or"):
        return where
    if isinstance(where, tuple):
        return ("and", where)
    return ("and",) + tuple(where) if where else None


def filtered_reference(cols, nulls, where, group_cols, aggs, float_cols=()):
    """PostgreSQL's FILTER by composition: the groups are those of WHERE alone; aggregate j of a group is the reference
    aggregate over ("and", WHERE, FILTER_j), or no input (count 0, SQL NULL) where that has no row of the group"""
    res = ref.aggregate(cols, nulls, where, group_cols, aggs, float_cols)
    w = as_tree(where)
    for j, a in enumerate(aggs):
        if getattr(a, "filter", None) is None:
            continue
        f = as_tree(a.filter)
        sub = ref.aggregate(cols, nulls, ("and", w, f) if w else f, group_cols, [a], float_cols)
        for key, per in res.groups.items():
            per[j] = sub.groups[key][0] if key in sub.groups else ref.AggResult()
    return res


def compile_check(cg, d, cols, kmin, kmax, rows, nullable=0):
    from citus_b200 import capi
    arr = (capi.CgColumnDesc * len(cols))()
    for i, (l, t) in enumerate(cols):
        arr[i].attlen, arr[i].type_class = l, t
    kind = C.c_int32(-1)
    src = C.create_string_buffer(1 << 20)
    rc = capi.lib().cg_jit_compile_check_nullable(C.byref(d), arr, len(cols), kmin, kmax, rows, nullable, C.byref(kind), src, len(src))
    return rc, kind.value, src.value.decode()


# --------------------------------------------------------------------------- descriptor
def test_make_desc_flattens_filters_into_their_own_pool(cg):
    from citus_b200 import capi
    aggs = [cg.count_star(filter=(1, ">", 5)), cg.sum_(2), cg.sum_(2, filter=("or", (1, "=", 65), (3, "<", 2.5))),
            cg.max_(3, True, filter=[(1, ">=", -3), (2, "<>", 7)])]
    d = cg.make_desc([(0, "<", 10), (0, ">", -10)], [0], aggs, float_cols=(3,))
    assert (d.nquals, d.nqual_expr) == (2, 0)                       # WHERE keeps its own atoms
    assert d.nfilter_quals == 5
    atoms = [(d.filter_quals[i].column, d.filter_quals[i].op, d.filter_quals[i].konst) for i in range(5)]
    assert atoms == [(1, capi.CG_OP[">"], 5), (1, capi.CG_OP["="], 65), (3, capi.CG_OP["<"], int(np.float64(2.5).view(np.int64))),
                     (1, capi.CG_OP[">="], -3), (2, capi.CG_OP["<>"], 7)]
    toks = [[d.filter_expr[a][i] for i in range(d.nfilter_expr[a])] for a in range(4)]
    assert toks == [[0], [], [1, 2, capi.CG_QX_OR], [3, 4, capi.CG_QX_AND]]
    plain = cg.make_desc([(0, "<", 10)], [0], [cg.count_star(), cg.sum_(2)])
    assert plain.nfilter_quals == 0 and list(plain.nfilter_expr) == [0] * 8
    with pytest.raises(capi.CitusGpuError):
        cg.make_desc([], [], [cg.count_star(filter=[(0, ">", i) for i in range(5)]), cg.count_star(filter=[(1, ">", i) for i in range(4)])])


def test_malformed_filters_are_einval(cg):
    from citus_b200 import capi
    cols = [(8, 0)] * 3
    good = lambda: cg.make_desc([], [0], [cg.count_star(), cg.sum_(1, filter=("or", (2, ">", 0), (1, "<", 5)))])
    assert compile_check(cg, good(), cols, 0, 9, 1000)[0] == 0
    cases = []
    d = good(); d.filter_expr[1][2] = capi.CG_QX_AND; d.filter_expr[1][1] = capi.CG_QX_OR; cases.append(d)   # operator without operands
    d = good(); d.nfilter_expr[1] = 2; cases.append(d)                                                       # two values left
    d = good(); d.filter_expr[1][0] = 2; cases.append(d)                                                     # atom index >= nfilter_quals
    d = good(); d.filter_expr[1][0] = -7; cases.append(d)                                                    # bad token
    d = good(); d.filter_quals[0].op = 6; cases.append(d)                                                    # bad operator
    d = good(); d.filter_quals[1].column = 3; cases.append(d)                                                # column out of range
    d = good(); d.nfilter_quals = 9; cases.append(d)
    d = good(); d.nfilter_expr[1] = 17; cases.append(d)
    d = good(); d.nfilter_expr[0] = -1; cases.append(d)
    d = good(); d.nfilter_expr[5] = 1; cases.append(d)                                                       # filter of a missing aggregate
    for d in cases:
        assert compile_check(cg, d, cols, 0, 9, 1000)[0] == capi.CG_EINVAL


def test_filter_columns_count_toward_the_column_limit(cg):
    from citus_b200 import capi
    cols = [(8, 0)] * 9
    aggs = [cg.sum_(c) for c in range(1, 8)]
    assert compile_check(cg, cg.make_desc([], [0], aggs), cols, 0, 9, 1000)[0] == 0
    aggs[0] = cg.sum_(1, filter=(8, ">", 0))
    assert compile_check(cg, cg.make_desc([], [0], aggs), cols, 0, 9, 1000)[0] == capi.CG_EUNSUPPORTED


# --------------------------------------------------------------------------- generated kernels
@pytest.mark.parametrize("nullable", [0, 0b111111])
def test_generated_kernels_with_filters_compile_for_every_kind(cg, nullable):
    """GLOBAL, SMALL (with the no-input cells), TABLE (dense with the packed word, and hash) with filtered count(*),
    count(x), integer / float sums, min / max and unbounded (overflow-checked) terms, plain and nullable forms"""
    cols = [(2, 0), (4, 0), (8, 0), (8, 1), (1, 0), (8, 0)]
    F = ("or", ("and", (2, ">", 5), (3, "<", 1.5)), (4, "=", 65))
    aggs = [cg.count_star(filter=(2, ">", 0)), cg.count_star(), cg.count(2, filter=F), cg.sum_(1, filter=(0, "<>", 3)),
            cg.sum_(3, True, filter=(3, ">=", 0.0)), cg.min_(5, filter=(1, "<", 0)), cg.Agg(2, [(2, 1, 3), (5, 0, 1)], filter=(0, ">", 1)),
            cg.max_(3, True)]
    bounded = [cg.Agg(a.kind, a.factors, a.is_float, 1000 if a.kind == 2 and not a.is_float and len(a.factors) == 1 else 0, a.filter)
               for a in aggs]
    seen = set()
    for group, kmin, kmax, want_kind in (([], 0, -1, 0), ([0], 0, 3, 1), ([0], 0, 20_000, 2), ([5], 0, -1, 2)):
        for a in (aggs, bounded):
            d = cg.make_desc([(1, ">", -100)], group, a, float_cols=(3,), expected_groups=100)
            rc, kind, src = compile_check(cg, d, cols, kmin, kmax, 1 << 20, nullable)
            assert rc == 0, src[-2000:]
            assert kind == want_kind
            assert "const bool f0 = " in src and "const bool u0 = " in src
            seen.add(kind)
            if kind == 1:
                assert "(uint64_t) an0" in src                    # the no-input counter is a shared-memory cell
    assert seen == {0, 1, 2}


def test_unfiltered_plans_generate_no_filter_code(cg):
    cols = [(8, 0)] * 4
    d = cg.make_desc([(1, ">", 0)], [0], [cg.count_star(), cg.sum_(2), cg.min_(3)])
    rc, _, src = compile_check(cg, d, cols, 0, 3, 1000)
    assert rc == 0 and "const bool u" not in src and "const bool f" not in src and "an0" not in src


# --------------------------------------------------------------------------- chunk skipping and bounds ignore filters
def test_chunk_mask_and_bounds_ignore_filters(cg):
    from test_where_reference import library_mask
    rng = np.random.default_rng(20261016)
    n, stripe_rows, chunk_rows = 12_000, 3000, 1000
    cols, nulls = edge_relation(rng, n, stripe_rows, chunk_rows)
    attlens, fc = [2, 4, 8, 8, 8, 8], (3,)
    rel = cg.Relation.write(attlens, cols, nulls, type_classes=[0, 0, 0, 1, 0, 0], stripe_row_limit=stripe_rows, chunk_row_limit=chunk_rows)
    minmax = ref.skip_minmax(cols, nulls, stripe_rows, chunk_rows, fc)
    pools = constant_pools(minmax, attlens, fc)

    def atom():
        c = int(rng.integers(0, 6))
        return (c, OPS[int(rng.integers(0, 6))], pools[c][int(rng.integers(0, len(pools[c])))])
    for _ in range(60):
        where = random_tree(rng, atom, 4)
        aggs = [cg.sum_(4), cg.count_star(), cg.max_(2)]
        plain = cg.make_desc(where, [5], aggs, float_cols=fc)
        filt = [cg.sum_(4, filter=random_tree(rng, atom, 3)), cg.count_star(filter=(4, ">", 10**7)), cg.max_(2, filter=random_tree(rng, atom, 3))]
        d = cg.make_desc(where, [5], filt, float_cols=fc)
        assert d.nfilter_quals > 0
        assert library_mask(cg, rel, d) == library_mask(cg, rel, plain)
        assert cg.relation_bounds(rel, d) == cg.relation_bounds(rel, plain)


# --------------------------------------------------------------------------- the composition the GPU tests use
def test_composition_reference_on_hand_made_tables():
    class A:
        def __init__(self, kind, factors=(), is_float=False, filter=None):
            self.kind, self.factors, self.is_float, self.filter = kind, list(factors), is_float, filter
    k = [1, 1, 1, 2, 2, 3]
    x = [5, -7, 9, 4, 4, 100]
    y = [0, 1, 1, 0, 0, 0]
    xn = [0, 1, 0, 0, 0, 0]                                      # row 1: x is NULL
    cols, nulls = [k, x, y], [None, xn, None]
    aggs = [A(0, filter=(2, "=", 1)), A(1, [(1, 0, 1)], filter=(2, "=", 1)), A(2, [(1, 0, 1)], filter=(2, "=", 1)),
            A(3, [(1, 0, 1)], filter=("or", (1, ">", 4), (2, "=", 1))), A(0), A(4, [(1, 0, 1)], filter=(1, ">", 1000))]
    r = filtered_reference(cols, nulls, [(0, "<", 3)], [0], aggs)
    assert set(r.groups) == {(1,), (2,)}                          # group 2 exists though every filter on y rejects it
    g1, g2 = r.groups[(1,)], r.groups[(2,)]
    assert [g1[0].count, g1[1].count, g1[2].count, g1[2].sum] == [2, 1, 1, 9]   # the NULL x of row 1 is no input of count(x)
    assert (g1[3].count, g1[3].min) == (2, 5)                     # row 1: x NULL, filter TRUE (y = 1): still no input
    assert [g2[0].count, g2[1].count, g2[2].count, g2[3].count, g2[4].count] == [0, 0, 0, 0, 2]
    assert g1[5].count == 0 and g1[5].max is None                 # a filter that matches nothing: NULL
    # a filter row that would overflow is no input: no overflow
    big = [2**62, 3, 2**62]
    r = filtered_reference([[0, 0, 0], big], None, [], [], [A(2, [(1, 0, 1), (1, 0, 1)], filter=(1, "<", 10))])
    assert not ref.overflows(r) and r.groups[()][0].sum == 9
    r = filtered_reference([[0, 0, 0], big], None, [], [], [A(2, [(1, 0, 1), (1, 0, 1)], filter=(1, ">", 10))])
    assert ref.overflows(r)
    # the plain aggregate over zero accepted rows keeps its group from WHERE
    r = filtered_reference(cols, nulls, [], [], [A(0, filter=(0, ">", 9)), A(2, [(1, 0, 1)], filter=(0, ">", 9))])
    assert r.groups[()][0].count == 0 and r.groups[()][1].count == 0
