"""Aggregate FILTER (WHERE ...) on the host side, without a GPU: the descriptor make_desc builds, the checks of the new
CgScanDesc fields, the generated kernels of every kind with filters, chunk-group skipping and bounds that ignore
filters, and FILTER in the exact reference against its composition from aggregates without filters."""
import ctypes as C
import dataclasses

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


# --------------------------------------------------------------------------- FILTER in the exact reference
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
    r = ref.aggregate(cols, nulls, [(0, "<", 3)], [0], aggs)
    assert set(r.groups) == {(1,), (2,)}                          # group 2 exists though every filter on y rejects it
    g1, g2 = r.groups[(1,)], r.groups[(2,)]
    assert [g1[0].count, g1[1].count, g1[2].count, g1[2].sum] == [2, 1, 1, 9]   # the NULL x of row 1 is no input of count(x)
    assert (g1[3].count, g1[3].min) == (2, 5)                     # row 1: x NULL, filter TRUE (y = 1): still no input
    assert [g2[0].count, g2[1].count, g2[2].count, g2[3].count, g2[4].count] == [0, 0, 0, 0, 2]
    assert g1[5].count == 0 and g1[5].max is None                 # a filter that matches nothing: NULL
    # a filter row that would overflow is no input: no overflow
    big = [2**62, 3, 2**62]
    r = ref.aggregate([[0, 0, 0], big], None, [], [], [A(2, [(1, 0, 1), (1, 0, 1)], filter=(1, "<", 10))])
    assert not ref.overflows(r) and r.groups[()][0].sum == 9
    r = ref.aggregate([[0, 0, 0], big], None, [], [], [A(2, [(1, 0, 1), (1, 0, 1)], filter=(1, ">", 10))])
    assert ref.overflows(r)
    # the plain aggregate over zero accepted rows keeps its group from WHERE
    r = ref.aggregate(cols, nulls, [], [], [A(0, filter=(0, ">", 9)), A(2, [(1, 0, 1)], filter=(0, ">", 9))])
    assert r.groups[()][0].count == 0 and r.groups[()][1].count == 0


ATTLENS, FC, SCALES = [2, 4, 8, 8, 8, 8], (3,), {4: 2}     # edge_relation's columns; column 4 read as numeric(p, 2)


def random_language(rng, n=300, forms=("const", "in", "null", "column")):
    """(cols, nulls, atom, agg): an edge_relation of n rows, a random atom of one of `forms` over it (edge constants of
    its chunks, IN lists with and without NULL, IS [NOT] NULL, column-to-column atoms) and agg(kind, filter), a random
    aggregate of that kind with that FILTER"""
    from citus_b200 import columnar
    cols, nulls = edge_relation(rng, n, 120, 30)
    pools = constant_pools(ref.skip_minmax(cols, nulls, 120, 30, FC), ATTLENS, FC)
    ints = (0, 1, 2, 4, 5)

    def pick(seq):
        return seq[int(rng.integers(0, len(seq)))]

    def atom():
        c, form = int(rng.integers(0, 6)), pick(forms)
        if form == "in":
            elems = [pick(pools[c]) for _ in range(int(rng.integers(0, 5)))] + ([None] if rng.random() < 0.3 else [])
            return (c, pick(("in", "not in")), tuple(elems))
        if form == "null":
            return (c, pick(("is null", "is not null")))
        if form == "column":
            return (c, pick(OPS), columnar.Col(3 if c == 3 else pick(ints)))
        return (c, pick(OPS), pick(pools[c]))

    def agg(kind, filter=None):
        if kind == ref.COUNT_STAR:
            return columnar.Agg(kind, filter=filter)
        if kind in (ref.BOOL_AND, ref.BOOL_OR):
            return columnar.Agg(kind, filter=filter, arg=random_tree(rng, atom, 3))
        is_float = kind in (ref.COUNT, ref.SUM, ref.MIN, ref.MAX) and rng.random() < 0.3
        col = 3 if is_float else pick(ints)
        if kind in (ref.BIT_AND, ref.BIT_OR) or rng.random() < 0.5:
            return columnar.Agg(kind, [(col, 0, 1)], is_float, filter=filter)
        return columnar.Agg(kind, [(col, int(rng.integers(-3, 4)), int(rng.integers(-2, 3)))], is_float, filter=filter)
    return cols, nulls, atom, agg


def map_atoms(tree, fn):
    """the condition as a tree with every atom replaced by fn(atom); None stays None"""
    tree = ref.as_tree(tree)
    if tree is None:
        return None
    return (tree[0],) + tuple(map_atoms(a, fn) if a[0] in ("and", "or") else fn(a) for a in tree[1:])


def test_filter_equals_its_composition_for_every_kind():
    """aggregate j with FILTER_j equals aggregate j without it over (WHERE AND FILTER_j), inside the groups of WHERE
    alone (no input where that leaves a group no row), for every kind and atom form"""
    rng = np.random.default_rng(20261016)
    for trial in range(120):
        if trial % 40 == 0:
            cols, nulls, atom, agg = random_language(rng)
        where = random_tree(rng, atom, 4) if trial % 5 else []
        group = [[], [5], [0]][trial % 3]
        aggs = [agg(int(k), random_tree(rng, atom, 3) if rng.random() < 0.7 else None) for k in rng.integers(0, 10, 4)]
        plain = [dataclasses.replace(a, filter=None) for a in aggs]
        got = ref.aggregate(cols, nulls, where, group, aggs, FC, SCALES)
        want = ref.aggregate(cols, nulls, where, group, plain, FC, SCALES)
        w = ref.as_tree(where)
        for j, a in enumerate(aggs):
            if a.filter is None:
                continue
            f = ref.as_tree(a.filter)
            sub = ref.aggregate(cols, nulls, ("and", w, f) if w else f, group, [plain[j]], FC, SCALES)
            for key, per in want.groups.items():
                per[j] = sub.groups[key][0] if key in sub.groups else ref.AggResult()
        assert repr(got) == repr(want), (where, group, aggs)
