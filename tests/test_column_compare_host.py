"""Column-to-column atoms (column, op, Col(other)) on the host side, without a GPU: the descriptor make_desc builds, the
checks of the comparison classes, chunk-group skipping and cg_relation_bounds against tests/reference.py
over random trees that mix column atoms with the other atoms, column atoms against a precomputed 1 / 0 / NULL column, the generated kernels of every kind and form, and the
generated source of query shapes without column atoms, which must stay byte for byte what it was."""
import ctypes as C
import hashlib
import math

import numpy as np
import pytest

import reference as ref
from test_in_null_atoms_host import PINNED, compile_check, existing_shapes
from test_variance_host import PARENT_SOURCE, existing_jit_shapes
from test_where_reference import OPS, constant_pools, edge_relation, library_mask, random_tree

BPCHAR1 = 3
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


def NUMERIC(s):
    return 2 | (s << 8)


@pytest.fixture(scope="module")
def cg():
    from citus_b200 import build
    build.build()
    from citus_b200 import capi, columnar
    capi.lib()
    return columnar


# --------------------------------------------------------------------------- descriptor and validation
def test_make_desc_writes_column_atoms(cg):
    from citus_b200 import capi
    assert [capi.CG_OP["col " + op] for op in OPS] == list(range(16, 22))
    Col = cg.Col
    assert hash(Col(3)) == hash(Col(3)) and Col(3) == Col(3) and Col(3) != 3
    where = ("or", (0, "<", Col(2)), ("and", (1, ">=", 5), (2, "<>", Col(2))))
    aggs = [cg.count_star(filter=(0, "<", Col(2))), cg.bool_and((1, "=", Col(0))), cg.count_star(filter=(0, "<", 2))]
    d = cg.make_desc(where, [], aggs)
    assert [(d.quals[i].column, d.quals[i].op, d.quals[i].konst) for i in range(d.nquals)] == [(0, 16, 2), (1, 3, 5), (2, 21, 2)]
    # the pool keeps (0, "<", Col(2)) and (0, "<", 2) apart, and reuses the first one
    assert [(d.filter_quals[i].column, d.filter_quals[i].op, d.filter_quals[i].konst) for i in range(d.nfilter_quals)] == \
        [(0, 16, 2), (1, 18, 0), (0, 0, 2)]
    assert d.nin_lists == 0


def test_bad_column_atoms_are_refused(cg):
    from citus_b200 import capi
    Col = cg.Col
    cols = [(8, 0), (4, 0), (8, 1), (4, 1), (-1, BPCHAR1), (-1, NUMERIC(2)), (1, 0), (2, 0)]
    assert compile_check(cg.make_desc([(0, "<", Col(1))], [], [cg.count_star()]), cols)[0] == 0
    # another column outside [0, natts) is CG_EINVAL, in WHERE and in the pool
    for k in (8, 9, -1, 1 << 40):
        d = cg.make_desc([(0, "<", Col(1))], [], [cg.count_star()])
        d.quals[0].konst = k
        assert compile_check(d, cols)[0] == capi.CG_EINVAL, k
        d = cg.make_desc([], [], [cg.count_star(filter=(0, "<", Col(1)))])
        d.filter_quals[0].konst = k
        assert compile_check(d, cols)[0] == capi.CG_EINVAL, k
    # the unused operators 10 .. 15 and those past the column atoms
    for op in (10, 12, 15, 22, 100, -1):
        d = cg.make_desc([(0, "<", Col(1))], [], [cg.count_star()])
        d.quals[0].op = op
        assert compile_check(d, cols)[0] == capi.CG_EINVAL, op
    # comparison classes: integer-like (int, bool, numeric) together, float together, char(1) with char(1) only
    ok = [(0, 1), (0, 5), (5, 6), (6, 7), (2, 3), (3, 3), (4, 4), (0, 0)]
    bad = [(0, 2), (1, 3), (5, 2), (3, 6), (4, 0), (4, 5), (2, 4), (6, 4)]
    for a, b in ok:
        for d in (cg.make_desc([(a, "<", Col(b))], [], [cg.count_star()]), cg.make_desc([], [], [cg.bool_or((a, "=", Col(b)))])):
            assert compile_check(d, cols)[0] == 0, (a, b)
    for a, b in bad:
        for d in (cg.make_desc([(a, "<", Col(b))], [], [cg.count_star()]), cg.make_desc([], [], [cg.bool_or((a, "=", Col(b)))])):
            assert compile_check(d, cols)[0] == capi.CG_EUNSUPPORTED, (a, b)


def test_both_columns_count_toward_the_column_limit(cg):
    from citus_b200 import capi
    Col = cg.Col
    cols = [(8, 0)] * 10
    aggs = [cg.sum_(c) for c in range(6)]
    assert compile_check(cg.make_desc([(6, "<", Col(7))], [], aggs), cols)[0] == 0            # 8 plan columns
    assert compile_check(cg.make_desc([(6, "<", Col(8))], [], aggs + [cg.count_star(filter=(7, ">", 0))]), cols)[0] == capi.CG_EUNSUPPORTED
    assert compile_check(cg.make_desc([(6, "<", Col(6)), (7, "<", Col(1))], [], aggs), cols)[0] == 0
    d = cg.make_desc([], [], aggs + [cg.count_star(filter=("or", (6, "=", Col(7)), (7, "<", Col(8))))])
    assert compile_check(d, cols)[0] == capi.CG_EUNSUPPORTED


# --------------------------------------------------------------------------- reference rows
def test_reference_row_semantics():
    from citus_b200.columnar import Col

    def v(op, x, x_null, y, y_null, is_float, sx=0, sy=0):
        return ref.atom_value((0, op, Col(1)), [x, y], [x_null, y_null], (0, 1) if is_float else (), {0: sx, 1: sy})
    assert v("<", 1, False, 2, False, False) is True and v(">=", 1, False, 2, False, False) is False
    assert v("<", 1, True, 2, False, False) is None and v("<>", 1, False, 2, True, False) is None
    assert v("=", math.nan, False, math.nan, False, True) is True
    assert v(">", math.nan, False, math.inf, False, True) is True
    assert v("=", -0.0, False, 0.0, False, True) is True
    assert v("<", INT64_MAX, False, INT64_MAX, False, False, 0, 18) is False          # INT64_MAX * 10^18 > INT64_MAX
    assert v(">", INT64_MIN, False, INT64_MIN, False, False, 18, 0) is True           # INT64_MIN > INT64_MIN * 10^18
    assert v("=", 5, False, 500, False, False, 0, 2) is True                          # 5 = 5.00



def test_column_atoms_equal_a_precomputed_column():
    """a column atom answers as "v = 1" over a column v holding the atom's three-valued result per row (1 / 0 / NULL), in
    WHERE, FILTER and bool_* arguments, integer-like sides at their numeric scales"""
    import dataclasses
    from test_agg_filter_host import FC, SCALES, map_atoms, random_language
    rng = np.random.default_rng(20261018)
    for trial in range(120):
        if trial % 40 == 0:
            cols, nulls, atom, agg = random_language(rng, forms=("const", "column", "column", "in"))
            n = len(cols[0])
            rows = [[float(c[r]) if i in FC else int(c[r]) for i, c in enumerate(cols)] for r in range(n)]
            isnull = [[bool(z[r]) if z is not None else False for z in nulls] for r in range(n)]
        virtual_cols, virtual_nulls, index = [], [], {}

        def virtual(a):
            if type(a[2] if len(a) > 2 else None).__name__ != "Col":
                return a
            if a not in index:
                v = [ref.atom_value(a, rows[r], isnull[r], FC, SCALES) for r in range(n)]
                index[a] = len(cols) + len(virtual_cols)
                virtual_cols.append([int(bool(x)) for x in v])
                virtual_nulls.append([x is None for x in v])
            return (index[a], "=", 1)
        where = random_tree(rng, atom, 4)
        aggs = [agg(int(k), random_tree(rng, atom, 3) if rng.random() < 0.5 else None) for k in rng.integers(0, 10, 3)]
        mapped = [dataclasses.replace(a, filter=map_atoms(a.filter, virtual), arg=map_atoms(a.arg, virtual)) for a in aggs]
        mapped_where = map_atoms(where, virtual)
        got = ref.aggregate(cols, nulls, where, [5], aggs, FC, SCALES)
        want = ref.aggregate(list(cols) + virtual_cols, list(nulls) + virtual_nulls, mapped_where, [5], mapped, FC, SCALES)
        assert repr(got) == repr(want), where
        assert index or trial % 40

# --------------------------------------------------------------------------- chunk-group skipping and bounds
def test_selected_chunk_mask_and_relation_bounds_against_reference(cg):
    """random trees mixing column atoms with comparisons, IN and IS atoms over int2 / int4 / int8 / float8 columns: a
    column atom refutes nothing (inside an OR it makes the OR unrefutable); the library's mask and cg_relation_bounds' row
    count equal the reference's"""
    from citus_b200 import capi
    Col = cg.Col
    seed = 20261018
    rng = np.random.default_rng(seed)
    n, stripe_rows, chunk_rows = 12_000, 3000, 1000
    cols, nulls = edge_relation(rng, n, stripe_rows, chunk_rows)
    attlens, fc = [2, 4, 8, 8, 8, 8], (3,)
    rel = cg.Relation.write(attlens, cols, nulls, type_classes=[0, 0, 0, 1, 0, 0], stripe_row_limit=stripe_rows,
                            chunk_row_limit=chunk_rows)
    minmax = ref.skip_minmax(cols, nulls, stripe_rows, chunk_rows, fc)
    pools = constant_pools(minmax, attlens, fc)
    ints = [0, 1, 2, 4, 5]

    def atom():
        r = rng.random()
        if r < 0.35:
            if rng.random() < 0.2:
                return (3, OPS[int(rng.integers(0, 6))], Col(3))
            a, b = (int(x) for x in rng.choice(ints, 2))
            return (a, OPS[int(rng.integers(0, 6))], Col(b))
        c = int(rng.integers(0, 6))
        if r < 0.45:
            return (c, "is null" if rng.random() < 0.5 else "is not null")
        if r < 0.55:
            return (c, "in", tuple(pools[c][int(rng.integers(0, len(pools[c])))] for _ in range(3)))
        return (c, OPS[int(rng.integers(0, 6))], pools[c][int(rng.integers(0, len(pools[c])))])
    trees = [[(4, "<", Col(5))], [(4, "<", 0), (4, "<", Col(5))], ("or", (4, "<", 0), (4, "<", Col(5)))]
    trees += [random_tree(rng, atom) for _ in range(300)]
    refuted = 0
    for where in trees:
        try:
            d = cg.make_desc(where, [], [cg.count_star()], float_cols=fc)
        except capi.CitusGpuError as e:
            assert e.code == capi.CG_EUNSUPPORTED
            continue
        want = ref.selected_chunk_mask(cols, nulls, where, stripe_rows, chunk_rows, float_cols=fc, minmax=minmax)
        got = library_mask(cg, rel, d)
        assert got == want, f"seed {seed} where {where}"
        refuted += ref.chunks_filtered(want)
        _, _, _, rows = cg.relation_bounds(rel, d)
        assert rows == ref.rows_kept(want, n, stripe_rows, chunk_rows), f"seed {seed} where {where}"
    assert refuted > 0
    # an AND with a refuting arm is refuted, an OR with a column-atom arm is not
    m = [library_mask(cg, rel, cg.make_desc(t, [], [cg.count_star()])) for t in trees[:3]]
    assert all(all(s) for s in m[0])
    want_and = ref.selected_chunk_mask(cols, nulls, trees[1], stripe_rows, chunk_rows, float_cols=fc, minmax=minmax)
    assert m[1] == want_and
    assert all(all(s) for s in m[2])
    # and the plain constant atom alone refutes what the AND refutes
    assert library_mask(cg, rel, cg.make_desc([(4, "<", 0)], [], [cg.count_star()])) == want_and


# --------------------------------------------------------------------------- generated kernels
@pytest.mark.parametrize("nullable", [0, 0b11111111])
def test_generated_kernels_compile_for_every_kind_and_form(cg, nullable):
    """column atoms in WHERE, FILTER and bool_and / bool_or arguments over int1 / int2 / int4 / int8 / float4 / float8 /
    char(1) / numeric columns (scale alignment on either side), with IN and IS atoms next to them, in the plain,
    shared-memory and table kinds, plain and nullable"""
    Col = cg.Col
    cols = [(1, 0), (2, 0), (4, 0), (8, 0), (4, 1), (8, 1), (-1, BPCHAR1), (-1, NUMERIC(2))]
    where = ("or", (3, "<", Col(7)), ("and", (5, ">=", Col(4)), (6, "<>", Col(6))))
    aggs = [cg.count_star(filter=(7, ">", Col(0))), cg.sum_(3, filter=("and", (1, "in", (4, 5, 6)), (2, "<=", Col(1)))),
            cg.bool_or(("or", (2, "=", Col(3)), (4, "<", Col(4)))), cg.bool_and((0, "<>", Col(1))), cg.min_(5, True),
            cg.count_star(filter=(3, "is null"))]
    seen = set()
    for group, kmin, kmax in (([], 0, -1), ([1], 0, 3), ([1], 0, 100_000), ([2], 0, -1)):
        d = cg.make_desc(where, group, aggs, float_cols=(4, 5), expected_groups=1000)
        rc, kind, src = compile_check(d, cols, kmin, kmax, nullable=nullable)
        assert rc == 0, src[-3000:]
        seen.add(kind)
        assert "cmp_scaled(v" in src and "col_code_f(v" in src
        assert "qcc" not in src and "KCmp" not in src              # the other side is written out, not read from the plan
        if nullable:
            assert "const bool uf" in src
    assert seen == {0, 1, 2}


def test_column_atom_source_shapes(cg):
    """equal scales compare the values directly; different scales multiply the side of the smaller scale; the nullable
    form tests both columns' NULL flags; a FALSE rail for bool_and arguments reads both too"""
    Col = cg.Col
    cols = [(8, 0), (4, 0), (-1, NUMERIC(2)), (-1, NUMERIC(18))]
    d = cg.make_desc([(0, "<", Col(1)), (0, ">=", Col(2)), (2, "=", Col(0)), (3, "<>", Col(2))], [], [cg.bool_and((1, "<=", Col(0)))])
    rc, _, src = compile_check(d, cols)
    assert rc == 0
    assert "const bool t0 = (v0 < v1);" in src
    plan_col = {0: 0, 1: 1, 2: 2, 3: 3}
    assert f"const bool t1 = (cmp_scaled(v{plan_col[0]}, 100ll, v{plan_col[2]}) >= 0);" in src
    assert f"const bool t2 = (0 == cmp_scaled(v{plan_col[0]}, 100ll, v{plan_col[2]}));" in src
    assert f"const bool t3 = (0 != cmp_scaled(v{plan_col[2]}, 10000000000000000ll, v{plan_col[3]}));" in src
    assert "const bool uf0 = !u0;" in src
    rc, _, src = compile_check(d, cols, nullable=0b1111)
    assert rc == 0
    assert "const bool t0 = !z0 && !z1 && (v0 < v1);" in src
    assert "const bool uf0 = !z1 && !z0 && !u0;" in src
    d = cg.make_desc([(0, "=", Col(0))], [], [cg.count_star()])
    rc, _, src = compile_check(d, cols, nullable=1)
    assert rc == 0 and "const bool t0 = !z0 && (v0 == v0);" in src


def test_the_same_shape_with_other_constants_generates_the_same_source(cg):
    Col = cg.Col
    cols = [(8, 0), (8, 0), (4, 1)]
    srcs = set()
    for k in (1, 5, -10**12):
        d = cg.make_desc([(0, "<", Col(1)), (1, ">", k)], [], [cg.count_star(filter=(2, "<", 0.5 * k))], float_cols=(2,))
        rc, _, src = compile_check(d, cols)
        assert rc == 0
        srcs.add(src)
    assert len(srcs) == 1


@pytest.mark.parametrize("name", sorted(PINNED))
def test_existing_shapes_generate_byte_identical_source(cg, name):
    d, cols, kmin, kmax, rows, nullable = existing_shapes(cg)[name]
    rc, _, src = compile_check(d, cols, kmin, kmax, rows, nullable)
    assert rc == 0
    assert hashlib.sha256(src.encode()).hexdigest() == PINNED[name]
    assert "cmp_scaled" not in src and "col_code_f" not in src


# plans with IN lists and with variance aggregates (taken at the commit before column atoms existed)
OTHER_SHAPES = ["lists_plain_0", "lists_hash_255", "lists_two_0", "filter_small_255", "composite3_255"]
VARIANCE_PINNED = {
    "variance_dense_0": (2, "ecc38051785aa91c837b1efabee73d67763fd3c37d033eca18d00261a66d2e32"),
    "variance_plain_255": (0, "a4b0462d3557a7d2495f589e75e234e2cd3b202296b55f7b3804dc90cfc1007b"),
}


@pytest.mark.parametrize("name", OTHER_SHAPES)
def test_list_and_other_shapes_generate_their_parent_source(cg, name):
    d, cols, kmin, kmax, rows, nullable = existing_jit_shapes(cg)[name]
    rc, kind, src = compile_check(d, cols, kmin, kmax, rows, nullable)
    assert rc == 0
    assert (kind, hashlib.sha256(src.encode()).hexdigest()) == tuple(PARENT_SOURCE[name])
    assert "cmp_scaled" not in src and "col_code_f" not in src


def variance_shapes(cg):
    cols = [(1, 0), (2, 0), (4, 0), (8, 0), (4, 1), (8, 1), (8, 0), (-1, NUMERIC(2))]
    aggs = [cg.count_star(), cg.variance(3), cg.variance(7, filter=(1, "in", (2, 3))), cg.sum_(2)]
    return {"variance_dense_0": (cg.make_desc([(6, "<", 100)], [1], aggs), cols, 0, 100_000, 1 << 24, 0),
            "variance_plain_255": (cg.make_desc([(0, "is not null")], [], aggs), cols, 0, -1, 1 << 24, 0xff)}


@pytest.mark.parametrize("name", sorted(VARIANCE_PINNED))
def test_variance_shapes_generate_their_parent_source(cg, name):
    d, cols, kmin, kmax, rows, nullable = variance_shapes(cg)[name]
    rc, kind, src = compile_check(d, cols, kmin, kmax, rows, nullable)
    assert rc == 0
    assert (kind, hashlib.sha256(src.encode()).hexdigest()) == VARIANCE_PINNED[name]
