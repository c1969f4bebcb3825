"""IN / NOT IN lists and IS [NOT] NULL atoms on the host side, without a GPU: the descriptor make_desc builds (the list
table), the checks of the new fields, chunk-group skipping and cg_relation_bounds against tests/reference.py over
random trees that mix the new atoms with the comparison atoms, IN lists against their OR of equalities, the generated kernels of every kind and form, and the
generated source of the existing query shapes, which must stay byte for byte what it was."""
import ctypes as C
import hashlib
import math

import numpy as np
import pytest

import reference as ref
from test_where_reference import OPS, constant_pools, edge_relation, library_mask, random_tree


@pytest.fixture(scope="module")
def cg():
    from citus_b200 import build
    build.build()
    from citus_b200 import capi, columnar
    capi.lib()
    return columnar


def compile_check(d, cols, kmin=0, kmax=-1, rows=1 << 20, nullable=0):
    from citus_b200 import capi
    arr = (capi.CgColumnDesc * len(cols))()
    for i, (l, t) in enumerate(cols):
        arr[i].attlen, arr[i].type_class = l, t
    kind = C.c_int32(-1)
    src = C.create_string_buffer(1 << 20)
    rc = capi.lib().cg_jit_compile_check_nullable(C.byref(d), arr, len(cols), kmin, kmax, rows, nullable, C.byref(kind), src, len(src))
    return rc, kind.value, src.value.decode()


# --------------------------------------------------------------------------- descriptor and validation
def test_make_desc_fills_the_list_table(cg):
    from citus_b200 import capi
    assert (capi.CG_OP["in"], capi.CG_OP["not in"], capi.CG_OP["is null"], capi.CG_OP["is not null"]) == (6, 7, 8, 9)
    where = ("or", (0, "in", (5, 3, None, 3)), ("and", (1, "is null"), (2, "not in", (1.5, math.nan))))
    aggs = [cg.count_star(filter=(0, "in", (5, 3, None, 3))), cg.bool_or((0, "is not null")), cg.count_star(filter=(0, "not in", (7,)))]
    d = cg.make_desc(where, [], aggs, float_cols=(2,))
    atoms = [(d.quals[i].column, d.quals[i].op, d.quals[i].konst) for i in range(d.nquals)]
    assert atoms == [(0, 6, 0), (1, 8, 0), (2, 7, 1)]
    pool = [(d.filter_quals[i].column, d.filter_quals[i].op, d.filter_quals[i].konst) for i in range(d.nfilter_quals)]
    assert pool == [(0, 6, 0), (0, 9, 0), (0, 7, 2)]            # the WHERE list and the FILTER share list 0
    assert d.nin_lists == 3 and d.nin_values == 6
    lists = [(d.in_lists[i].first, d.in_lists[i].nvalues, d.in_lists[i].nnulls) for i in range(3)]
    assert lists == [(0, 3, 1), (3, 2, 0), (5, 1, 0)]
    assert list(d.in_values[:6])[:3] == [5, 3, 3]                # as written: order and duplicates kept
    assert d.in_values[3] == int(np.float64(1.5).view(np.int64))
    assert math.isnan(np.int64(d.in_values[4]).view(np.float64))
    plain = cg.make_desc([(0, "<", 3)], [], [cg.count_star()])
    assert plain.nin_lists == 0 and plain.nin_values == 0
    with pytest.raises(capi.CitusGpuError) as e:
        cg.make_desc([(0, "in", tuple(range(1025)))], [], [cg.count_star()])
    assert e.value.code == capi.CG_EUNSUPPORTED
    full = cg.make_desc([(0, "in", tuple(range(1024)) + (None, None))], [], [cg.count_star()])    # NULLs take no value slot
    assert (full.nin_values, full.in_lists[0].nvalues, full.in_lists[0].nnulls) == (1024, 1024, 2)
    assert compile_check(full, [(8, 0)])[0] == 0
    with pytest.raises(capi.CitusGpuError) as e:
        cg.make_desc([(0, "in", (i,)) for i in range(8)] + [(1, "in", (1, 2))], [], [cg.count_star()])
    assert e.value.code == capi.CG_EUNSUPPORTED
    with pytest.raises(capi.CitusGpuError) as e:
        cg.make_desc([(0, "in", ())], [], [cg.count_star()])
    assert e.value.code == capi.CG_EUNSUPPORTED


def test_malformed_lists_and_null_tests_are_einval(cg):
    from citus_b200 import capi
    cols = [(8, 0), (4, 0), (8, 1)]

    def good():
        return cg.make_desc([(0, "in", (1, 2, None)), (2, "not in", (0.5,)), (1, "is null")], [],
                            [cg.count_star(filter=(1, "in", (4,))), cg.bool_or((0, "is not null"))], float_cols=(2,))
    assert compile_check(good(), cols)[0] == 0
    cases = []
    d = good(); d.quals[0].op = 10; cases.append(d)                                  # operator out of range
    d = good(); d.quals[0].op = -1; cases.append(d)
    d = good(); d.quals[0].konst = 3; cases.append(d)                                # list index >= nin_lists
    d = good(); d.quals[0].konst = -1; cases.append(d)
    d = good(); d.filter_quals[0].konst = 3; cases.append(d)                         # ... in the pool too
    d = good(); d.nin_lists = 9; cases.append(d)                                     # counts out of range
    d = good(); d.nin_lists = -1; cases.append(d)
    d = good(); d.nin_values = 1025; cases.append(d)
    d = good(); d.nin_values = -1; cases.append(d)
    d = good(); d.in_lists[1].nvalues = 0; d.in_lists[1].nnulls = 0; cases.append(d)    # an empty list
    d = good(); d.in_lists[0].nnulls = -1; cases.append(d)                           # negative counts
    d = good(); d.in_lists[0].nvalues = -1; cases.append(d)
    d = good(); d.in_lists[0].first = -1; cases.append(d)
    d = good(); d.in_lists[2].first = 4; d.in_lists[2].nvalues = 2; cases.append(d)  # first + nvalues > nin_values
    d = good(); d.quals[2].konst = 1; cases.append(d)                                # IS NULL with a constant
    d = good(); d.filter_quals[1].konst = 7; cases.append(d)
    for i, d in enumerate(cases):
        assert compile_check(d, cols)[0] == capi.CG_EINVAL, i
    # lists of NULLs only are valid, and a zero-filled tail validates as before
    d = cg.make_desc([(0, "in", (None,)), (0, "not in", (None, None))], [], [cg.count_star()])
    assert compile_check(d, cols)[0] == 0
    d = cg.make_desc([(0, "<", 5)], [], [cg.count_star()])
    assert (d.nin_lists, d.nin_values) == (0, 0) and compile_check(d, cols)[0] == 0
    d.quals[0].op = 6                                                                # IN without any list
    assert compile_check(d, cols)[0] == capi.CG_EINVAL


def test_list_and_null_test_columns_count_toward_the_column_limit(cg):
    from citus_b200 import capi
    cols = [(8, 0)] * 10
    aggs = [cg.sum_(c) for c in range(6)]
    assert compile_check(cg.make_desc([(6, "in", (1, 2))], [], aggs), cols)[0] == 0
    d = cg.make_desc([(6, "in", (1, 2)), (7, "is null")], [], aggs)
    assert compile_check(d, cols)[0] == 0
    d = cg.make_desc([(6, "in", (1, 2)), (7, "is null")], [], aggs + [cg.count_star(filter=(8, "is not null"))])
    assert compile_check(d, cols)[0] == capi.CG_EUNSUPPORTED


# --------------------------------------------------------------------------- reference rows
def test_reference_row_semantics():
    def v(atom, x, isnull, is_float):
        return ref.atom_value(atom, [x], [isnull], (0,) if is_float else ())
    assert v((0, "in", (1, 2)), 1, False, False) is True
    assert v((0, "in", (1, 2)), 3, False, False) is False
    assert v((0, "in", (1, None)), 3, False, False) is None
    assert v((0, "in", (1, None)), 1, False, False) is True
    assert v((0, "in", (1,)), 0, True, False) is None
    assert v((0, "not in", (1, 2)), 3, False, False) is True
    assert v((0, "not in", (1, None)), 3, False, False) is None
    assert v((0, "not in", (1, None)), 1, False, False) is False
    assert v((0, "not in", (1,)), 0, True, False) is None
    assert v((0, "is null"), 0, True, False) is True and v((0, "is null"), 0, False, False) is False
    assert v((0, "is not null"), 0, True, False) is False
    assert v((0, "in", (math.nan,)), math.nan, False, True) is True
    assert v((0, "in", (-0.0,)), 0.0, False, True) is True
    assert v((0, "not in", (0.0,)), -0.0, False, True) is False



def test_in_lists_equal_their_or_of_equalities():
    """a non-empty IN list without NULL elements answers as the OR of its "=" atoms and NOT IN as the AND of its "<>" atoms, in
    WHERE, FILTER and bool_* arguments, for the rows and for the chunk mask"""
    import dataclasses
    from test_agg_filter_host import FC, map_atoms, random_language

    def expand(atom):
        if atom[1] not in ("in", "not in"):
            return atom
        return ("or" if atom[1] == "in" else "and",) + tuple((atom[0], "=" if atom[1] == "in" else "<>", e) for e in atom[2])
    rng = np.random.default_rng(20261017)
    lists = 0
    for trial in range(120):
        if trial % 40 == 0:
            cols, nulls, atom, agg = random_language(rng, forms=("const", "in", "in", "null"))
            minmax = ref.skip_minmax(cols, nulls, 120, 30, FC)

        def no_null_atom():
            while True:
                a = atom()
                if a[1] not in ("in", "not in"):
                    return a
                if any(e is not None for e in a[2]):
                    return a[:2] + (tuple(e for e in a[2] if e is not None),)
        where = random_tree(rng, no_null_atom, 4)
        aggs = [agg(int(k), random_tree(rng, no_null_atom, 3) if rng.random() < 0.5 else None) for k in rng.integers(0, 10, 3)]
        aggs = [dataclasses.replace(a, arg=random_tree(rng, no_null_atom, 3)) if a.arg is not None else a for a in aggs]
        lists += sum(a[1] in ("in", "not in") for a in ref._atoms(ref.as_tree(where)))
        ors = [dataclasses.replace(a, filter=map_atoms(a.filter, expand), arg=map_atoms(a.arg, expand)) for a in aggs]
        got = ref.aggregate(cols, nulls, where, [5], aggs, FC)
        want = ref.aggregate(cols, nulls, map_atoms(where, expand), [5], ors, FC)
        assert repr(got) == repr(want), where
        assert ref.selected_chunk_mask(cols, nulls, where, 120, 30, FC, minmax=minmax) == \
            ref.selected_chunk_mask(cols, nulls, map_atoms(where, expand), 120, 30, FC, minmax=minmax), where
    assert lists > 50

# --------------------------------------------------------------------------- chunk-group skipping and bounds
def _list_atom(rng, pools, c, minmax_vals):
    """an IN / NOT IN atom on column c: 1..130 elements (lists of exactly 100 and 101 among them) from the column's
    constant pool and its chunk min / max, with NULL elements and duplicates, unsorted"""
    pool = pools[c]
    size = int(rng.choice([1, 2, 3, 8, 99, 100, 101, 130]))
    vals = [pool[int(rng.integers(0, len(pool)))] for _ in range(size)]
    if minmax_vals and rng.random() < 0.5:
        vals[0] = minmax_vals[int(rng.integers(0, len(minmax_vals)))]
    if rng.random() < 0.2:
        vals[int(rng.integers(0, size))] = None
    if size > 1 and rng.random() < 0.3:
        vals[-1] = vals[0]
    return (c, "in" if rng.random() < 0.7 else "not in", tuple(vals))


def test_selected_chunk_mask_and_relation_bounds_against_reference(cg):
    """random trees mixing IN / NOT IN / IS [NOT] NULL with the comparison atoms over int2 / int4 / int8 / float8
    columns, NaN, +-inf and +-0.0, NULL-bearing and all-NULL chunks and a column added after the stripes were written:
    the library's mask and cg_relation_bounds' row count equal the reference's"""
    from citus_b200 import capi
    seed = 20261017
    rng = np.random.default_rng(seed)
    n, stripe_rows, chunk_rows = 12_000, 3000, 1000
    cols, nulls = edge_relation(rng, n, stripe_rows, chunk_rows)
    attlens, fc = [2, 4, 8, 8, 8, 8], (3,)
    rel = cg.Relation.write(attlens, cols, nulls, type_classes=[0, 0, 0, 1, 0, 0], stripe_row_limit=stripe_rows,
                            chunk_row_limit=chunk_rows)
    rel7 = cg.Relation.from_image(rel.pages(), rel.stripes_bytes(), rel.nodes_bytes(), attlens + [8], [0, 0, 0, 1, 0, 0, 0])
    cols7 = cols + [np.zeros(n, np.int64)]
    nulls7 = nulls + [np.ones(n, np.uint8)]
    minmax = ref.skip_minmax(cols7, nulls7, stripe_rows, chunk_rows, fc)
    pools = constant_pools(minmax, attlens + [8], fc)
    ends = [[v for stripe in minmax[c] for mm in stripe if mm for v in mm] for c in range(7)]
    # the chunks of column 4 (sorted) hold ~[-10^6, 10^6]: a list of exactly 100 / 101 values outside one chunk only
    lo4, hi4 = minmax[4][0][0]
    outside = [hi4 + 1 + i for i in range(101)]
    trees = [[(4, "in", tuple(outside[:100]))], [(4, "in", tuple(outside))], [(4, "in", tuple(outside[:99]) + (None,))],
             [(4, "not in", tuple(outside[:5]))], [(4, "is not null")], [(2, "is null")], [(6, "is null")],
             [(3, "in", (math.nan, -0.0, math.inf, -math.inf))], [(3, "in", (0.0,))], [(3, "not in", (math.nan,))]]
    trees += [[_list_atom(rng, pools, c, ends[c])] for c in range(7) for _ in range(6)]

    def atom():
        c = int(rng.integers(0, 7))
        r = rng.random()
        if r < 0.35:
            return _list_atom(rng, pools, c, ends[c])
        if r < 0.5:
            return (c, "is null" if rng.random() < 0.5 else "is not null")
        return (c, OPS[int(rng.integers(0, 6))], pools[c][int(rng.integers(0, len(pools[c])))])
    trees += [random_tree(rng, atom) for _ in range(300)]
    refuted = 0
    for where in trees:
        try:
            d = cg.make_desc(where, [], [cg.count_star()], float_cols=fc)
        except capi.CitusGpuError as e:                         # more than 8 lists or 1024 values: refused, as documented
            assert e.code == capi.CG_EUNSUPPORTED
            continue
        want = ref.selected_chunk_mask(cols7, nulls7, where, stripe_rows, chunk_rows, float_cols=fc, minmax=minmax)
        got = library_mask(cg, rel7, d)
        assert got == want, f"seed {seed} where {where}"
        refuted += ref.chunks_filtered(want)
        _, _, _, rows = cg.relation_bounds(rel7, d)
        assert rows == ref.rows_kept(want, n, stripe_rows, chunk_rows), f"seed {seed} where {where}"
        d = cg.make_desc(where, [], [cg.count_star()], float_cols=fc, qual_pushdown=False)
        assert all(all(s) for s in library_mask(cg, rel7, d))
    assert refuted > 0
    # the 100 / 101 edge, stated directly: 100 elements outside a chunk refute it, 101 (or a NULL among them) do not
    one = [cg.make_desc(t, [], [cg.count_star()]) for t in trees[:3]]
    assert not library_mask(cg, rel7, one[0])[0][0]
    assert library_mask(cg, rel7, one[1])[0][0] and library_mask(cg, rel7, one[2])[0][0]


def test_in_list_over_four_chunk_groups_restates_citus_5803(cg):
    """four chunk groups holding two values each and WHERE c IN (three values) falling in two of them: two chunk groups are
    removed by the filter, and of the rows kept only the one holding the fourth value is removed by the qual (the integer
    form of the text case citus issue 5803 adds to columnar_chunk_filtering, with the writer's smallest chunk group of 1000
    rows instead of two)"""
    c = np.concatenate([[10] + [11] * 999, [20] * 500 + [21] * 500, [30] * 500 + [31] * 500, [40] * 500 + [41] * 500]).astype(np.int64)
    rel = cg.Relation.write([8], [c], None, stripe_row_limit=4000, chunk_row_limit=1000)
    where = [(0, "in", (11, 20, 21))]
    d = cg.make_desc(where, [], [cg.count_star()])
    mask = library_mask(cg, rel, d)
    want = ref.selected_chunk_mask([c], None, where, 4000, 1000)
    assert mask == want == [[True, True, False, False]]
    assert ref.chunks_filtered(want) == 2
    res = ref.aggregate([c], None, where, [], [cg.count_star()])
    kept = ref.rows_kept(want, 4000, 4000, 1000)
    assert (kept, kept - res.rows_passed, res.rows_passed) == (2000, 1, 1999)
    assert cg.relation_bounds(rel, d)[3] == 2000


# --------------------------------------------------------------------------- generated kernels
BPCHAR1 = 3


@pytest.mark.parametrize("nullable", [0, 0b11111111])
def test_generated_kernels_compile_for_every_kind_and_form(cg, nullable):
    """the new atoms in WHERE, FILTER and a bool_or argument, on int1 / int2 / int4 / int8 / float4 / float8 / char(1) /
    numeric columns, in the plain, shared-memory and table kinds, plain and nullable"""
    cols = [(1, 0), (2, 0), (4, 0), (8, 0), (4, 1), (8, 1), (-1, BPCHAR1), (-1, 2 | (2 << 8))]
    where = ("or", (0, "in", (1, 2, None)), ("and", (5, "not in", (0.5, math.nan)), (6, "is not null")))
    aggs = [cg.count_star(filter=(3, "is null")), cg.sum_(3, filter=(1, "in", (4, 5, 6))),
            cg.bool_or(("or", (2, "not in", (7, None)), (4, "in", (1.5,)))), cg.bool_and((7, "is null")), cg.min_(5, True)]
    seen = set()
    for group, kmin, kmax in (([], 0, -1), ([1], 0, 3), ([1], 0, 100_000), ([2], 0, -1)):
        d = cg.make_desc(where, group, aggs, float_cols=(4, 5), expected_groups=1000)
        rc, kind, src = compile_check(d, cols, kmin, kmax, nullable=nullable)
        assert rc == 0, src[-3000:]
        seen.add(kind)
        assert "in_set(P.sets, P.qset[0]" in src and "in_set(P.sets, P.fset[" in src
        assert "const uint64_t *sets; KSet qset[8]; KSet fset[8]; };" in src
        for v in ("1, 2", "0.5", "4, 5, 6"):                     # values never appear in the source
            assert "{" + v not in src
        if nullable:
            assert "!z3" not in src.split("const bool u0 = ")[1].split(";")[0]      # IS NULL is z3, not "!z3 && ..."
    assert seen == {0, 1, 2}


def test_null_tests_are_constants_in_the_plain_form(cg):
    cols = [(8, 0), (8, 0)]
    d = cg.make_desc([(0, "is not null")], [], [cg.count_star(filter=(1, "is null")), cg.bool_or((1, "is not null"))])
    rc, _, src = compile_check(d, cols)
    assert rc == 0
    assert "const bool t0 = true;" in src and "const bool u0 = false;" in src and "const bool u1 = true;" in src
    assert "in_set" not in src and "KSet" not in src                # no list: the struct is restated as before
    rc, _, src = compile_check(d, cols, nullable=0b11)
    assert rc == 0 and "const bool t0 = !z0;" in src and "const bool u0 = z1;" in src
    assert "const bool uf1 = !u1;" in src                          # never UNKNOWN: FALSE is "not TRUE"


def test_the_same_shape_with_other_lists_generates_the_same_source(cg):
    cols = [(8, 0), (4, 1)]
    srcs = set()
    for vals in ((1,), (5, 9, 3), tuple(range(1000)), (None, 4)):
        d = cg.make_desc([(0, "in", vals), (1, "not in", (2.5,))], [], [cg.count_star(filter=(0, "not in", vals))], float_cols=(1,))
        rc, _, src = compile_check(d, cols)
        assert rc == 0
        srcs.add(src)
    assert len(srcs) == 1


# the generated source of existing query shapes, SHA-256 taken at the commit before list and NULL-test atoms existed
PINNED = {
    "q6": "203d1097baf8fc3b30dd6902d097fc2adc097f6aaf1f1960d68c270425969637",
    "q1": "c21b7f19155287fe08b871ac3881845ada184f3dfc9dd7f1b682d7bad041405a",
    "c2": "3913a5150235f6b947dfdf362e9826500462076ee82b1d4c6547a1c79c9f0261",
    "c2_null": "c533e601d3d99ef10f4dc839dd8c5293fde384470662a81b372f89b912164b26",
    "c2_hash": "e78bc7200241a2242aaff7cf3e34ee1efaa5d1493d84bf03530baac482731fc0",
}


def existing_shapes(cg):
    """TPC-H Q6 and Q1 on the synthetic lineitem, C2 (plain and with NULLs in the summed column) and C2 on a hash table"""
    lineitem = [(8, 0)] * 4 + [(1, 0), (1, 0), (4, 0), (4, 0)]
    c2cols = [(8, 0)] * 8
    q6 = cg.make_desc([(6, ">=", -2192), (6, "<", -1827), (2, ">=", 5), (2, "<=", 7), (0, "<", 2400)], [],
                      [cg.Agg(2, [(1, 0, 1), (2, 0, 1)], term_abs_bound=10499999 * 10)])
    q1 = cg.make_desc([(6, "<=", -486)], [4, 5],
                      [cg.Agg(2, [(0, 0, 1)], term_abs_bound=5100), cg.Agg(2, [(1, 0, 1)], term_abs_bound=10500000),
                       cg.Agg(2, [(1, 0, 1), (2, 100, -1)], term_abs_bound=10500000 * 100),
                       cg.Agg(2, [(1, 0, 1), (2, 100, -1), (3, 100, 1)], term_abs_bound=10500000 * 100 * 109),
                       cg.Agg(2, [(2, 0, 1)], term_abs_bound=11), cg.count_star()], expected_groups=16)
    c2 = cg.make_desc([(1, "<", 50)], [0], [cg.Agg(2, [(2, 0, 1)], term_abs_bound=10**9), cg.count_star()])
    c2h = cg.make_desc([(1, "<", 50)], [0], [cg.Agg(2, [(2, 0, 1)], term_abs_bound=10**9), cg.count_star()], expected_groups=1_000_000)
    return {"q6": (q6, lineitem, 0, -1, 600_000_000, 0),
            "q1": (q1, lineitem, 65 | (70 << 32), 68 | (72 << 32), 600_000_000, 0),
            "c2": (c2, c2cols, 0, 999_999, 1_000_000_000, 0),
            "c2_null": (c2, c2cols, 0, 999_999, 1_000_000_000, 0b100),
            "c2_hash": (c2h, c2cols, 0, -1, 1_000_000_000, 0)}


@pytest.mark.parametrize("name", sorted(PINNED))
def test_existing_shapes_generate_byte_identical_source(cg, name):
    d, cols, kmin, kmax, rows, nullable = existing_shapes(cg)[name]
    rc, _, src = compile_check(d, cols, kmin, kmax, rows, nullable)
    assert rc == 0
    assert hashlib.sha256(src.encode()).hexdigest() == PINNED[name]
    assert "KSet" not in src and "in_set" not in src
