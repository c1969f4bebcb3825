"""bit_and / bit_or / bool_and / bool_or on the host side, without a GPU: the descriptor make_desc builds (one atom pool
shared by FILTERs and predicate arguments), the checks of the new fields and kinds, the generated kernels of every
kind, chunk-group skipping and bounds that ignore argument atoms, and the reference against the bool_agg goldens.
(The accumulator layout and the ahead-of-time kernel's refusal need a partial on the GPU: test_gpu_bool_bit_agg.)"""
import json
import os

import numpy as np
import pytest

import reference as ref
from test_agg_filter_host import compile_check
from test_where_reference import constant_pools, edge_relation, random_tree

OPS = ("<", "<=", "=", ">=", ">", "<>")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bool_agg.json")


@pytest.fixture(scope="module")
def cg():
    from citus_b200 import build
    build.build()
    from citus_b200 import capi, columnar
    capi.lib()
    return columnar


# --------------------------------------------------------------------------- descriptor
def test_make_desc_shares_one_pool_between_filters_and_arguments(cg):
    from citus_b200 import capi
    P = ("or", (1, ">", 2), (0, "<", 2))
    aggs = [cg.bool_or(P), cg.bool_and((1, "<", 3), filter=(1, ">", 2)), cg.count_star(filter=(0, "<", 2)), cg.bit_and(1, filter=(3, "=", 1)),
            cg.bool_and((3, "=", 1)), cg.bit_or(1)]
    d = cg.make_desc([], [2], aggs)
    atoms = [(d.filter_quals[i].column, d.filter_quals[i].op, d.filter_quals[i].konst) for i in range(d.nfilter_quals)]
    assert atoms == [(1, capi.CG_OP[">"], 2), (0, capi.CG_OP["<"], 2), (1, capi.CG_OP["<"], 3), (3, capi.CG_OP["="], 1)]
    args = [[d.arg_expr[a][i] for i in range(d.narg_expr[a])] for a in range(6)]
    filt = [[d.filter_expr[a][i] for i in range(d.nfilter_expr[a])] for a in range(6)]
    assert args == [[0, 1, capi.CG_QX_OR], [2], [], [], [3], []]
    assert filt == [[], [0], [1], [3], [], []]                     # the same atom is one pool entry for FILTER and argument
    assert [d.aggs[a].kind for a in range(6)] == [capi.CG_AGG_BOOL_OR, capi.CG_AGG_BOOL_AND, 0, capi.CG_AGG_BIT_AND,
                                                  capi.CG_AGG_BOOL_AND, capi.CG_AGG_BIT_OR]
    assert [d.aggs[a].nfactors for a in range(6)] == [0, 0, 0, 1, 0, 1]
    assert (capi.CG_AGG_BIT_AND, capi.CG_AGG_BIT_OR, capi.CG_AGG_BOOL_AND, capi.CG_AGG_BOOL_OR) == (5, 6, 7, 8)
    assert (capi.CG_WORD_AND, capi.CG_WORD_OR) == (6, 7)
    plain = cg.make_desc([], [0], [cg.count_star(), cg.bit_or(1)])
    assert plain.nfilter_quals == 0 and list(plain.narg_expr) == [0] * 8
    with pytest.raises(capi.CitusGpuError) as e:                   # 9 atoms: the pool overflows
        cg.make_desc([], [], [cg.bool_and([(0, ">", i) for i in range(5)]), cg.bool_or([(1, ">", i) for i in range(4)])])
    assert e.value.code == capi.CG_EUNSUPPORTED
    with pytest.raises(capi.CitusGpuError) as e:                   # 17 tokens: the tree overflows
        cg.make_desc([], [], [cg.bool_and(("or",) + tuple([(0, ">", i % 3) for i in range(9)]))])
    assert e.value.code == capi.CG_EUNSUPPORTED


def test_malformed_bit_and_bool_aggregates_are_einval(cg):
    from citus_b200 import capi
    cols = [(8, 0), (4, 0), (8, 1), (-1, 2 | (2 << 8)), (-1, 3), (2, 0)]
    good = lambda: cg.make_desc([], [0], [cg.count_star(), cg.bool_or(("or", (1, ">", 0), (5, "<", 5))), cg.bit_and(1), cg.bit_or(5)],
                                float_cols=(2,))
    assert compile_check(cg, good(), cols, 0, 9, 1000)[0] == 0
    cases = []
    d = good(); d.aggs[2].a[0] = 1; cases.append(d)                                 # bit over an expression
    d = good(); d.aggs[2].b[0] = 2; cases.append(d)
    d = good(); d.aggs[2].nfactors = 2; d.aggs[2].column[1] = 1; d.aggs[2].b[1] = 1; cases.append(d)
    d = good(); d.aggs[2].column[0] = 2; d.aggs[2].is_float = 1; cases.append(d)    # float
    d = good(); d.aggs[2].column[0] = 2; cases.append(d)
    d = good(); d.aggs[2].column[0] = 3; cases.append(d)                            # numeric
    d = good(); d.aggs[3].column[0] = 4; cases.append(d)                            # char(1)
    d = good(); d.aggs[1].nfactors = 1; d.aggs[1].column[0] = 1; d.aggs[1].b[0] = 1; cases.append(d)   # bool with factors
    d = good(); d.narg_expr[1] = 0; cases.append(d)                                 # bool without a predicate
    d = good(); d.narg_expr[1] = 17; cases.append(d)
    d = good(); d.narg_expr[1] = -1; cases.append(d)
    d = good(); d.arg_expr[1][2] = capi.CG_QX_AND; d.arg_expr[1][1] = capi.CG_QX_OR; cases.append(d)  # operator without operands
    d = good(); d.narg_expr[1] = 2; cases.append(d)                                 # two values left
    d = good(); d.arg_expr[1][0] = 2; cases.append(d)                               # atom index >= nfilter_quals
    d = good(); d.arg_expr[1][0] = -7; cases.append(d)                              # bad token
    d = good(); d.narg_expr[2] = 1; cases.append(d)                                 # argument tree on bit_and
    d = good(); d.narg_expr[0] = 1; cases.append(d)                                 # ... on count(*)
    d = good(); d.narg_expr[6] = 1; cases.append(d)                                 # ... on a missing aggregate
    for a in (1, 2, 3):
        d = good(); d.aggs[a].term_abs_bound = 100; cases.append(d)                 # a bound on a new kind
    d = good(); d.aggs[1].kind = 9; cases.append(d)
    for i, d in enumerate(cases):
        assert compile_check(cg, d, cols, 0, 9, 1000)[0] == capi.CG_EINVAL, i


def test_argument_columns_count_toward_the_column_limit(cg):
    from citus_b200 import capi
    cols = [(8, 0)] * 9
    aggs = [cg.sum_(c) for c in range(1, 8)]
    assert compile_check(cg, cg.make_desc([], [0], aggs), cols, 0, 9, 1000)[0] == 0
    assert compile_check(cg, cg.make_desc([], [0], aggs + [cg.bool_and((7, ">", 0))]), cols, 0, 9, 1000)[0] == 0
    aggs.append(cg.bool_and((8, ">", 0)))
    assert compile_check(cg, cg.make_desc([], [0], aggs), cols, 0, 9, 1000)[0] == capi.CG_EUNSUPPORTED


def word_ops(src):
    """which AND / OR reductions on accumulator words the generated code issues (the prelude's error-flag atomicOr on
    the counters is not one)"""
    return {k: (k + "((unsigned long long *) (" if k.startswith("atomic") else k) in src
            for k in ("atomicAnd", "atomicOr", "__reduce_and_sync", "__reduce_or_sync")}


# --------------------------------------------------------------------------- generated kernels
@pytest.mark.parametrize("nullable", [0, 0b111111])
@pytest.mark.parametrize("new", ["bit_and", "bit_or", "bool_and", "bool_or"])
def test_generated_kernels_compile_for_every_kind(cg, nullable, new):
    """GLOBAL (redux.sync), SMALL (AND / OR cells and the bool no-input cells), TABLE (dense with the packed word, and
    hash: native 64-bit atomicAnd / atomicOr) with each new aggregate next to count(*), a bounded sum and a filtered
    one, plain and nullable forms"""
    cols = [(2, 0), (4, 0), (8, 0), (8, 1), (1, 0), (8, 0)]
    P = ("or", ("and", (2, ">", 5), (3, "<", 1.5)), (4, "=", 1))
    mk = {"bit_and": lambda f=None: cg.bit_and(1, filter=f), "bit_or": lambda f=None: cg.bit_or(2, filter=f),
          "bool_and": lambda f=None: cg.bool_and(P, filter=f), "bool_or": lambda f=None: cg.bool_or((3, ">=", 0.0), filter=f)}[new]
    aggs = [cg.count_star(), cg.sum_(5), mk(), mk((0, "<>", 3))]
    aggs[1].term_abs_bound = 1000
    seen = set()
    for group, kmin, kmax, want_kind in (([], 0, -1, 0), ([0], 0, 3, 1), ([0], 0, 20_000, 2), ([5], 0, -1, 2)):
        d = cg.make_desc([(1, ">", -100)], group, aggs, float_cols=(3,), expected_groups=100)
        rc, kind, src = compile_check(cg, d, cols, kmin, kmax, 1 << 20, nullable)
        assert rc == 0, src[-3000:]
        assert kind == want_kind
        seen.add(kind)
        ops = word_ops(src)
        want_and = new in ("bit_and", "bool_and")
        if kind == 0:
            assert ops["__reduce_and_sync"] == want_and and ops["__reduce_or_sync"] == (not want_and)
        else:
            assert ops["atomicAnd"] == want_and and ops["atomicOr"] == (not want_and)
        if new.startswith("bool"):
            assert "const bool at2 = " in src and "const bool af2 = " in src
            if kind == 1:
                assert "(uint64_t) an2" in src                      # the no-input counter is a shared-memory cell
    assert seen == {0, 1, 2}


def test_existing_shapes_generate_no_new_reductions(cg):
    """Q1 / Q6 / C2 shapes: no AND / OR code, no argument rails, the prelude without the argument fields"""
    lin = [(8, 0)] * 4 + [(1, 0), (1, 0), (4, 0), (4, 0)]
    q1 = [cg.sum_(0), cg.sum_(1), cg.Agg(2, [(1, 0, 1), (2, 100, -1)]), cg.Agg(2, [(1, 0, 1), (2, 100, -1), (3, 100, 1)]), cg.sum_(2),
          cg.count_star()]
    shapes = [(cg.make_desc([(6, "<=", -486)], [4, 5], q1), lin, 65 | (70 << 32), 68 | (72 << 32), 0),
              (cg.make_desc([(6, ">=", -2192), (6, "<", -1827), (2, ">=", 5), (2, "<=", 7), (0, "<", 2400)], [], [cg.Agg(2, [(1, 0, 1), (2, 0, 1)])]),
               lin, 0, -1, 0),
              (cg.make_desc([(1, "<", 50)], [0], [cg.sum_(2), cg.count_star()]), [(8, 0)] * 8, 0, 999_999, 0),
              (cg.make_desc([(1, "<", 50)], [0], [cg.sum_(2), cg.count_star()]), [(8, 0)] * 8, 0, 999_999, 0b100)]
    for d, cols, kmin, kmax, nullable in shapes:
        rc, _, src = compile_check(cg, d, cols, kmin, kmax, 1 << 24, nullable)
        assert rc == 0
        assert not any(word_ops(src).values())
        assert "nargexpr" not in src and "barg" not in src and "const bool at" not in src


# --------------------------------------------------------------------------- chunk skipping and bounds ignore arguments
def test_chunk_mask_and_bounds_ignore_argument_atoms(cg):
    from test_where_reference import library_mask
    rng = np.random.default_rng(20261018)
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
        plain = cg.make_desc(where, [5], [cg.sum_(4), cg.count_star(), cg.bit_or(2)], float_cols=fc)
        args = [cg.sum_(4), cg.count_star(), cg.bit_or(2, filter=random_tree(rng, atom, 2)), cg.bool_and(random_tree(rng, atom, 3)),
                cg.bool_or(random_tree(rng, atom, 3))]
        d = cg.make_desc(where, [5], args, float_cols=fc)
        assert d.nfilter_quals > 0 and d.narg_expr[3] > 0
        assert library_mask(cg, rel, d) == library_mask(cg, rel, plain)
        b, bp = cg.relation_bounds(rel, d), cg.relation_bounds(rel, plain)
        assert (b[0], b[1], b[3]) == (bp[0], bp[1], bp[3]) and b[2][:2] == bp[2][:2] and b[2][2:] == [0, 0, 0]


# --------------------------------------------------------------------------- the reference against bool_agg.out
class A:
    def __init__(self, kind, factors=(), arg=None, filter=None):
        self.kind, self.factors, self.is_float, self.arg, self.filter = kind, list(factors), False, arg, filter


def bool_agg_case():
    """bool_test(id, val, flag, kind) as columns: flag is 0 / 1"""
    g = json.load(open(GOLDEN))
    rows = g["rows"]
    cols = [[r[0] for r in rows], [r[1] for r in rows], [int(r[2]) for r in rows], [r[3] for r in rows]]
    return g, cols


def bool_agg_queries():
    """the six bool_agg.out queries: (WHERE, GROUP BY, aggregates); every(p) is bool_and(p)"""
    ID, VAL, FLAG, KIND = range(4)
    flag = (FLAG, "=", 1)
    three = [A(ref.BOOL_AND, arg=flag), A(ref.BOOL_OR, arg=flag), A(ref.BOOL_AND, arg=flag)]
    expr = [A(ref.BOOL_OR, arg=("or", (VAL, ">", 2), (ID, "<", 2))), A(ref.BOOL_AND, arg=(VAL, "<", 3))]
    bits = [A(ref.BIT_AND, [(VAL, 0, 1)]), A(ref.BIT_OR, [(VAL, 0, 1)])]
    return [([], [], three), ([], [KIND], three), ([], [], expr), ([], [KIND], expr), ([flag], [], bits), ([], [FLAG], bits)]


def golden_rows(result, group_cols, aggs):
    """a reference Result as psql prints the query: [key..., value...] per group, "t" / "f" for bool, flag keys as bool"""
    out = []
    for key, per in result.groups.items():
        cells = [("t" if k else "f") if group_cols == [2] else str(k) for k in key]
        for a, st in zip(aggs, per):
            if st.value is None:
                cells.append("")
            elif a.kind in (ref.BOOL_AND, ref.BOOL_OR):
                cells.append("t" if st.value else "f")
            else:
                cells.append(str(st.value))
        out.append(cells)
    return out


def test_reference_reproduces_the_bool_agg_goldens():
    g, cols = bool_agg_case()
    assert len(g["queries"]) == 6
    for (sql, want), (where, group, aggs) in zip(g["queries"], bool_agg_queries()):
        got = golden_rows(ref.aggregate(cols, None, where, group, aggs), group, aggs)
        assert sorted(got) == sorted(want), sql


def test_reference_three_valued_bool_aggregates_by_hand():
    # x: 5, NULL, -1, NULL; a NULL atom is UNKNOWN, (NULL > 0 OR TRUE) is TRUE, (NULL > 0 AND FALSE) is FALSE,
    # (NULL > 0 AND TRUE) is UNKNOWN: no input
    k = [1, 1, 2, 2]
    x = [5, 0, -1, 0]
    y = [0, 1, 1, 0]
    cols, nulls = [k, x, y], [None, [0, 1, 0, 1], None]
    aggs = [A(ref.BOOL_AND, arg=(1, ">", 0)), A(ref.BOOL_OR, arg=(1, ">", 0)), A(ref.BOOL_OR, arg=("or", (1, ">", 0), (2, "=", 1))),
            A(ref.BOOL_AND, arg=("and", (1, ">", 0), (2, "=", 1))), A(ref.BIT_AND, [(1, 0, 1)]), A(ref.BIT_OR, [(1, 0, 1)])]
    r = ref.aggregate(cols, nulls, [], [0], aggs)
    g1, g2 = r.groups[(1,)], r.groups[(2,)]
    assert [(s.count, s.value) for s in g1] == [(1, True), (1, True), (2, True), (1, False), (1, 5), (1, 5)]
    assert [(s.count, s.value) for s in g2] == [(1, False), (1, False), (1, True), (2, False), (1, -1), (1, -1)]
    r = ref.aggregate([[0, 0], [0, 0]], [None, [1, 1]], [], [], aggs[:2] + aggs[4:])     # every row UNKNOWN / NULL: no input
    assert all(s.count == 0 and s.value is None for s in r.groups[()])
    r = ref.aggregate([[0, 0, 0], [-2**63, -1, 2**63 - 1]], None, [], [], aggs[4:])
    assert [s.value for s in r.groups[()]] == [0, -1]
