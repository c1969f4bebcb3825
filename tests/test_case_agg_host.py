"""CASE aggregate arguments (columnar.Case) on the host side, without a GPU: tests/reference.py against a
row-at-a-time loop and against FILTER, the descriptor make_desc writes, every refusal of a CASE descriptor, cg_relation_bounds of CASE
aggregates against the skip lists, and the generated kernels of every kind and form with CASE arms, their source shape,
and one source for one shape whatever its constants."""
import ctypes as C
import itertools

import numpy as np
import pytest

import reference as ref
from test_in_null_atoms_host import compile_check

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
BPCHAR1 = 3


def NUMERIC(s):
    return 2 | (s << 8)


@pytest.fixture(scope="module")
def cg():
    from citus_b200 import build
    build.build()
    from citus_b200 import capi, columnar
    capi.lib()
    return columnar


# --------------------------------------------------------------------------- the reference
def test_reference_against_a_row_loop(cg):
    """random CASE sums, counts, mins and maxes with NULLs in WHEN and THEN columns against plain Python written per row"""
    Case, Const = cg.Case, cg.Const
    rng = np.random.default_rng(7)
    n = 400
    cols = [rng.integers(0, 4, n), rng.integers(-5, 6, n), rng.integers(-1000, 1000, n)]
    nulls = [None, (rng.random(n) < 0.2).astype(np.uint8), (rng.random(n) < 0.2).astype(np.uint8)]
    for trial in range(40):
        k1, k2, k3 = (int(x) for x in rng.integers(-3, 4, 3))
        els = [Const(k3), None, 2, [(2, 1, -2)]][trial % 4]
        case = Case([((1, "<", k1), 2), (("or", (1, ">", k2), (2, "is null")), Const(k3))],
                    **({} if trial % 5 == 0 else {"else_": els}))
        aggs = [cg.sum_(case), cg.count(case), cg.min_(case), cg.max_(case, filter=(0, "<>", 1))]
        got = ref.aggregate(cols, nulls, [], [0], aggs)

        def value(r):
            x1 = None if nulls[1][r] else int(cols[1][r])
            x2 = None if nulls[2][r] else int(cols[2][r])
            if x1 is not None and x1 < k1:
                return x2
            if (x1 is not None and x1 > k2) or x2 is None:
                return k3
            if trial % 5 == 0:
                return None
            return {0: k3, 1: None, 2: x2, 3: None if x2 is None else 1 - 2 * x2}[trial % 4]
        for g in range(4):
            rows = [r for r in range(n) if cols[0][r] == g]
            vals = [v for v in (value(r) for r in rows) if v is not None]
            fv = [v for v in (value(r) for r in rows if g != 1) if v is not None]
            st = got.groups[(g,)]
            assert (st[0].count, st[0].sum) == (len(vals), sum(vals))
            assert st[1].count == len(vals)
            assert st[2].min == (min(vals) if vals else None)
            assert st[3].count == len(fv) and st[3].max == (max(fv) if fv else None)


def test_reference_evaluates_only_the_chosen_arm():
    from citus_b200 import columnar as cgm
    big = [(0, 0, 2**40)]             # 2^40 * x leaves int64 for |x| >= 2^23
    case = cgm.Case([((1, "=", 1), big)], else_=cgm.Const(0))
    cols = [[2**30, 2**30], [0, 1]]
    r = ref.aggregate(cols, [None, None], [], [], [cgm.sum_(case)])
    assert r.groups[()][0].overflow
    r = ref.aggregate([cols[0][:1], cols[1][:1]], [None, None], [], [], [cgm.sum_(case)])
    assert not r.groups[()][0].overflow and r.groups[()][0].sum == 0



def test_case_without_else_equals_a_filter():
    """CASE WHEN p THEN e END (no ELSE) as the argument of count, sum, min, max and variance equals the aggregate of e
    FILTER (WHERE p): a row whose p is FALSE or UNKNOWN is no input on both sides"""
    import dataclasses
    from citus_b200.columnar import Case
    from test_agg_filter_host import FC, SCALES, random_language
    from test_where_reference import random_tree
    rng = np.random.default_rng(20261020)
    for trial in range(120):
        if trial % 40 == 0:
            cols, nulls, atom, agg = random_language(rng)
        where = random_tree(rng, atom, 3) if trial % 4 else []
        cases, filters = [], []
        for k in rng.integers(0, 5, 4):
            kind = [ref.COUNT, ref.SUM, ref.MIN, ref.MAX, ref.VARIANCE][int(k)]
            e, p = agg(kind), random_tree(rng, atom, 3)
            cases.append(dataclasses.replace(e, factors=[], case=Case([(p, e.factors)])))
            filters.append(dataclasses.replace(e, filter=p))
        got = ref.aggregate(cols, nulls, where, [5], cases, FC, SCALES)
        want = ref.aggregate(cols, nulls, where, [5], filters, FC, SCALES)
        assert repr(got) == repr(want), (where, cases)

# --------------------------------------------------------------------------- descriptor
def test_make_desc_writes_the_arms(cg):
    from citus_b200 import capi
    Case, Const = cg.Case, cg.Const
    c = Case([((0, "=", 3), [(1, 0, 1), (2, 100, -1)]), ((0, "in", (4, 5)), Const(7))], else_=None)
    aggs = [cg.sum_(c), cg.count(c), cg.sum_(Case([((0, "=", 3), 1)])), cg.count_star(filter=(0, "=", 3))]
    d = cg.make_desc([], [0], aggs)
    # one pool: (0 = 3) is shared by the CASEs and the FILTER; avg's sum and count share one arm range
    assert d.nfilter_quals == 2
    assert [(d.case_first[a], d.case_narms[a]) for a in range(4)] == [(0, 3), (0, 3), (3, 1), (0, 0)]
    assert d.ncase_arms == 4
    A = d.case_arms
    assert (A[0].nwhen, list(A[0].when[:1]), A[0].form, A[0].nfactors) == (1, [0], capi.CG_CASE_PRODUCT, 2)
    assert (list(A[0].column[:2]), list(A[0].a[:2]), list(A[0].b[:2])) == ([1, 2], [0, 100], [1, -1])
    assert (A[1].nwhen, A[1].when[0], A[1].form, A[1].a[0]) == (1, 1, capi.CG_CASE_CONST, 7)
    assert (A[2].nwhen, A[2].form) == (0, capi.CG_CASE_NULL)
    assert (A[3].nwhen, A[3].form, A[3].nfactors, A[3].column[0], A[3].a[0], A[3].b[0]) == (1, capi.CG_CASE_PRODUCT, 1, 1, 0, 1)
    assert all(d.aggs[a].nfactors == 0 for a in range(3))
    # a float CASE holds float8 bits
    d = cg.make_desc([], [], [cg.sum_(Case([((0, ">", 0), Const(1.5))], else_=[(1, 0.5, 2.0)]), is_float=True)])
    assert d.case_arms[0].a[0] == int(np.float64(1.5).view(np.int64))
    assert d.case_arms[1].b[0] == int(np.float64(2.0).view(np.int64))
    # a zero-filled tail is a query without CASE
    d = cg.make_desc([], [], [cg.sum_(1)])
    assert d.ncase_arms == 0 and list(d.case_narms) == [0] * 8


# --------------------------------------------------------------------------- refusals
COLS = [(8, 0), (8, 0), (8, 1), (-1, BPCHAR1), (4, 0), (8, 0), (8, 0), (8, 0), (8, 0)]


def _rc(d, cols=COLS):
    return compile_check(d, cols)[0]


def test_refusals(cg):
    from citus_b200 import capi
    Case, Const = cg.Case, cg.Const
    c = Case([((0, "=", 1), 1)], else_=Const(0))
    ok = cg.make_desc([], [], [cg.sum_(c)])
    assert _rc(ok) == 0

    def edited(fn, aggs=None):
        d = cg.make_desc([], [], aggs or [cg.sum_(c)])
        fn(d)
        return _rc(d)
    E, U = capi.CG_EINVAL, capi.CG_EUNSUPPORTED
    # a CASE on a kind that takes none
    for kind in (capi.CG_AGG_COUNT_STAR, capi.CG_AGG_BIT_AND, capi.CG_AGG_BIT_OR, capi.CG_AGG_BOOL_AND, capi.CG_AGG_BOOL_OR):
        assert edited(lambda d: setattr(d.aggs[0], "kind", kind)) == E, kind
    # factors next to the arms
    assert edited(lambda d: (setattr(d.aggs[0], "nfactors", 1))) == E
    # arm ranges
    assert edited(lambda d: d.case_first.__setitem__(0, 1)) == E
    assert edited(lambda d: d.case_first.__setitem__(0, -1)) == E
    assert edited(lambda d: d.case_narms.__setitem__(0, 3)) == E
    assert edited(lambda d: d.case_narms.__setitem__(0, -1)) == E
    assert edited(lambda d: setattr(d, "ncase_arms", capi.CG_MAX_CASE_ARMS + 1)) == E
    assert edited(lambda d: setattr(d, "ncase_arms", -1)) == E
    assert edited(lambda d: d.case_narms.__setitem__(1, 1)) == E                 # an aggregate that does not exist
    # the ELSE arm must be last
    d = cg.make_desc([], [], [cg.sum_(c)])
    d.case_arms[0], d.case_arms[1] = capi.CgCaseArm.from_buffer_copy(d.case_arms[1]), capi.CgCaseArm.from_buffer_copy(d.case_arms[0])
    assert _rc(d) == E
    # malformed WHEN trees and tokens outside the pool
    assert edited(lambda d: setattr(d.case_arms[0], "nwhen", 17)) == E
    assert edited(lambda d: d.case_arms[0].when.__setitem__(0, 1)) == E
    assert edited(lambda d: d.case_arms[0].when.__setitem__(0, -1)) == E
    assert edited(lambda d: d.case_arms[0].when.__setitem__(0, -3)) == E
    assert edited(lambda d: (setattr(d.case_arms[0], "nwhen", 2), d.case_arms[0].when.__setitem__(1, 0))) == E
    # result forms, factor counts and columns
    assert edited(lambda d: setattr(d.case_arms[1], "form", 3)) == E
    assert edited(lambda d: setattr(d.case_arms[0], "nfactors", 4)) == E
    assert edited(lambda d: setattr(d.case_arms[0], "nfactors", 0)) == E
    assert edited(lambda d: d.case_arms[0].column.__setitem__(0, len(COLS))) == E
    assert edited(lambda d: d.case_arms[0].column.__setitem__(0, -1)) == E
    # column types, as for a plain argument of the kind
    assert _rc(cg.make_desc([], [], [cg.sum_(Case([((0, "=", 1), 2)]))])) == E                           # float column, integer CASE
    assert _rc(cg.make_desc([], [], [cg.sum_(Case([((0, "=", 1), 1)]), is_float=True)])) == E           # integer column, float CASE
    assert _rc(cg.make_desc([], [], [cg.count(Case([((0, "=", 1), 2)]))])) == 0                          # count takes any type
    assert _rc(cg.make_desc([], [], [cg.variance(Case([((0, "=", 1), 2)]))])) == U
    assert _rc(cg.make_desc([], [], [cg.variance(Case([((0, "=", 1), 3)]))])) == E                       # char(1)
    d = cg.make_desc([], [], [cg.variance(Case([((0, "=", 1), Const(1))]))])
    d.aggs[0].is_float = 1
    assert _rc(d) == U
    # columns read only by arms are plan columns: at most 8
    arms = [((2, ">", 0.5), 1), ((3, "=", 65), 4), ((0, "=", 1), [(5, 0, 1), (6, 0, 1)]), ((0, "=", 2), [(7, 0, 1), (8, 0, 1)])]
    assert _rc(cg.make_desc([], [], [cg.sum_(Case(arms))], float_cols=(2,))) == U           # 9 plan columns
    assert _rc(cg.make_desc([], [], [cg.sum_(Case(arms[:3] + [((0, "=", 2), 7)]))], float_cols=(2,))) == 0
    # the arm atoms share the pool's limit
    with pytest.raises(capi.CitusGpuError):
        cg.make_desc([], [], [cg.sum_(Case([((0, "=", k), 1) for k in range(9)]))])


def test_too_many_arms_in_python(cg):
    from citus_b200 import capi
    Case, Const = cg.Case, cg.Const
    aggs = [cg.sum_(Case([((0, "=", k), Const(k)) for k in range(5)])), cg.min_(Case([((0, "=", k), Const(-k)) for k in range(5)])),
            cg.max_(Case([((0, "=", k), Const(2 * k)) for k in range(5)])), cg.count(Case([((0, "=", 1), Const(1)), ((0, "=", 2), 1)]))]
    with pytest.raises(capi.CitusGpuError) as e:
        cg.make_desc([], [], aggs)
    assert e.value.code == capi.CG_EINVAL


# --------------------------------------------------------------------------- bounds
def test_relation_bounds_of_case_sums_against_the_skip_lists(cg):
    """the term bound of a CASE sum is the largest over its arms: |k| for a constant, the factors' interval bound for a
    product, 0 for NULL; the WHEN atoms take no part"""
    Case, Const = cg.Case, cg.Const
    rng = np.random.default_rng(11)
    for trial in range(25):
        n = 3000
        lo, hi = sorted(int(x) for x in rng.integers(-10**6, 10**6, 2))
        cols = [rng.integers(0, 10, n), rng.integers(lo, hi + 1, n), rng.integers(-50, 50, n)]
        nulls = [None, (rng.random(n) < 0.1).astype(np.uint8), None]
        rel = cg.Relation.write([8, 8, 8], cols, nulls, stripe_row_limit=2000, chunk_row_limit=1000)
        k = int(rng.integers(-10**7, 10**7))
        a, b = (int(x) for x in rng.integers(-20, 20, 2))
        arms = [((0, "<", int(rng.integers(0, 10))), [(1, a, b)]), ((0, "=", 5), Const(k)), ((2, ">", 0), [(1, 0, 1), (2, 1, 1)])]
        case = Case(arms[:1 + trial % 3], **({"else_": None} if trial % 2 else {}))
        d = cg.make_desc([], [], [cg.sum_(case), cg.variance(case), cg.min_(case)])
        _, _, bounds, _ = cg.relation_bounds(rel, d)
        v1 = cols[1][nulls[1] == 0]
        m1 = max(abs(a + b * int(v1.min())), abs(a + b * int(v1.max())))
        m2 = max(abs(int(v1.min())), abs(int(v1.max()))) * max(abs(1 + int(cols[2].min())), abs(1 + int(cols[2].max())))
        want = max([m1, abs(k), m2][:1 + trial % 3])
        assert bounds[:3] == [max(want, 1), max(want, 1), 0], trial
    # a NULL arm alone bounds nothing away from zero
    d = cg.make_desc([], [], [cg.sum_(Case([((0, "<", 1), None)]))])
    assert cg.relation_bounds(rel, d)[2][0] == 1


# --------------------------------------------------------------------------- generated kernels
CASE_COLS = [(1, 0), (2, 0), (4, 0), (8, 0), (4, 1), (8, 1), (-1, BPCHAR1), (-1, NUMERIC(2))]


def _case_aggs(cg):
    Case, Const, Col = cg.Case, cg.Const, cg.Col
    when_in = ("and", (1, "in", (4, 5, None)), (2, "<=", Col(1)))
    when_null = ("or", (3, "is null"), (7, ">", 150))
    ic = Case([(when_in, [(3, 2, -3), (2, 1, 1)]), (when_null, Const(-9)), ((6, "=", 65), 7)], else_=Const(0))
    fc = Case([((5, ">", Col(4)), [(5, 0.5, 2.0)]), ((0, "not in", (1, 2)), 4)], else_=None)
    return [cg.sum_(ic), cg.count(ic), cg.min_(ic, filter=(0, ">", 0)), cg.max_(fc, is_float=True), cg.sum_(fc, is_float=True),
            cg.variance(Case([(when_null, 2)], else_=[(3, 1, 1)])), cg.count_star(), cg.sum_(3)]


@pytest.mark.parametrize("nullable", [0, 0b11111111])
def test_generated_kernels_compile_for_every_kind_and_form(cg, nullable):
    """CASE arms with comparison, IN, IS NULL and column atoms, constant, product and NULL results, integer and float,
    next to FILTERs and plain aggregates, in the plain, shared-memory and table kinds, plain and nullable"""
    aggs = _case_aggs(cg)
    seen = set()
    for group, kmin, kmax in (([], 0, -1), ([1], 0, 3), ([1], 0, 100_000), ([2], 0, -1)):
        d = cg.make_desc([(3, ">", -100)], group, aggs, float_cols=(4, 5), expected_groups=1000)
        rc, kind, src = compile_check(d, CASE_COLS, kmin, kmax, nullable=nullable)
        assert rc == 0, src[-3000:]
        seen.add(kind)
        assert "struct KArm" in src and "P.arms[" in src
    assert seen == {0, 1, 2}


def test_case_source_shape(cg):
    """first-TRUE selection as an if / else chain over the WHEN trees; constants read from the plan; a bare column written
    out; a product arm's NULL flag from its factor columns in the nullable form; no ELSE: NULL"""
    Case, Const = cg.Case, cg.Const
    cols = [(8, 0), (8, 0), (8, 0)]
    d = cg.make_desc([], [], [cg.sum_(Case([((0, "=", 1), 1), ((0, "=", 2), [(2, 3, 4)])], else_=Const(5)))])
    rc, _, src = compile_check(d, cols)
    assert rc == 0
    assert "bool cn0 = true;" in src and "bool ov0 = false;" in src
    # plan columns: the arms' columns first (1 -> v0, 2 -> v1), then the pool's (0 -> v2)
    assert "if (u0) { cn0 = false; it0 = v0; }" in src
    assert "else if (u1) { cn0 = false; it0 = add_ovf(P.arms[1].a[0], mul_ovf(P.arms[1].b[0], v1, ov0), ov0); }" in src
    assert "else { cn0 = false; it0 = P.arms[2].a[0]; }" in src
    assert "const bool an0 = cn0;" in src
    rc, _, src = compile_check(d, cols, nullable=0b111)
    assert rc == 0 and "{ cn0 = (z0); it0 = v0; }" in src
    d = cg.make_desc([], [], [cg.count(Case([((0, "=", 1), None), ((0, "=", 2), 1)]))])
    rc, _, src = compile_check(d, cols)
    assert rc == 0 and "if (u0) { }" in src and "else if (u1) { cn0 = false; it0 = v0; }" in src


def test_the_same_shape_with_other_constants_generates_the_same_source(cg):
    Case, Const = cg.Case, cg.Const
    cols = [(8, 0), (8, 0), (8, 1)]
    srcs = set()
    for k in (3, -7, 10**12):
        aggs = [cg.sum_(Case([((0, "<", k), [(1, k, 2 * k)]), ((0, "in", (k, k + 1)), Const(k))], else_=Const(-k))),
                cg.max_(Case([((2, ">", 0.5 * k), [(2, 0.25 * k, 3.0)])], else_=Const(1.5 * k)), is_float=True)]
        for group, kmin, kmax in (([], 0, -1), ([1], 0, 3), ([1], 0, -1)):
            d = cg.make_desc([], group, aggs, float_cols=(2,))
            rc, kind, src = compile_check(d, cols, kmin, kmax)
            assert rc == 0
            srcs.add((kind, src))
    assert len(srcs) == 3

