"""CPU checks of the arithmetic at the edges of the number types: the exact reference (tests/reference.py) itself,
the oracle against it on NaN / inf / -0.0 / overflow data, and the overflow check in the generated kernels.
No kernel is launched here."""
import ctypes as C
import math
import re
import struct

import numpy as np
import pytest

import reference as ref

NEG_NAN = struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000000))[0]     # the default NaN of inf - inf on x86 / CUDA
SUBNORMAL = 5e-324


def _agg(kind, factors, is_float=False):
    from oracle import oracle as orc
    return orc.Agg(kind, factors, is_float)


# --------------------------------------------------------------------------- the reference itself
def test_reference_float8_order_and_three_valued_where():
    assert math.copysign(1.0, NEG_NAN) < 0 and NEG_NAN != NEG_NAN
    assert ref.float8_cmp(NEG_NAN, math.inf) > 0 and ref.float8_cmp(math.nan, NEG_NAN) == 0
    assert ref.float8_cmp(-0.0, 0.0) == 0 and ref.float8_cmp(-math.inf, -1e308) < 0
    vals = [1.0, NEG_NAN, -math.inf, -0.0, SUBNORMAL]
    r = ref.aggregate([vals], None, [], [], [_agg(3, [(0, 0, 1)], True), _agg(4, [(0, 0, 1)], True)], float_cols=(0,))
    mn, mx = r.groups[()]
    assert mn.min == -math.inf and ref.isnan(mx.max)
    # FALSE OR NULL drops the row, TRUE OR NULL keeps it; an atom on NULL is not TRUE
    a, b = [1, 5, 5, 1], [0, 0, 0, 0]
    nb = [1, 1, 0, 0]
    where = ("or", (0, ">", 3), (1, "=", 0))
    r = ref.aggregate([a, b], [None, nb], where, [], [_agg(0, [])])
    assert (r.rows_passed, r.rows_removed) == (3, 1)
    assert ref.unpack_two_column_key((3 << 32) | 0xFFFFFFFB) == (-5, 3)
    assert ref.unpack_two_column_key(-1) == (-1, -1)


def test_reference_int_overflow_and_float_sum_bound():
    x = [2**40, 3, -2**62]
    r = ref.aggregate([x, x], None, [], [], [_agg(2, [(0, 0, 1), (1, 0, 1)])])
    assert r.groups[()][0].overflow and r.groups[()][0].sum == 2**80 + 9 + 2**124
    r = ref.aggregate([[2**63 - 1, -2**63]], None, [], [], [_agg(2, [(0, 0, 1)]), _agg(3, [(0, 1, -1)])])
    assert not r.groups[()][0].overflow and r.groups[()][0].sum == -1
    assert r.groups[()][1].overflow                 # 1 - (-2^63) leaves int64
    # the bound admits every summation order and rejects a wrong answer
    terms = [1e16, 1.0, -1e16, 3.0, 1e-3] * 100
    r = ref.aggregate([terms], None, [], [], [_agg(2, [(0, 0, 1)], True)], float_cols=(0,))
    st = r.groups[()][0]
    assert st.float_sum_ok(math.fsum(terms)) and st.float_sum_ok(sum(terms)) and st.float_sum_ok(sum(reversed(terms)))
    assert not st.float_sum_ok(math.fsum(terms) + 1e6)         # the bound here is 499 * 2^-53 * 2e18 ~ 1.1e5
    r = ref.aggregate([[math.inf, 1.0, -math.inf]], None, [], [], [_agg(2, [(0, 0, 1)], True)], float_cols=(0,))
    assert ref.isnan(r.groups[()][0].float_sum()) and r.groups[()][0].float_sum_ok(NEG_NAN)


# --------------------------------------------------------------------------- the oracle against the reference
def _oracle_scan(oracle, cols, attlen, atttype, nulls, where, group_cols, aggs, chunk=1000):
    t = oracle.Table(attlen, atttype, stripe_row_limit=chunk * 4, chunk_row_limit=chunk)
    t.insert(cols, nulls)
    return t.scan(where, group_cols, aggs)


def _float_data(rng, n):
    specials = np.array([math.nan, NEG_NAN, math.inf, -math.inf, -0.0, 0.0, SUBNORMAL, -SUBNORMAL, 1.5, -2.25])
    f = rng.normal(size=n) * 1e3
    pick = rng.random(n) < 0.02
    f[pick] = specials[rng.integers(0, len(specials), int(pick.sum()))]
    return f


@pytest.mark.parametrize("nan_first", [False, True])
def test_oracle_float_min_max_follow_postgres_order(oracle, nan_first):
    """min / max / sum / count of float8 and float4 columns with +NaN, -NaN, +-inf, -0.0 and subnormals, with and
    without GROUP BY, and a NaN that comes first or last in its group"""
    rng = np.random.default_rng(7)
    n = 6000
    k = rng.integers(-3, 4, n)
    f8 = _float_data(rng, n)
    f4 = _float_data(rng, n).astype(np.float32).astype(np.float64)
    f8[k == 2] = 1.0
    f8[np.flatnonzero(k == 2)[0 if nan_first else -1]] = NEG_NAN       # the only NaN of group 2
    f4[k == -3] = -7.0
    f4[np.flatnonzero(k == -3)[0 if nan_first else -1]] = math.nan
    cols = [k, f8, f4]
    nulls = [None, (rng.random(n) < 0.05).astype(np.uint8), None]
    aggs = [_agg(3, [(1, 0, 1)], True), _agg(4, [(1, 0, 1)], True), _agg(3, [(2, 0, 1)], True), _agg(4, [(2, 0, 1)], True),
            _agg(2, [(1, 0, 1)], True), _agg(1, [(1, 0, 1)]), _agg(0, [])]
    for group in ([], [0]):
        got = _oracle_scan(oracle, cols, [8, 8, 4], [0, 1, 1], nulls, [], group, aggs).groups()
        want = ref.aggregate(cols, nulls, [], group, aggs, float_cols=(1, 2)).groups
        assert len(got) == len(want)
        for key, per in want.items():
            g = got[key[0] if group else 0]
            for a, st in enumerate(per):
                assert g[a]["count"] == st.count, (key, a)
                if st.count == 0:
                    continue
                if aggs[a].kind == 3:
                    assert ref.float8_eq(g[a]["fmin"], st.min), (key, a, g[a]["fmin"], st.min)
                elif aggs[a].kind == 4:
                    assert ref.float8_eq(g[a]["fmax"], st.max), (key, a, g[a]["fmax"], st.max)
                elif aggs[a].kind == 2:
                    assert st.float_sum_ok(g[a]["fsum"]), (key, a)
    # group 2's max is NaN whichever row held it; combine keeps it too
    t = oracle.Table([8, 8, 4], [0, 1, 1], stripe_row_limit=4000, chunk_row_limit=1000)
    t.insert(cols, nulls)
    half = t.scan([(0, "<", 0)], [], aggs)
    half.combine(t.scan([(0, ">=", 0)], [], aggs))
    whole = ref.aggregate(cols, nulls, [], [], aggs, float_cols=(1, 2)).groups[()]
    g = half.groups()[0]
    assert ref.isnan(g[1]["fmax"]) and ref.float8_eq(g[0]["fmin"], whole[0].min)
    assert ref.isnan(g[3]["fmax"]) and ref.float8_eq(g[2]["fmin"], whole[2].min)


def test_oracle_float_quals_against_nan_inf_and_zero(oracle):
    rng = np.random.default_rng(3)
    n = 5000
    f = _float_data(rng, n)
    v = rng.integers(-100, 100, n)
    cols = [f, v]
    for k in (math.nan, math.inf, -math.inf, 0.0, -0.0):
        for op in ("<", "<=", "=", ">=", ">", "<>"):
            where = [(0, op, k)]
            r = _oracle_scan(oracle, cols, [8, 8], [1, 0], None, where, [], [_agg(0, []), _agg(2, [(1, 0, 1)])])
            w = ref.aggregate(cols, None, where, [], [_agg(0, [])], float_cols=(0,))
            skipped = n - r.rows_scanned                     # rows of chunk groups the skip lists refuted
            assert (r.rows_passed, r.rows_removed_by_filter + skipped) == (w.rows_passed, w.rows_removed), (op, k)
    where = ("or", (0, ">", math.inf), ("and", (0, "<", 0.0), (1, ">", 50)))
    r = _oracle_scan(oracle, cols, [8, 8], [1, 0], None, where, [], [_agg(0, [])])
    w = ref.aggregate(cols, None, where, [], [_agg(0, [])], float_cols=(0,))
    assert (r.rows_passed, r.rows_removed_by_filter + n - r.rows_scanned) == (w.rows_passed, w.rows_removed)


def test_oracle_integer_terms_exact_or_bigint_out_of_range(oracle):
    """sum / min / max of x*y and (a + b*x)*(c + d*y)*z: exact 128-bit answers while every step fits int64,
    PostgreSQL's "bigint out of range" once one step does not"""
    rng = np.random.default_rng(11)
    n = 3000
    seen = set()
    for scale in (2**31, 2**40, 2**62):
        x = rng.integers(-scale, scale, n)
        y = rng.integers(-scale, scale, n)
        z = rng.integers(-3, 4, n)
        x[:2] = [scale - 1, -scale]
        y[:2] = [scale - 1, -scale]
        for aggs in ([_agg(2, [(0, 0, 1), (1, 0, 1)]), _agg(3, [(0, 0, 1), (1, 0, 1)]), _agg(4, [(0, 0, 1), (1, 0, 1)])],
                     [_agg(2, [(0, 7, 1), (1, -5, 2), (2, 0, 1)])]):
            want = ref.aggregate([x, y, z], None, [], [], aggs)
            seen.add(ref.overflows(want))
            if ref.overflows(want):
                with pytest.raises(oracle.OracleError, match="bigint out of range"):
                    _oracle_scan(oracle, [x, y, z], [8, 8, 8], None, None, [], [], aggs)
                continue
            got = _oracle_scan(oracle, [x, y, z], [8, 8, 8], None, None, [], [], aggs).groups()[0]
            for a, st in enumerate(want.groups[()]):
                field = {2: "sum", 3: "min", 4: "max"}[aggs[a].kind]
                assert got[a][field] == getattr(st, field), (scale, a)
    assert seen == {False, True}
    # INT64_MIN / INT64_MAX as bare columns never overflow: the sum is exact in 128 bits
    x = np.array([2**63 - 1, 2**63 - 1, -2**63, 5], np.int64)
    got = _oracle_scan(oracle, [x], [8], None, None, [], [], [_agg(2, [(0, 0, 1)]), _agg(3, [(0, 0, 1)])]).groups()[0]
    assert got[0]["sum"] == int(sum(int(v) for v in x)) and got[1]["min"] == -2**63
    # the overflowing row filtered out by WHERE does not count
    x = np.array([2**40, 3, 4], np.int64)
    got = _oracle_scan(oracle, [x, x], [8, 8], None, None, [(0, "<", 100)], [], [_agg(2, [(0, 0, 1), (1, 0, 1)])]).groups()[0]
    assert got[0]["sum"] == 25


# --------------------------------------------------------------------------- the generated kernels' overflow check
@pytest.fixture(scope="module")
def cg():
    from citus_b200 import build
    build.build()
    from citus_b200 import capi, columnar
    capi.lib()
    return columnar


def _jit_source(cg, aggs, group, lens, kmin, kmax, nullable):
    from citus_b200 import capi
    d = cg.make_desc([(1, "<", 50)], group, aggs)
    cols = (capi.CgColumnDesc * len(lens))()
    for i, l in enumerate(lens):
        cols[i].attlen, cols[i].type_class = l, 0
    kind = C.c_int32(-1)
    buf = C.create_string_buffer(1 << 19)
    rc = capi.lib().cg_jit_compile_check_nullable(C.byref(d), cols, len(lens), kmin, kmax, 10**6, nullable, C.byref(kind), buf, len(buf))
    assert rc == 0, capi.lib().cg_last_error().decode()
    return kind.value, buf.value.decode()


def test_jit_checks_term_overflow_only_without_a_proven_bound(cg):
    try:
        C.CDLL("libnvrtc.so.12")
    except OSError:
        pytest.skip("libnvrtc missing")
    flag = "raise_flag(P.stats, 64ull)"
    for group, kmin, kmax in (([], 0, -1), ([0], 0, 3), ([0], 0, 50_000), ([0], 0, -1)):
        for nullable in (0, 0b1110):
            prod = cg.Agg(2, [(2, 0, 1), (3, 0, 1)])
            q1 = cg.Agg(2, [(2, 0, 1), (3, 100, -1), (1, 100, 1)])
            mm = cg.Agg(4, [(2, 0, 1), (3, 0, 1)])
            kind, src = _jit_source(cg, [prod, q1, mm, cg.sum_(2), cg.count_star()], group, [8, 8, 8, 8], kmin, kmax, nullable)
            assert flag in src and re.search(r"mul_ovf\(v\d, v\d, ov0\)", src) and "add_ovf(P.aggs[1].a[1]" in src, (group, kind)
            assert "bool ov0" in src and "bool ov1" in src and "bool ov2" in src and "bool ov3" not in src
            prod.term_abs_bound, q1.term_abs_bound = 10**12, 2 * 10**11
            kind, src = _jit_source(cg, [prod, q1, mm, cg.sum_(2), cg.count_star()], group, [8, 8, 8, 8], kmin, kmax, nullable)
            assert flag in src and "bool ov2" in src, (group, kind)                     # min / max: no bound is proven
            assert "bool ov0" not in src and "bool ov1" not in src, (group, kind)
            kind, src = _jit_source(cg, [prod, q1, cg.sum_(2), cg.count_star()], group, [8, 8, 8, 8], kmin, kmax, nullable)
            assert flag not in src and "bool ov" not in src, (group, kind)
