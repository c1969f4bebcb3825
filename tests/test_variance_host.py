"""var_pop / var_samp / stddev_pop / stddev_samp on the host side, without a GPU: cg_numeric_var_out against the independent
reference tests/reference.py (the reference's goldens and seeded states at the edges), the reference's variance state
against its sum over the same argument, the descriptor checks of
CG_AGG_VARIANCE, the generated kernels of variance plans, and the generated source of the plans without the kind, which
must stay byte for byte what the parent commit's generator emitted."""
import ctypes as C
import hashlib
import json
import os
import random

import pytest

import reference as ref

HERE = os.path.dirname(os.path.abspath(__file__))
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
FINALS = (ref.VAR_POP, ref.VAR_SAMP, ref.STDDEV_POP, ref.STDDEV_SAMP)


@pytest.fixture(scope="module")
def cg():
    from citus_b200 import build
    build.build()
    from citus_b200 import capi, columnar
    capi.lib()
    return columnar


def golden():
    with open(os.path.join(HERE, "golden", "variance.json")) as f:
        return json.load(f)


def state(values):
    """(N, sum(x), sum(x^2)) of the non-NULL values"""
    xs = [v for v in values if v is not None]
    return len(xs), sum(xs), sum(x * x for x in xs)


def compile_check(d, cols, kmin=0, kmax=-1, rows=1 << 20, nullable=0):
    from citus_b200 import capi
    arr = (capi.CgColumnDesc * len(cols))()
    for i, (l, t) in enumerate(cols):
        arr[i].attlen, arr[i].type_class = l, t
    kind = C.c_int32(-1)
    src = C.create_string_buffer(1 << 20)
    rc = capi.lib().cg_jit_compile_check_nullable(C.byref(d), arr, len(cols), kmin, kmax, rows, nullable, C.byref(kind), src, len(src))
    return rc, kind.value, src.value.decode()


# --------------------------------------------------------------------------- the final functions
def test_constants(cg):
    from citus_b200 import capi
    assert capi.CG_AGG_VARIANCE == 9
    assert (capi.CG_VAR_POP, capi.CG_VAR_SAMP, capi.CG_STDDEV_POP, capi.CG_STDDEV_SAMP) == FINALS == (0, 1, 2, 3)


def test_contestant_stddev_samp_golden(cg):
    """SELECT avg(rating), stddev_samp(rating) FROM contestant (columnar_query.out): 433.746119785032"""
    g = golden()["contestant"]
    n, s, q = state(g["rating"])
    assert ref.var_out(ref.STDDEV_SAMP, n, s, q, 0) == g["stddev_samp"] == "433.746119785032"
    assert cg.numeric_var_out(ref.STDDEV_SAMP, n, s, q, 0) == g["stddev_samp"]
    assert cg.numeric_var_out(ref.VAR_SAMP, n, s, q, 0) == ref.var_out(ref.VAR_SAMP, n, s, q, 0) == "188135.696428571429"


def test_aggdata_stddev_by_id_golden_is_null(cg):
    """select id, stddev(val) from aggdata group by id: one row per id, so N <= 1 and every stddev is NULL"""
    g = golden()["aggdata"]
    by_id = {}
    for i, _, v in g["rows"]:
        by_id.setdefault(i, []).append(v)
    assert sorted(by_id) == [i for i, _ in g["stddev_by_id"]]
    for i, want in g["stddev_by_id"]:
        assert want == ""
        n, s, q = state(by_id[i])
        assert n <= 1
        for final in (ref.STDDEV_SAMP, ref.VAR_SAMP):
            assert ref.var_out(final, n, s, q, 0) is None
            assert cg.numeric_var_out(final, n, s, q, 0) is None


def check(cg, final, n, s, q, scale):
    want = ref.var_out(final, n, s, q, scale)
    got = cg.numeric_var_out(final, n, s, q, scale)
    assert got == want, (final, n, s, q, scale)
    return got


def test_small_counts_and_constant_inputs(cg):
    for final in FINALS:
        sample = final in (ref.VAR_SAMP, ref.STDDEV_SAMP)
        assert check(cg, final, 0, 0, 0, 0) is None
        one = check(cg, final, 1, -7, 49, 0)
        assert (one is None) if sample else (one == "0")
        assert check(cg, final, 2, 3, 5, 0) is not None                  # {1, 2}
        for scale in (0, 2, 4, 18):
            for v in (0, 5, -123456789, INT64_MAX, INT64_MIN):
                n = 1000
                assert check(cg, final, n, n * v, n * v * v, scale) == "0"  # all equal: num = 0, the numeric zero


def random_states(rng, count):
    """states of real data (a few values, negative sums, every scale) and states at the edges: N near 2^62, sum(x^2) near
    2^158, huge N with a tiny variance (a large rscale)"""
    for _ in range(count):
        kind = rng.randrange(6)
        scale = rng.choice((0, 0, 2, 4, 18, rng.randrange(31)))
        if kind == 0:
            xs = [rng.randrange(-10**rng.randrange(1, 19), 10**rng.randrange(1, 19)) for _ in range(rng.randrange(1, 12))]
            yield scale, state(xs)
        elif kind == 1:
            xs = [rng.randrange(INT64_MIN, 0) for _ in range(rng.randrange(1, 6))]         # negative sum(x)
            yield scale, state(xs)
        elif kind == 2:
            n = (1 << 62) - rng.randrange(1 << 20)
            x = rng.randrange(1, 1 << 30)
            yield scale, (n, n * x - rng.randrange(3), n * x * x + rng.randrange(1 << 40))
        elif kind == 3:
            n = (1 << 32) - 1
            s = rng.randrange(-(1 << 94), 1 << 94)
            q = (1 << 158) - rng.randrange(1 << 100)
            yield scale, (n, s, max(q, (s * s) // n))
        elif kind == 4:
            n = rng.randrange(1 << 40, 1 << 62)                                    # one value differs by 1: tiny variance
            x = rng.randrange(-(1 << 20), 1 << 20)
            yield scale, (n, n * x + 1, n * x * x + 2 * x + 1)
        else:
            xs = [rng.choice((INT64_MIN, INT64_MAX, 0, 1, -1)) for _ in range(rng.randrange(1, 8))]
            yield scale, state(xs)


def test_var_out_matches_the_reference_on_seeded_states(cg):
    rng = random.Random(20261017)
    big_rscale = 0
    for scale, (n, s, q) in random_states(rng, 3000):
        for final in FINALS:
            got = check(cg, final, n, s, q, scale)
            if got and "." in got:
                big_rscale = max(big_rscale, len(got.split(".")[1]))
    assert big_rscale > 40                                                        # the tiny variances reached a large rscale


def test_var_out_errors(cg):
    from citus_b200 import capi
    q = (C.c_uint64 * 3)(1000, 0, 0)
    buf = C.create_string_buffer(64)
    isnull = C.c_int32()
    L = capi.lib()
    assert L.cg_numeric_var_out(ref.STDDEV_SAMP, 8, 0, 18755, q, 0, buf, 64, C.byref(isnull)) == 0
    # the text of a tiny variance has many fraction digits: a buffer that is too small is CG_EINVAL
    n, s, qq = (1 << 62), (1 << 62) * 5 + 1, (1 << 62) * 25 + 11
    need = len(ref.var_out(ref.VAR_POP, n, s, qq, 0)) + 1
    qs = (C.c_uint64 * 3)(qq & (2**64 - 1), qq >> 64, 0)
    small = C.create_string_buffer(need - 1)
    assert L.cg_numeric_var_out(ref.VAR_POP, n, s >> 64, s & (2**64 - 1), qs, 0, small, need - 1, C.byref(isnull)) == capi.CG_EINVAL
    exact = C.create_string_buffer(need)
    assert L.cg_numeric_var_out(ref.VAR_POP, n, s >> 64, s & (2**64 - 1), qs, 0, exact, need, C.byref(isnull)) == 0
    assert exact.value.decode() == ref.var_out(ref.VAR_POP, n, s, qq, 0)
    for final, scale, cnt in ((4, 0, 2), (-1, 0, 2), (0, 31, 2), (0, -1, 2), (0, 0, -1)):
        assert L.cg_numeric_var_out(final, cnt, 0, 0, q, scale, buf, 64, C.byref(isnull)) == capi.CG_EINVAL



def test_variance_counts_and_sums_like_sum():
    """a variance aggregate's count, sum and overflow equal those of sum over the same argument, with FILTERs and WHERE
    trees of every atom form; its sumsq is the sum of the squared inputs"""
    import dataclasses

    import numpy as np
    from test_agg_filter_host import FC, SCALES, random_language
    from test_where_reference import random_tree
    rng = np.random.default_rng(20261019)
    for trial in range(90):
        if trial % 30 == 0:
            cols, nulls, atom, agg = random_language(rng)
        where = random_tree(rng, atom, 4)
        group = [[], [5]][trial % 2]
        aggs = [agg(ref.VARIANCE, random_tree(rng, atom, 3) if rng.random() < 0.5 else None) for _ in range(3)]
        got = ref.aggregate(cols, nulls, where, group, aggs, FC, SCALES)
        want = ref.aggregate(cols, nulls, where, group, [dataclasses.replace(a, kind=ref.SUM) for a in aggs], FC, SCALES)
        assert set(got.groups) == set(want.groups)
        for key, per in got.groups.items():
            for v, s in zip(per, want.groups[key]):
                assert (v.count, v.sum, v.overflow, v.sumsq) == (s.count, s.sum, s.overflow, s.sumsq), (where, key)

# --------------------------------------------------------------------------- descriptors and generated kernels
COLS = [(1, 0), (2, 0), (4, 0), (8, 0), (4, 1), (8, 1), (-1, 3), (-1, 2 | (2 << 8))]


def test_descriptor_checks(cg):
    from citus_b200 import capi
    ok = cg.make_desc([], [], [cg.variance(3)])
    assert compile_check(ok, COLS)[0] == 0
    for c in (0, 1, 2, 7):                                                     # int1 / int2 / int4 / numeric
        assert compile_check(cg.make_desc([], [], [cg.variance(c)]), COLS)[0] == 0
    assert compile_check(cg.make_desc([], [], [cg.Agg(capi.CG_AGG_VARIANCE, [(3, 0, 1), (2, 1, 2)])]), COLS)[0] == 0
    assert compile_check(cg.make_desc([], [], [cg.Agg(capi.CG_AGG_VARIANCE, [(3, 0, 1)], term_abs_bound=1000)]), COLS)[0] == 0
    for c in (4, 5):                                                           # float4 / float8
        assert compile_check(cg.make_desc([], [], [cg.Agg(capi.CG_AGG_VARIANCE, [(c, 0, 1)], True)]), COLS)[0] == capi.CG_EUNSUPPORTED
        assert compile_check(cg.make_desc([], [], [cg.variance(c)]), COLS)[0] == capi.CG_EUNSUPPORTED
    assert compile_check(cg.make_desc([], [], [cg.variance(6)]), COLS)[0] == capi.CG_EINVAL      # char(1)
    assert compile_check(cg.make_desc([], [], [cg.Agg(capi.CG_AGG_VARIANCE, [])]), COLS)[0] == capi.CG_EINVAL
    assert compile_check(cg.make_desc([], [], [cg.Agg(10, [(3, 0, 1)])]), COLS)[0] == capi.CG_EINVAL


def test_accumulator_word_budget(cg):
    """an unbounded variance aggregate over int8 takes 7 words (two-limb sum(x), four-limb sum(x^2), NULL inputs): four
    of them and a two-limb sum fill the CG_MAX_WORDS = 32 words exactly, one more word is refused with CG_EUNSUPPORTED
    before any word is laid out"""
    from citus_b200 import capi
    assert capi.CG_MAX_WORDS == 32
    var = cg.variance(3)
    for aggs, rc in (([var] * 4, 0),                                             # 1 + 28
                     ([var] * 4 + [cg.sum_(3)], 0),                              # 1 + 28 + 3 = 32
                     ([var] * 4 + [cg.sum_(3), cg.count(3)], capi.CG_EUNSUPPORTED),
                     ([var] * 5, capi.CG_EUNSUPPORTED),                          # 36
                     ([var] * 8, capi.CG_EUNSUPPORTED),                          # 57
                     ([cg.sum_(3), var, var, var, var, var], capi.CG_EUNSUPPORTED)):
        assert compile_check(cg.make_desc([], [], aggs), COLS)[0] == rc, (len(aggs), rc)
        assert compile_check(cg.make_desc([], [1], aggs), COLS, 0, 100)[0] == rc
    # with bounds the same list is shorter: five variance aggregates of one-word sum(x) and sum(x^2) are 1 + 15 words
    bounded = [cg.Agg(capi.CG_AGG_VARIANCE, [(2, 0, 1)], term_abs_bound=1000)] * 5
    assert compile_check(cg.make_desc([], [], bounded), COLS, rows=1 << 20)[0] == 0


@pytest.mark.parametrize("nullable", [0, 0xff])
def test_generated_kernels_of_variance_plans_compile(cg, nullable):
    """the one-, two- and four-limb sum(x^2) forms (term_abs_bound, max_rows), with FILTER and WHERE, in every table kind"""
    from citus_b200 import capi
    seen = set()
    for bound, rows, words in ((1000, 1 << 20, 1), (1 << 20, 1 << 40, 2), (0, 1 << 20, 4), (1 << 40, 1 << 20, 4)):
        aggs = [cg.count_star(), cg.Agg(capi.CG_AGG_VARIANCE, [(3, 0, 1)], term_abs_bound=bound),
                cg.Agg(capi.CG_AGG_VARIANCE, [(2, 0, 1), (1, 3, 2)], filter=("or", (0, "<", 3), (5, ">", 0.5))), cg.sum_(3)]
        for group, kmin, kmax in (([], 0, -1), ([1], 0, 3), ([1], 0, 100_000), ([2], 0, -1)):
            d = cg.make_desc([(0, ">", -100)], group, aggs, float_cols=(4, 5), expected_groups=100)
            rc, kind, src = compile_check(d, COLS, kmin, kmax, rows, nullable)
            assert rc == 0, src[-3000:]
            seen.add(kind)
            assert "int8_t qlimbs; int8_t qword;" in src
            assert "__umul64hi(qa1, qa1)" in src
            if kind == 0:
                assert sum(f"g_q1_{l}" in src for l in range(4)) == words
            elif kind == 2:
                assert sum(f"red_add(e + {w}, (q" in src or f"red_add(e + {w}, ql1)" in src for w in range(32)) >= words
    assert seen == {0, 1, 2}                                                    # the plain, shared-memory and table kinds


# the generated source of plans without a variance aggregate: (kind, SHA-256) as the parent commit's generator emitted it
PARENT_SOURCE = {
    "boolbit_dense_0": (2, "b1c60e22ba82f67e48c672b46607968dcd9291d1e3525cf3e50e0755fb8bff88"),
    "boolbit_dense_255": (2, "763062ade6a7e97b714da57e76020746c517402949d1a1da989cad88d287b518"),
    "boolbit_hash_0": (2, "ea44c5380e4aa7cd60b82987af9211e0ae98ccfd4ca13f8be5868919eb12e3f3"),
    "boolbit_hash_255": (2, "a7d56e002bbfe61005fc283a2ceb189e641364e782cfd14c2a33aa0f3cda5b4b"),
    "boolbit_plain_0": (0, "a087f6fc0eefb855870d4c6a9d51ced6215f2c404c7cc113161bf92752593de6"),
    "boolbit_plain_255": (0, "18d69f6822aa1b63582b17d06f2489628423cec119c45e1b72c51d17d0303d96"),
    "boolbit_small_0": (1, "6bbdd4e6b53f47e9a051bf34940bc43f6ac390593869b523f2e028b689f02b0a"),
    "boolbit_small_255": (1, "9be0fdb5bfc13b60eac3df6c9d6c31a71802e483135817ad5084b77b6b964af0"),
    "boolbit_two_0": (2, "b8987c23d3f15dd85bcf6a2ea6fabfbf8a0601135ecbffbd9a4f4b374508a9bf"),
    "boolbit_two_255": (2, "19d1536c4b10cb26c7b5a80c44f31c782740bf7274ae17d461f0ddc21644fbc0"),
    "c2": (2, "3913a5150235f6b947dfdf362e9826500462076ee82b1d4c6547a1c79c9f0261"),
    "c2_hash": (2, "e78bc7200241a2242aaff7cf3e34ee1efaa5d1493d84bf03530baac482731fc0"),
    "c2_null": (2, "c533e601d3d99ef10f4dc839dd8c5293fde384470662a81b372f89b912164b26"),
    "composite1_0": (1, "231cf06d5b06844dfec024b38f1a944a6562f2973102a3242961f69bb18ca168"),
    "composite1_255": (1, "6bbd171f8a57b25c9bd871c4fa12f7aba99b10cb21fb3ccde971c3319e463267"),
    "composite3_0": (2, "376e21fab3a0077e4afc2ab86cafcc9e43fd7a8b0e170d6c082ba1b884c9fd6e"),
    "composite3_255": (2, "613918f69a02cb3fa828db2bc0c6f70d6225ecefdf9eff3285940086a803c1f5"),
    "filter_dense_0": (2, "13829141f20efa6da2770b60dc1b3e63754f620a5f0a466a5847271781a16ed7"),
    "filter_dense_255": (2, "76fc239ef6ff916b37b2bf95f05bc3c16229c3f2aed97137a94a0338368b44d5"),
    "filter_hash_0": (2, "1f24b4277cefbb307558347809efe25138cdaec9815b0cd6e9440af769814425"),
    "filter_hash_255": (2, "48372b31d384087db134d0f620bc24b2cf1fea1c0b8807b1023e7ef2bc2ff995"),
    "filter_plain_0": (0, "faecf66608d3b7c5898178f16d5396eb4fc6859b6c0dcf5c5d9fc82f810d8af1"),
    "filter_plain_255": (0, "2e11d28612df53e17d060c7a17833a18f78c3f12949e12cb96007ac0613e7a89"),
    "filter_small_0": (1, "3f46f210a2db7b85dcd63b192724bdf4aa80ae7dcdea7ab2b783554b0ca28da2"),
    "filter_small_255": (1, "3d77ec78d5a048af034364ac1f2fc5b128b289e8f2f23471be5c4873ef149b77"),
    "filter_two_0": (2, "4807fdba561b118342903d7b68045849722b78a732b948e95675f488e3deead3"),
    "filter_two_255": (2, "ac133f08e300b268e8fdde680413fa2aed9a0e66acf1a79cff2beaa434b0f797"),
    "lists_dense_0": (2, "30fa55102c06e474236be46a00a55216009bc4001dc8f22a96f6d19333d898ea"),
    "lists_dense_255": (2, "85b1befe98d38a566a4d4c715c17674559779646c77e78de1af6b73f00f770d0"),
    "lists_hash_0": (2, "0b551bc1d073b4dea249bc4ff9c7611b5e0e52a3bfb93a2c94aa799a7085d778"),
    "lists_hash_255": (2, "86a82ba10d1e0e7598e00f09861328dfbd67505e7fde80fa7129292dbd2cc0aa"),
    "lists_plain_0": (0, "514f47a46447596fe6563dc72702212b21547f3ba7412adf4a8c1b6375f1cdf5"),
    "lists_plain_255": (0, "7f208147fda1b972b7654219fe66d1b3e773805280e368c47e0b02fcb1238481"),
    "lists_small_0": (1, "d5c7b66ec8b7baaa8e9bcd0d948a3c8deda734b53266b6aba62e59211adf34f4"),
    "lists_small_255": (1, "fa9fc4d537c92ecbb0a170223d0a46085aa02ac1e81c1d2a21483f282cc0ac74"),
    "lists_two_0": (2, "e6cee6c69081bb952c2446f84824e28c87a7fa8fa764d9d45937e283a9cea3d8"),
    "lists_two_255": (2, "4691a5c9b64890552f9e8aa1eb4b8d39bf17d38c0f3466658d85a4602d8434df"),
    "minmax_dense_0": (2, "14f7339d3378bef309e2fe2aeb7f539f2c47c874135e86d32306dabe181f460c"),
    "minmax_dense_255": (2, "4928285c12afedb0cd8a5ec951a01b1196ca39348e945194f241dbc821049889"),
    "minmax_hash_0": (2, "a989a59338c81c3eb4422412af21318233dcbd1bc24b7e0262c6a99e86cfb7b9"),
    "minmax_hash_255": (2, "d36a3eb662dcf91825a0e4d3273595a2b573ff7876c714fa75ebb51f59825646"),
    "minmax_plain_0": (0, "f91941afb0912d4d760f751059c553065732db89a2861113116e519c05828f77"),
    "minmax_plain_255": (0, "181b662f4a1298df61f9a257602ca18807b8551b9a34331e6b480277213216b7"),
    "minmax_small_0": (1, "97ae17607ee9ed6b210d023af46edc5eeba78a0be0734fa8831ea5cfe5cc2e30"),
    "minmax_small_255": (1, "4c57533bae3c98f7bc72c44ab1d97ec5a9d1ee34d54db5e6d170f02712b57fa2"),
    "minmax_two_0": (1, "c09a341e245f4989258f45d1fc048612862aba5c9e6b062e1b00b43e58d16ff8"),
    "minmax_two_255": (1, "a8aff84b34295c343400f9d2e9231a0d9e2b30905fefced888fce9f3bf967d2a"),
    "q1": (1, "c21b7f19155287fe08b871ac3881845ada184f3dfc9dd7f1b682d7bad041405a"),
    "q6": (0, "203d1097baf8fc3b30dd6902d097fc2adc097f6aaf1f1960d68c270425969637"),
    "sums_dense_0": (2, "fdfc18cf7c6622ededba9e992349cfd3bea0b504f1f2c46c10a11c9f01a0ff35"),
    "sums_dense_255": (2, "91b38ab8c43145ab16533abb68a2a733811c6a45684ad6d3ba31e37e18b59ec8"),
    "sums_hash_0": (2, "7d4b71626467f8cb1b224a470b2a7b53f5e100110bf670b7d30416875bd0622f"),
    "sums_hash_255": (2, "9142f38c18aca407160bae47e481424199da8e67bfb32fd5ab7abf3d7569acd0"),
    "sums_plain_0": (0, "ce77bd4b92f4c62f9aa178569fa2ba0d3330fba4ae8e2bd277066946b21dcd33"),
    "sums_plain_255": (0, "3a2a3f6900923f9cfbf3f28762dd3f978ae1ad9b008bd0ed91ddc86484676dc6"),
    "sums_small_0": (1, "9319953e2c34398f75c3197716f9bf53976ec2327ed4ac7d77a89ae7db9c923d"),
    "sums_small_255": (1, "2cdfe3413d89f314068d636fe8c84ccea0b094bbd8226860d260d05c6502bfff"),
    "sums_two_0": (2, "8298d92341f7169ebe43f4860b3395579d141e3df1786ec728b0506906f0aa1e"),
    "sums_two_255": (2, "3a88ce471010a0615083e3fe0079e4cc69d3e6fe3b2ca9527c522be21c366b78"),
}




def existing_jit_shapes(cg):
    """TPC-H Q6 and Q1, C2 (plain, NULLs, hash), and a grid of every other aggregate kind and key form"""
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
    shapes = {"q6": (q6, lineitem, 0, -1, 600_000_000, 0),
              "q1": (q1, lineitem, 65 | (70 << 32), 68 | (72 << 32), 600_000_000, 0),
              "c2": (c2, c2cols, 0, 999_999, 1_000_000_000, 0),
              "c2_null": (c2, c2cols, 0, 999_999, 1_000_000_000, 0b100),
              "c2_hash": (c2h, c2cols, 0, -1, 1_000_000_000, 0)}
    # every aggregate kind and argument form, FILTER, bool / bit, IN lists and composite keys, in every table kind
    cols = [(1, 0), (2, 0), (4, 0), (8, 0), (4, 1), (8, 1), (8, 0), (-1, 2 | (2 << 8))]
    aggsets = {
        "sums": [cg.count_star(), cg.sum_(3), cg.Agg(2, [(2, 0, 1)], term_abs_bound=1000), cg.Agg(2, [(1, 0, 1), (2, 7, -1)]),
                 cg.sum_(5, True), cg.count(7)],
        "minmax": [cg.min_(3), cg.max_(5, True), cg.min_(7), cg.count_star()],
        "filter": [cg.count_star(filter=(3, "<", 10)), cg.sum_(3, filter=("or", (1, ">", 2), (5, "<", 0.5))), cg.max_(2)],
        "boolbit": [cg.bool_and((3, ">", 0)), cg.bool_or(("and", (1, "<", 3), (5, ">=", 1.0))), cg.bit_and(2), cg.bit_or(3)],
        "lists": [cg.count_star(filter=(3, "in", (1, 2, None))), cg.sum_(6, filter=(2, "not in", (5,)))],
    }
    where = {"sums": [(6, "<", 100)], "minmax": ("or", (0, ">", 1), (7, "<=", 40)), "filter": [],
             "boolbit": [(2, ">=", -5)], "lists": [(0, "in", (1, 2, 3)), (6, "is not null")]}
    groups = {"plain": ([], 0, -1, 0), "small": ([1], 0, 3, 0), "dense": ([1], 0, 100_000, 0), "hash": ([2], 0, -1, 1000),
              "two": ([0, 1], 0 | (0 << 32), 3 | (5 << 32), 0)}
    for an, aggs in aggsets.items():
        for gn, (g, kmin, kmax, eg) in groups.items():
            d = cg.make_desc(where[an], g, aggs, float_cols=(4, 5), expected_groups=eg)
            for nullable in (0, 0xff):
                shapes[f"{an}_{gn}_{nullable}"] = (d, cols, kmin, kmax, 1 << 24, nullable)
    for k in (1, 3):
        g = [0, 1, 3][:k]
        bounds = [(-3, 4), (0, 9), (-1000, 1000)][:k]
        d = cg.make_desc([(6, ">", 0)], g, [cg.count_star(), cg.sum_(3)], composite=True, key_bounds=bounds)
        for nullable in (0, 0xff):
            shapes[f"composite{k}_{nullable}"] = (d, cols, 0, -1, 1 << 24, nullable)
    return shapes


@pytest.mark.parametrize("name", sorted(PARENT_SOURCE))
def test_plans_without_the_kind_generate_the_parent_source(cg, name):
    d, cols, kmin, kmax, rows, nullable = existing_jit_shapes(cg)[name]
    rc, kind, src = compile_check(d, cols, kmin, kmax, rows, nullable)
    assert rc == 0
    assert (kind, hashlib.sha256(src.encode()).hexdigest()) == tuple(PARENT_SOURCE[name])
    assert "qlimbs" not in src
