"""Composite GROUP BY keys on the host side, without a GPU: the checks of the new CgScanDesc fields, the key codec
(cg_group_key_encode / cg_group_key_decode) against a plain restatement of the formula, the per-column bounds of
cg_relation_key_bounds against the rows of the chunk groups the reference keeps, and the generated kernels of every
table kind with 1..4 key columns of every width."""
import ctypes as C
import itertools

import numpy as np
import pytest

import reference as ref

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
BPCHAR1, NUMERIC2 = 3, 2 | (2 << 8)


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


# --------------------------------------------------------------------------- the formula, restated
def radix(lo, hi):
    return 1 if lo > hi else hi - lo + 2


def encode(bounds, key):
    code = 0
    for (lo, hi), v in zip(bounds, key):
        code = code * radix(lo, hi) + (0 if v is None else v - lo + 1)
    return code


def domain(bounds):
    d = 1
    for lo, hi in bounds:
        d *= radix(lo, hi)
    return d


def composite_desc(cg, bounds, group_cols=None, aggs=None):
    group_cols = list(range(len(bounds))) if group_cols is None else group_cols
    return cg.make_desc([], group_cols, aggs or [cg.count_star()], composite=True, key_bounds=bounds)


# --------------------------------------------------------------------------- validation
def test_more_than_two_columns_need_the_composite_form(cg):
    from citus_b200 import capi
    cols = [(4, 0)] * 5
    for k in (3, 4):
        d = cg.make_desc([], list(range(k)), [cg.count_star()])
        assert compile_check(d, cols, 0, 9)[0] == capi.CG_EINVAL
        assert compile_check(composite_desc(cg, [(0, 9)] * k), cols)[0] == 0
    d = composite_desc(cg, [(0, 9)] * 4)
    d.ngroup_cols = 5
    assert compile_check(d, cols)[0] == capi.CG_EINVAL
    d = composite_desc(cg, [(0, 9)])
    d.ngroup_cols = 0
    assert compile_check(d, cols)[0] == capi.CG_EINVAL
    d = composite_desc(cg, [(0, 9)])
    d.composite_key = 2
    assert compile_check(d, cols)[0] == capi.CG_EINVAL


def test_wide_and_float_key_columns(cg):
    from citus_b200 import capi
    cols = [(8, 0), (4, 0), (8, 1)]
    # the packed form refuses a wide column in a two-column key; the composite form takes it
    assert compile_check(cg.make_desc([], [0, 1], [cg.count_star()]), cols, 0, 9)[0] == capi.CG_EUNSUPPORTED
    assert compile_check(composite_desc(cg, [(-5, 5), (0, 3)], [0, 1]), cols)[0] == 0
    assert compile_check(composite_desc(cg, [(-5, 5), (0, 3)], [0, 2]), cols)[0] == capi.CG_EUNSUPPORTED
    assert compile_check(composite_desc(cg, [(0, 3)], [2]), cols)[0] == capi.CG_EUNSUPPORTED


@pytest.mark.parametrize("bounds, ok", [
    ([(0, 2**63 - 2)], True),                                   # R = 2^63
    ([(0, 2**63 - 1)], False),                                  # R = 2^63 + 1
    ([(INT64_MIN, INT64_MAX)], False),                          # R = 2^64 + 1
    ([(0, 2**31 - 2), (-7, 2**32 - 9)], True),                  # 2^31 * 2^32
    ([(0, 1), ((-(2**63 + 1) // 3) + 2, 0)], False),           # 3 * (2^63 + 1) / 3 = 2^63 + 1
    ([(0, 3), (0, 2**61 - 2), (5, 4)], False),                  # 5 * 2^61 * 1
    ([(0, 0), (0, 0), (0, 2**61 - 2), (5, 4)], True),           # 2 * 2 * 2^61 * 1 = 2^63
    ([(0, 0), (0, 2), (0, 2**61 - 2), (5, 4)], False),          # 2 * 4 * 2^61
])
def test_domain_limit_is_two_to_the_63(cg, bounds, ok):
    from citus_b200 import capi
    assert (domain(bounds) <= 2**63) == ok
    cols = [(8, 0)] * len(bounds)
    rc, kind, _ = compile_check(composite_desc(cg, bounds), cols)
    assert rc == (0 if ok else capi.CG_EUNSUPPORTED)
    if ok:
        assert kind == 2                                        # a domain this large is hashed
    codes = np.zeros(1, np.int64)
    rc = capi.lib().cg_group_key_encode(C.byref(composite_desc(cg, bounds)), 1, np.zeros(len(bounds), np.int64).ctypes.data,
                                        np.ones(len(bounds), np.uint8).ctypes.data, codes.ctypes.data)
    assert rc == (0 if ok else capi.CG_EUNSUPPORTED)


def test_key_bounds_are_ignored_by_other_forms(cg):
    """a zero-filled tail is today's forms; the packed form reads key_min / key_max only"""
    cols = [(4, 0), (4, 0)]
    d = cg.make_desc([], [0, 1], [cg.count_star()])
    assert d.composite_key == 0 and list(d.key_col_min) == [0] * 4
    rc, kind, src = compile_check(d, cols, 0, 9)
    assert rc == 0 and "kcode" not in src and "kradix" not in src


# --------------------------------------------------------------------------- encode / decode
def _edge_bounds(rng, k):
    """bounds of k columns whose domain stays <= 2^63: int64 edges, single values, all-NULL columns"""
    choices = [(INT64_MIN, INT64_MIN + 5), (INT64_MAX - 9, INT64_MAX), (7, 7), (3, 2), (INT64_MAX, INT64_MIN), (-3, 300),
               (INT64_MIN, INT64_MIN), (INT64_MAX, INT64_MAX), (-(2**40), -(2**40) + 1000), (0, 2**62)]
    while True:
        b = [choices[int(rng.integers(0, len(choices)))] for _ in range(k)]
        if domain(b) <= 2**63:
            return b


def _keys_in(rng, bounds, n):
    keys = []
    for _ in range(n):
        key = []
        for lo, hi in bounds:
            if lo > hi or rng.random() < 0.2:
                key.append(None)
            else:
                key.append(int(lo + int(rng.integers(0, min(hi - lo, 2**62) + 1, dtype=np.int64))) if rng.random() < 0.6 else
                           [lo, hi][int(rng.integers(0, 2))])
        keys.append(tuple(key))
    return keys


@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_encode_decode_round_trip_at_the_edges(cg, k):
    rng = np.random.default_rng(4000 + k)
    for _ in range(40):
        bounds = _edge_bounds(rng, k)
        d = composite_desc(cg, bounds)
        keys = _keys_in(rng, bounds, 50)
        keys += [tuple(None if (i >> c) & 1 or lo > hi else lo for c, (lo, hi) in enumerate(bounds)) for i in range(1 << k)]
        keys += [tuple(None if lo > hi else hi for lo, hi in bounds)]
        codes = cg.group_key_encode(d, keys)
        assert [int(c) for c in codes] == [encode(bounds, key) for key in keys]
        assert all(0 <= int(c) < domain(bounds) for c in codes)
        assert cg.group_key_decode(d, codes) == keys


@pytest.mark.parametrize("k", [2, 3, 4])
def test_codes_sort_like_the_tuples_with_null_lowest(cg, k):
    rng = np.random.default_rng(5000 + k)
    bounds = [(-2, 3), (5, 4), (10, 12), (INT64_MAX - 1, INT64_MAX)][:k]
    d = composite_desc(cg, bounds)
    values = [[None] + (list(range(lo, hi + 1)) if lo <= hi else []) for lo, hi in bounds]
    keys = list(itertools.product(*values))
    assert len(keys) == domain(bounds)
    order = sorted(keys, key=lambda t: tuple((0, 0) if v is None else (1, v) for v in t))
    codes = cg.group_key_encode(d, order)
    assert [int(c) for c in codes] == list(range(domain(bounds)))    # dense, and in tuple order
    rng.shuffle(keys)
    assert cg.group_key_decode(d, cg.group_key_encode(d, keys)) == keys


def test_codec_refuses_what_lies_outside(cg):
    from citus_b200 import capi
    bounds = [(-2, 3), (0, 0)]
    d = composite_desc(cg, bounds)
    for key in ((4, 0), (-3, None), (0, 1)):
        with pytest.raises(capi.CitusGpuError) as e:
            cg.group_key_encode(d, [key])
        assert e.value.code == capi.CG_EINVAL
    for code in (-1, domain(bounds), INT64_MAX):
        with pytest.raises(capi.CitusGpuError) as e:
            cg.group_key_decode(d, [code])
        assert e.value.code == capi.CG_EINVAL
    plain = cg.make_desc([], [0, 1], [cg.count_star()])
    with pytest.raises(capi.CitusGpuError) as e:
        cg.group_key_decode(plain, [0])
    assert e.value.code == capi.CG_EINVAL


# --------------------------------------------------------------------------- bounds from the skip lists
def _rows_bounds(cols, nulls, where, group_cols, stripe_rows, chunk_rows):
    """per group column: (min, max) over the non-NULL values of the chunk groups selected_chunk_mask keeps"""
    mask = ref.selected_chunk_mask(cols, nulls, where, stripe_rows, chunk_rows)
    layout = ref.chunk_layout(len(cols[0]), stripe_rows, chunk_rows)
    out = []
    for c in group_cols:
        vals = [int(cols[c][r]) for stripe, m in zip(layout, mask) for (f, n), keep in zip(stripe, m) if keep
                for r in range(f, f + n) if nulls[c] is None or not nulls[c][r]]
        out.append((min(vals), max(vals)) if vals else (INT64_MAX, INT64_MIN))
    return out


def test_relation_key_bounds_follow_the_kept_chunks(cg, oracle):
    """skipped chunk groups, all-NULL chunks, char(1) and numeric(12, 2) key columns"""
    rng = np.random.default_rng(20261016)
    n, stripe_rows, chunk_rows = 8000, 2000, 500
    sorted_col = np.sort(rng.integers(-10**6, 10**6, n))               # chunks skipped on it
    flag = rng.integers(0, 256, n)
    money = rng.integers(-10**9, 10**9, n)                            # numeric(12, 2) as scaled integers
    small = rng.integers(-128, 128, n)
    wide = rng.integers(INT64_MIN, INT64_MAX, n, endpoint=True)
    wide[:2] = [INT64_MIN, INT64_MAX]
    allnull = np.zeros(n, np.int64)
    nulls = [None, rng.random(n) < 0.1, rng.random(n) < 0.1, None, rng.random(n) < 0.05, np.ones(n, bool)]
    nulls[2][1000:1500] = True                                        # an all-NULL chunk of the numeric column
    nulls[1][:500] = True
    cols = [sorted_col, flag, money, small, wide, allnull]
    t = oracle.Table([8, -1, -1, 2, 8, 4], [0, BPCHAR1, NUMERIC2, 0, 0, 0], stripe_row_limit=stripe_rows, chunk_row_limit=chunk_rows)
    t.insert(cols, [None if x is None else x.astype(np.uint8) for x in nulls])
    rel = cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), [8, -1, -1, 2, 8, 4], [0, BPCHAR1, NUMERIC2, 0, 0, 0])
    for where in ([], [(0, "<", -500_000)], [(0, ">", 900_000)], ("or", (0, "<", -900_000), (0, ">", 990_000)),
                  [(0, ">", 10**7)]):
        for group in ([1, 2], [0, 3, 4], [5, 1], [2, 3, 4, 5]):
            d = cg.make_desc(where, group, [cg.count_star()])
            assert cg.relation_key_bounds(rel, d) == _rows_bounds(cols, nulls, where, group, stripe_rows, chunk_rows), (where, group)


def test_relation_key_bounds_refuse_unknown_bounds(cg):
    from citus_b200 import capi
    rel = cg.Relation.write([8, 8], [np.arange(3000), np.arange(3000) * 0.5], type_classes=[0, 1], chunk_row_limit=1000)
    with pytest.raises(capi.CitusGpuError) as e:
        cg.relation_key_bounds(rel, cg.make_desc([], [0, 1], [cg.count_star()]))
    assert e.value.code == capi.CG_EUNSUPPORTED
    assert cg.relation_key_bounds(rel, cg.make_desc([], [0], [cg.count_star()])) == [(0, 2999)]


# --------------------------------------------------------------------------- generated kernels
@pytest.mark.parametrize("nullable", [0, 0b1111111])
@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_generated_kernels_compile_for_every_kind(cg, k, nullable):
    """1-, 2-, 4- and 8-byte key columns; small-domain, direct-indexed (with the packed word) and hash kinds; WHERE,
    FILTER and a bool_or argument"""
    cols = [(1, 0), (2, 0), (4, 0), (8, 0), (8, 0), (8, 1), (-1, BPCHAR1)]
    widths = [(0, 1, 2, 3), (3, 2, 1, 0), (6, 0, 3, 2), (2, 3, 6, 1)]
    aggs = [cg.count_star(), cg.Agg(2, [(4, 0, 1)], term_abs_bound=1000), cg.min_(5, True), cg.bool_or(("or", (4, ">", 0), (1, "<", 3))),
            cg.sum_(4, filter=(2, "<>", 7))]
    seen = set()
    for group in widths:
        group = list(group[:k])
        # spans 0: 2^k codes (shared-memory cells up to three columns); 40: direct-indexed; 2^15: hashed from two columns
        for span in (0, 40, 2**15):
            bounds = [(-3, -3 + span)] * k
            d = cg.make_desc([(3, ">", -100)], group, aggs, float_cols=(5,), expected_groups=1000, composite=True, key_bounds=bounds)
            rc, kind, src = compile_check(d, cols, nullable=nullable)
            assert rc == 0, src[-3000:]
            hashed = "? h : hash_slot_slow(P, key, h)" in src
            form = "small" if kind == 1 else "hash" if hashed else "dense"
            assert form == ("small" if span == 0 and k <= 3 else "hash" if domain(bounds) > 2**26 else "dense"), (group, span)
            rows = src.count("const uint64_t kcode = ")
            assert rows > 0 and src.count(f"const uint64_t kd{k - 1} = ") == rows and f"kd{k} " not in src
            if form != "small":
                assert "red_add(P.packed + slot" in src                   # optimistic packing applies to composite tables
            seen.add(form)
    assert seen == {"small", "dense", "hash"} - ({"hash"} if k == 1 else set()) - ({"small"} if k == 4 else set())


def test_existing_plans_generate_no_composite_code(cg):
    cols = [(8, 0), (4, 0), (2, 0), (8, 0)]
    for group, kmin, kmax in (([], 0, -1), ([0], 0, 9), ([0], 0, 10**8), ([1, 2], 0, (9 << 32) | 9)):
        d = cg.make_desc([(3, ">", 0)], group, [cg.count_star(), cg.sum_(3)])
        for nullable in (0, 0b1111):
            rc, _, src = compile_check(d, cols, kmin, kmax, nullable=nullable)
            assert rc == 0
            assert "composite" not in src and "kcode" not in src and "uint8_t gcol[2]" in src
