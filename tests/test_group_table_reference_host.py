"""tests/group_table_reference.py against brute force, and its shape rules against what the library reports without a GPU
(the table kind through cg_jit_compile_check_nullable's kernel kind and generated source)."""
import random

import pytest

import group_table_reference as gt


# --------------------------------------------------------------------------- the model against brute force
def test_pack_shift_rule():
    for bound in list(range(1, 70)) + [(1 << r) + d for r in range(1, 64) for d in (-1, 0, 1)]:
        if bound <= 0 or bound >= 1 << 63:
            continue
        r = next(r for r in range(63) if r == 62 or (1 << r) > bound)
        c = (63 - r) // 2
        assert gt.pack_shift(bound) == (None if c < 12 else min(c, 24)), bound
    for c in range(12, 25):
        assert gt.pack_shift(gt.bound_for_shift(c)) == c
        if c < 24:
            assert gt.pack_shift(gt.bound_for_shift(c) + 1) == c - 1 or c == 12
    assert gt.pack_shift(gt.bound_for_shift(12) + 1) is None


def test_packed_word_round_trip_at_the_extremes():
    for c in range(12, 25):
        b = gt.bound_for_shift(c)
        for n in (1, 2, (1 << c) - 1):
            for term in (b, -b, 0, 1, -1):
                w = 0
                for _ in range(min(n, 3)):
                    w = (w + gt.pack(term, 1, c)) & gt.MASK64
                w = (w + gt.pack(term * (n - min(n, 3)), n - min(n, 3), c)) & gt.MASK64
                assert gt.unpack(w, c) == (n, term * n), (c, n, term)
        # 2^C rows: the row count wraps to 0 and the sum is off by one -- the overflow the bookkeeping must catch
        n = 1 << c
        assert gt.unpack(gt.pack(-b * n, n, c), c)[0] == 0


def test_drain_schedule_predicts_retry_exactly():
    """a simulation with real word arithmetic agrees with the claim "retry iff some slot took >= 2^C rows between two
    drains", and the drains happen where the limit says"""
    rng = random.Random(5)
    for trial in range(300):
        c = rng.choice([12, 13, 14])
        cap = rng.choice([32, 64, 1024])
        t = gt.PackedTable(cap, c)
        truth = {}
        for _ in range(rng.randint(1, 8)):
            per = {}
            for s in rng.sample(range(cap), rng.randint(1, 4)):
                n = rng.choice([1, 100, (1 << c) // 3, (1 << c) - 1, 1 << c])
                term = rng.choice([gt.bound_for_shift(c), -gt.bound_for_shift(c), 7])
                per[s] = (n, term * n)
                a = truth.setdefault(s, [0, 0])
                a[0] += n
                a[1] += term * n
            rows = sum(n for n, _ in per.values()) + rng.randint(0, cap << c >> 4)
            due = (t.rows_since_drain + rows) * 32 > cap << c
            t.launch(rows, per)
            assert (t.rows_since_drain == 0) == due
            if rng.random() < 0.2:
                got = t.read()
                assert (got is None) == t.overflowed
                if got is not None:
                    assert got == {k: (v[0], gt.s64(v[1])) for k, v in truth.items() if v[0]}
                t.read_direct = True
        got = t.read()
        assert (got is None) == t.overflowed, trial


def test_narrow_cells_and_launch_cutting():
    tb = 13421772
    assert tb * 160 < 1 << 31 <= (tb + 1) * 160
    s = gt.narrow_shape(3, [(tb, 1)] * 4)
    assert (s.kind, s.rows_partner, s.pairs, s.nhot, s.lane_rows_cap) == ("small", 0, [(1, 2)], 3, 160)
    assert gt.narrow_shape(3, [(tb, 1, True)] * 4).pairs == []
    assert gt.narrow_shape(3, [(tb, 1, False), (tb, 1, True), (tb, 1, False)]).pairs == [(2, 1)]
    s = gt.narrow_shape(3, [(tb + 1, 1)] * 4)
    assert (s.candidates, s.pairs, s.nhot, s.lane_rows_cap) == ([], [], 5, 1 << 22)
    # 2 KB per cell and entry: 200 KB are 100 cells, so the 4096-entry limit never binds before the byte limit
    assert gt.narrow_shape(100, [(5, 1)]).kind == "small" and gt.narrow_shape(101, [(5, 1)]).kind == "table"
    assert gt.narrow_shape(33, [(tb, 1)] * 4).kind == "small" and gt.narrow_shape(34, [(tb, 1)] * 4).kind == "table"
    assert gt.narrow_shape(25, [(5, 1)]).min_blocks == 4 and gt.narrow_shape(26, [(5, 1)]).min_blocks == 0
    for rows, per in ((10000, 4), (10241, 3), (20480, 2), (40960, 1), (40961, 0)):
        assert gt.cgs_per_cta(rows) == per, rows
        assert gt.rows_per_cg_lane(rows) * max(per, 1) <= 160 or per == 0
    assert gt.jit_small_launches(4 * 528 + 1, 10000, 528) == 2
    assert gt.jit_small_launches(4 * 528, 10000, 528) == 1


def test_probe_runs_do_not_depend_on_the_order():
    rng = random.Random(11)
    for trial in range(200):
        cap = rng.choice([8, 16, 64])
        hot = rng.randrange(cap)
        keys = [gt.key_with_home(hot, j, cap) for j in range(rng.randint(0, cap // 2))]
        keys += [rng.randrange(-(1 << 63), 1 << 63) for _ in range(rng.randint(0, cap))]
        distinct = sorted(set(keys))
        ref, _ = gt.probe(distinct, cap, limit=cap)
        occupied = sorted(s for s in ref.values() if s is not None)
        for _ in range(3):
            order = distinct[:]
            rng.shuffle(order)
            where, longest = gt.probe(order, cap, limit=cap)
            assert sorted(s for s in where.values() if s is not None) == occupied
            if distinct and len(distinct) <= cap:
                assert longest <= max(gt.occupied_runs(occupied, cap))
        verdict = gt.hash_verdict(keys, cap)
        assert verdict == ("full" if len(distinct) > cap else "exact")


def test_keys_sharing_a_home_slot_and_wrapping_clusters():
    cap = 1 << 12
    keys = [gt.key_with_home(cap - 1, j, cap) for j in range(3000)]
    assert {gt.home_slot(k, cap) for k in keys} == {cap - 1} and len(set(keys)) == 3000
    where, longest = gt.probe(keys, cap)
    assert longest == 3000 and where[keys[1]] == 0 and where[keys[-1]] == 2998      # wraps to slot 0
    assert gt.occupied_runs(where.values(), cap) == [3000]
    assert gt.hash_verdict(keys, cap) == "exact"
    big = 1 << 14
    run = [gt.key_with_home(5, j, big) for j in range(8191)]
    assert gt.hash_verdict(run, big) == "exact"
    assert gt.hash_verdict(run + [gt.key_with_home(5, 9000, big)], big) == "either"
    assert gt.hash_verdict([gt.key_with_home(1, j, 1024) for j in range(1025)], 1024) == "full"
    assert gt.hash_verdict([gt.HASH_EMPTY, None] + keys[:10], cap) == "exact"


def test_table_shape_rules():
    assert gt.table_shape(1, 0, (1 << 26) - 1, 0, 3) == gt.Shape("dense", 1 << 26, (1 << 26) + 1, 4)
    assert gt.table_shape(1, 0, 1 << 26, 0, 3) == gt.Shape("hash", 1 << 22, (1 << 22) + 2, 4)
    assert gt.table_shape(1, gt.I64_MIN, gt.I64_MAX, 300, 5) == gt.Shape("hash", 2048, 2050, 8)
    assert gt.table_shape(1, gt.I64_MIN, gt.I64_MAX, 1, 2).capacity == 1024
    assert gt.table_shape(1, gt.I64_MAX - 10, gt.I64_MAX, 0, 3).capacity == 11
    two = lambda lo0, hi0, lo1, hi1: ((lo0 & 0xFFFFFFFF) | ((lo1 & 0xFFFFFFFF) << 32),
                                      (hi0 & 0xFFFFFFFF) | ((hi1 & 0xFFFFFFFF) << 32))
    lo, hi = two(-(1 << 31), -(1 << 31) + 8191, (1 << 31) - 8192, (1 << 31) - 1)
    assert gt.table_shape(2, gt.s64(lo), gt.s64(hi), 0, 3).mode == "hash"          # a product of 2^26 is not below 2^26
    lo, hi = two(-(1 << 31), -(1 << 31) + 8191, (1 << 31) - 8191, (1 << 31) - 1)
    assert gt.table_shape(2, gt.s64(lo), gt.s64(hi), 0, 3).mode == "dense"
    assert gt.dense_slot(gt.s64(hi), -(1 << 31), (1 << 31) - 8191, 8191) == 8192 * 8191 - 1


# --------------------------------------------------------------------------- the library's own shape decisions (no GPU)
@pytest.fixture(scope="module")
def cg():
    from citus_b200 import build
    build.build()
    from citus_b200 import columnar
    return columnar


def compile_check(cg, d, cols, kmin, kmax, rows, nullable=0):
    import ctypes as C
    from citus_b200 import capi
    arr = (capi.CgColumnDesc * len(cols))()
    for i, (l, t) in enumerate(cols):
        arr[i].attlen, arr[i].type_class = l, t
    kind = C.c_int32(-1)
    src = C.create_string_buffer(1 << 20)
    rc = capi.lib().cg_jit_compile_check_nullable(C.byref(d), arr, len(cols), kmin, kmax, rows, nullable, C.byref(kind), src,
                                                  len(src))
    return rc, kind.value, src.value.decode()


def sums_desc(cg, ncols, tbound):
    aggs = [cg.count_star()] + [cg.sum_(1 + i) for i in range(ncols)]
    for a in aggs[1:]:
        a.term_abs_bound = tbound
    return cg.make_desc([], [0], aggs)


@pytest.mark.parametrize("tbound", [13421772, 13421773])
def test_narrow_cells_in_the_generated_source(cg, tbound):
    """three sums at tbound 13421772: one rides with the row count, two share a biased cell (lo_ / r_ / hi_) unless the
    low half's input may be NULL; at 13421773 no sum is a candidate"""
    cols = [(2, 0)] + [(4, 0)] * 3
    for nullable in (0, 0b1110, 0b0100):          # attribute 2 = the second sum, the first choice for a low half
        rc, kind, src = compile_check(cg, sums_desc(cg, 3, tbound), cols, 0, 2, 1 << 20, nullable)
        want = gt.narrow_shape(3, [(tbound, 1, bool(nullable >> (1 + i) & 1)) for i in range(3)])
        assert (rc, kind) == (0, 1)
        assert ("lo_" in src and "r_" in src and "hi_" in src) == bool(want.pairs) == \
               (tbound == 13421772 and nullable != 0b1110)
        if nullable == 0b0100 and want.pairs:
            assert want.pairs == [(2, 1)]


@pytest.mark.parametrize("cap", [25, 26, 33, 34, 100, 101, 4096, 4097])
def test_small_or_table_at_the_limits(cg, cap):
    """the shared-memory kind while capacity * cells * 2 KB fits 200 KB (and capacity <= 4096), four CTAs per SM while
    it fits 55 KB less 4 KB: with one cell (the row count, or a narrow sum riding with it) and with three (four sums
    at the narrow bound: row partner, one pair, one alone)"""
    cols = [(4, 0)] * 5
    tb = 13421772
    for nsums in (0, 1, 4):
        rc, kind, src = compile_check(cg, sums_desc(cg, nsums, tb), cols, 0, cap - 1, 1 << 20)
        want = gt.narrow_shape(cap, [(tb, 1)] * nsums)
        assert rc == 0 and kind == {"small": 1, "table": 2}[want.kind], (cap, nsums, want)
        assert ("__launch_bounds__(256, 4)" in src) == (want.min_blocks == 4), (cap, nsums)


def test_dense_or_hash_at_the_key_range_limit(cg):
    """a key range of 2^26 - 1 is direct-indexed, 2^26 is a hash table: the generated table kernel probes (calls
    hash_slot_slow) only in the second"""
    cols = [(8, 0), (8, 0)]
    d = sums_desc(cg, 1, 1000)
    for lo, hi in ((0, (1 << 26) - 1), (0, 1 << 26), (gt.I64_MAX - (1 << 26) + 1, gt.I64_MAX), (gt.I64_MIN, gt.I64_MIN + (1 << 26))):
        rc, kind, src = compile_check(cg, d, cols, lo, hi, 1 << 20)
        assert (rc, kind) == (0, 2)
        assert ("hash_slot_slow(P, key, h)" in src) == (gt.table_shape(1, lo, hi, 0, 3).mode == "hash"), (lo, hi)
