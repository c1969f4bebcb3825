"""The fast kernel over narrow (bit-packed) column images gives, bit for bit, what the interpretive kernel gives over the
plain arena of the same staged shards: direct-indexed, hash and plain-aggregate plans; shards whose chunk groups have
NULLs in some chunk groups only; plans that read a column without images next to ones that read only columns with
them, and plans of more than three columns, which take the plain arena; widths 0 and 32; several shards chained into one
partial; and WHERE lists that skip chunk groups."""
import numpy as np
import pytest
from gpu_harness import cg  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

ROWS = 100_000 + 37          # 11 chunk groups, the last one short


def make_rel(cg, seed, nulls=False, key_base=0, nkeys=5000):
    """key (sorted within the shard, so that WHERE lists on it skip chunk groups), f in [0, 100), v in +-1e9,
    w spanning 2^40 (no images), c constant (width 0), x spanning exactly 2^32 - 1 in every chunk group (width 32)"""
    rng = np.random.default_rng(seed)
    key = np.sort(rng.integers(0, nkeys, ROWS)) + key_base
    f = rng.integers(0, 100, ROWS)
    v = rng.integers(-10**9, 10**9 + 1, ROWS)
    v[:5] = [-10**9, 10**9, 0, -1, 1]
    w = rng.integers(-(1 << 40), 1 << 40, ROWS)
    c = np.full(ROWS, -123456789012)
    x = rng.integers(-(1 << 31), 1 << 31, ROWS)
    x[0::10_000] = -(1 << 31)
    x[1::10_000] = (1 << 31) - 1
    vn = None
    if nulls:
        vn = np.zeros(ROWS, np.uint8)
        vn[50_000:] = rng.random(ROWS - 50_000) < 0.05     # NULLs in the second half of the chunk groups only
    return cg.Relation.write([8] * 6, [key, f, v, w, c, x], nulls=[None, None, vn, None, None, None])


def run(cg, rels, shards, quals, group, aggs, hash_=False, reference=False):
    d = cg.make_desc(quals, group, aggs)
    kmin, kmax = None, None
    bounds = [0] * len(aggs)
    for r in rels:
        a, b, bs, _ = cg.relation_bounds(r, d)
        kmin = a if kmin is None else min(kmin, a)
        kmax = b if kmax is None else max(kmax, b)
        bounds = [max(x, y) for x, y in zip(bounds, bs)]
    for a, b in zip(aggs, bounds):
        a.term_abs_bound = b
    d = cg.make_desc(quals, group, aggs)
    if hash_ or not group:
        kmin, kmax = 0, -1
    if reference:
        cg.set_option("force_general", 1)
    try:
        agg = cg.GpuColumnarAgg(d, rels[0].column_descs(), kmin, kmax, ROWS * len(rels))
        stats = [agg.scan_shard(sh) for sh in shards]
        got = agg.groups()
        agg.free()
    finally:
        cg.set_option("force_general", 0)
    return got, stats


def check(cg, rels, quals, group, aggs_fn, hash_=False, expect_narrow=True):
    shards = [cg.Shard(r) for r in rels]
    try:
        from citus_b200 import capi
        for sh in shards:
            assert [capi.lib().cg_shard_narrow_column(sh.h, a) for a in range(6)] == [1, 1, 1, 0, 1, 1]
            assert capi.lib().cg_shard_narrow_bytes(sh.h) > 0
        got, st = run(cg, rels, shards, quals, group, aggs_fn(), hash_)
        want, st_ref = run(cg, rels, shards, quals, group, aggs_fn(), hash_, reference=True)
        assert got == want
        for a, b in zip(st, st_ref):
            assert (a.rows_scanned, a.rows_removed_by_filter, a.chunk_groups_scanned, a.chunk_groups_filtered) == \
                   (b.rows_scanned, b.rows_removed_by_filter, b.chunk_groups_scanned, b.chunk_groups_filtered)
            if expect_narrow:
                # the narrow streams are what the fast kernel read (a shard whose chunk groups were all skipped read none)
                assert a.bytes_scanned < b.bytes_scanned or a.bytes_scanned == b.bytes_scanned == 0
            else:
                assert a.bytes_scanned == b.bytes_scanned
        return got
    finally:
        for sh in shards:
            sh.free()


@pytest.mark.parametrize("nulls", [False, True])
def test_dense_c2_shape(cg, nulls):
    rels = [make_rel(cg, 1, nulls), make_rel(cg, 2, nulls)]
    check(cg, rels, [(1, "<", 50)], [0], lambda: [cg.sum_(2), cg.count_star()])


def test_widths_zero_and_32(cg):
    rels = [make_rel(cg, 3), make_rel(cg, 4)]
    check(cg, rels, [(1, "<", 50)], [0], lambda: [cg.sum_(4), cg.count_star()])              # c: width 0
    check(cg, rels, [(1, "<", 50)], [0], lambda: [cg.sum_(5), cg.count_star()])              # x: width 32
    check(cg, rels, [(1, "<", 50)], [], lambda: [cg.sum_(5), cg.count_star()])              # two columns: two row pairs a lane
    check(cg, rels, [(4, "=", -123456789012)], [], lambda: [cg.sum_(5), cg.count_star()])


def test_more_than_three_columns_take_the_plain_arena(cg):
    rels = [make_rel(cg, 3), make_rel(cg, 4)]
    check(cg, rels, [(1, ">=", 10), (2, "<", 0)], [0], lambda: [cg.sum_(4), cg.count_star()], expect_narrow=False)
    check(cg, rels, [(1, "<>", 7)], [0], lambda: [cg.sum_(2), cg.sum_(5), cg.count_star()], expect_narrow=False)


@pytest.mark.parametrize("nulls", [False, True])
def test_hash_table(cg, nulls):
    # keys near INT64_MAX: the image's base carries all the high bits
    big = (1 << 63) - 1 - 10_000
    rels = [make_rel(cg, 5, nulls, key_base=big), make_rel(cg, 6, nulls, key_base=big)]
    check(cg, rels, [(1, "<", 50)], [0], lambda: [cg.sum_(2), cg.count_star()], hash_=True)


@pytest.mark.parametrize("nulls", [False, True])
def test_plain_aggregate(cg, nulls):
    rels = [make_rel(cg, 7, nulls), make_rel(cg, 8, nulls), make_rel(cg, 9, nulls)]
    check(cg, rels, [(1, "<", 50)], [], lambda: [cg.sum_(2), cg.sum_(4), cg.count_star()])
    check(cg, rels, [], [], lambda: [cg.sum_(0), cg.count_star()])


def test_column_without_images_takes_the_plain_arena(cg):
    # w spans 2^40: a plan that reads it runs the plain fast kernel on the same shard
    rels = [make_rel(cg, 10), make_rel(cg, 11)]
    check(cg, rels, [(1, "<", 50)], [0], lambda: [cg.sum_(3), cg.count_star()], expect_narrow=False)
    check(cg, rels, [(1, "<", 50)], [0], lambda: [cg.sum_(2), cg.count_star()])


def test_chunk_group_skipping(cg):
    rels = [make_rel(cg, 12, key_base=0), make_rel(cg, 13, key_base=2500)]
    check(cg, rels, [(0, ">=", 1000), (0, "<", 3000)], [], lambda: [cg.sum_(2), cg.count_star()])
    got = check(cg, rels, [(1, "<", 50), (0, ">=", 6000)], [], lambda: [cg.sum_(2), cg.count_star()])
    assert got == {} or len(got) == 1
