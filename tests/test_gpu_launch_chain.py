"""Consecutive scan launches on the library's stream overlap (programmatic dependent launch of the fast and the generated
scan kernels).  Every case here scans several shards into one partial, back to back, with and without the library
enqueues that end a chain in between (a reset, packed-word drains, an IN-list upload, a WHERE change that rewrites the
selected chunk-group list, statistics read-backs, cg_scan_relation's staging kernels, a second partial), and checks the
groups bit for bit against the oracle or the exact reference; and the scan profiling counters around such chains."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import reference as ref
from test_gpu_scan import assert_same_groups, oracle_table, to_oracle_aggs
from gpu_harness import cg  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

ROWS = 120_000            # per shard: 12 chunk groups of 10 000 rows
NSHARDS = 6
NKEYS = 5_000             # a direct-indexed table too large for the shared-memory kernel


@pytest.fixture
def kernel_family(cg):
    def use(name):
        cg.set_option("jit", {"jit": 1, "aot": 0}[name])
    yield use
    cg.set_option("jit", 1)


def make_shards(cg, seed, null_mode="none", nkeys=NKEYS, nshards=NSHARDS, rows=ROWS):
    """(relation, arrays) per shard: key, f in [0, 100), v; null_mode 'all' puts NULLs in v of every chunk group,
    'half' in the second half of the chunk groups only (one call then takes both the fast and the generated kernel)"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(nshards):
        key = rng.integers(0, nkeys, rows)
        f = rng.integers(0, 100, rows)
        v = rng.integers(-10**9, 10**9, rows)
        vn = None
        if null_mode != "none":
            vn = (rng.random(rows) < 0.05).astype(np.uint8)
            if null_mode == "half":
                vn[: rows // 2] = 0
        rel = cg.Relation.write([8, 8, 8], [key, f, v], nulls=[None, None, vn])
        out.append((rel, (key, f, v), vn))
    return out


def make_partial(cg, shards, quals, aggs, where=None):
    aggs = [dataclasses.replace(a) for a in aggs]
    d = cg.make_desc(where if where is not None else quals, [0], aggs)
    bounds = [0] * len(aggs)
    kmin, kmax = None, None
    for rel, _, _ in shards:
        a, b, bs, _ = cg.relation_bounds(rel, d)
        bounds = [max(x, y) for x, y in zip(bounds, bs)]
        kmin = a if kmin is None else min(kmin, a)
        kmax = b if kmax is None else max(kmax, b)
    for a, b in zip(aggs, bounds):
        a.term_abs_bound = b
    d = cg.make_desc(where if where is not None else quals, [0], aggs)
    return cg.GpuColumnarAgg(d, shards[0][0].column_descs(), kmin, kmax, ROWS * len(shards) * 4), aggs


def oracle_groups(oracle, shards, quals, aggs, times=1):
    want = oracle.Result(to_oracle_aggs(oracle, aggs))
    for _ in range(times):
        for rel, _, _ in shards:
            oracle_table(oracle, rel).scan(quals, [0], to_oracle_aggs(oracle, aggs), into=want)
    return want.groups()


def c2_aggs(cg):
    return [cg.sum_(2), cg.count_star()]


def scan_all(agg, staged):
    for sh in staged:
        agg.scan_shard(sh, want_stats=False)


@pytest.mark.parametrize("null_mode,family", [("none", "aot"), ("none", "jit"), ("all", "jit"), ("half", "aot")])
def test_back_to_back_shards_into_one_partial(cg, oracle, kernel_family, null_mode, family):
    """fast kernel (NULL-free, aot), generated kernel (jit, and NULL-bearing chunk groups), a call whose chunk groups go
    to both (half): every shard's launch chained onto the previous one"""
    kernel_family(family)
    shards = make_shards(cg, 11, null_mode)
    quals = [(1, "<", 50)]
    aggs = c2_aggs(cg)
    agg, aggs = make_partial(cg, shards, quals, aggs)
    staged = [cg.Shard(rel) for rel, _, _ in shards]
    scan_all(agg, staged)
    assert_same_groups(agg.groups(), oracle_groups(oracle, shards, quals, aggs), aggs)


def test_reset_between_queries(cg, oracle):
    shards = make_shards(cg, 12)
    quals = [(1, "<", 50)]
    agg, aggs = make_partial(cg, shards, quals, c2_aggs(cg))
    staged = [cg.Shard(rel) for rel, _, _ in shards]
    want = oracle_groups(oracle, shards, quals, aggs)
    for _ in range(3):
        agg.reset()
        scan_all(agg, staged)
        agg.reset()                      # a reset right behind a chain, then the same chain again
        scan_all(agg, staged)
        assert_same_groups(agg.groups(), want, aggs)


def test_packed_drains_between_chained_scans(cg, oracle):
    """a small key domain makes the library drain the packed words in the middle of the shard sequence (the rows since
    the last drain pass capacity * 2^C / 32), and reads between launches drain them too"""
    from citus_b200 import capi
    shards = make_shards(cg, 13, nkeys=500, nshards=12, rows=200_000)
    quals = [(1, "<", 90)]
    agg, aggs = make_partial(cg, shards, quals, c2_aggs(cg))
    staged = [cg.Shard(rel) for rel, _, _ in shards]
    before = capi.lib().cg_kernel_launches()
    scan_all(agg, staged)
    launches = capi.lib().cg_kernel_launches() - before
    assert launches > len(staged)        # at least one drain kernel among the scans
    assert_same_groups(agg.groups(), oracle_groups(oracle, shards, quals, aggs), aggs)
    agg.reset()
    for i, sh in enumerate(staged):
        agg.scan_shard(sh, want_stats=False)
        if i % 3 == 1:
            agg.ngroups()                # a read in between: the next scan drains first
    assert_same_groups(agg.groups(), oracle_groups(oracle, shards, quals, aggs), aggs)


def test_in_list_change_between_shards(cg):
    """each shard its own IN list: the list upload between two scans of one partial ends the chain, and the scan behind
    it reads the new list"""
    shards = make_shards(cg, 14, nshards=4, rows=30_000)
    aggs = c2_aggs(cg)
    lists = [tuple(range(0, 100, 3)), tuple(range(1, 100, 7)), tuple(range(0, 100, 3)), (5, 6, 7, 50, 99)]
    where0 = [(1, "in", lists[0])]
    agg, aggs = make_partial(cg, shards, None, aggs, where=where0)
    want = {}
    for (rel, cols, vn), lst in zip(shards, lists):
        where = [(1, "in", lst)]
        d = cg.make_desc(where, [0], aggs)
        agg.desc = d
        sh = cg.Shard(rel)
        agg.scan_shard(sh, want_stats=False)
        r = ref.aggregate(list(cols), [None, None, vn], where, [0], aggs)
        for k, per in r.groups.items():
            acc = want.setdefault(k[0], [[0, 0] for _ in aggs])
            for a, st in enumerate(per):
                acc[a][0] += st.sum
                acc[a][1] += st.count
    got = agg.groups()
    assert set(got) == set(want)
    for k, per in want.items():
        for a, (s, n) in enumerate(per):
            assert got[k][a]["count"] == n, (k, a)
            if aggs[a].kind == 2 and n:
                assert got[k][a]["sum"] == s, (k, a)


def test_where_change_rewrites_selected_list(cg, oracle):
    """a sorted filter column, so the two WHERE lists select different chunk groups: the rewrite of the shard's
    selected list between two scans ends the chain"""
    rng = np.random.default_rng(15)
    shards = []
    for s in range(4):
        key = rng.integers(0, NKEYS, ROWS)
        f = np.sort(rng.integers(0, 100, ROWS))
        v = rng.integers(-10**9, 10**9, ROWS)
        shards.append((cg.Relation.write([8, 8, 8], [key, f, v]), None, None))
    q1, q2 = [(1, "<", 30)], [(1, ">=", 60)]
    agg, aggs = make_partial(cg, shards, q1, c2_aggs(cg))
    staged = [cg.Shard(rel) for rel, _, _ in shards]
    d1, d2 = cg.make_desc(q1, [0], aggs), cg.make_desc(q2, [0], aggs)
    want = oracle.Result(to_oracle_aggs(oracle, aggs))
    for (rel, _, _), sh in zip(shards, staged):
        for d, q in ((d1, q1), (d2, q2)):
            agg.desc = d
            agg.scan_shard(sh, want_stats=False)
            oracle_table(oracle, rel).scan(q, [0], to_oracle_aggs(oracle, aggs), into=want)
    assert_same_groups(agg.groups(), want.groups(), aggs)


def test_statistics_on_some_calls(cg, oracle):
    shards = make_shards(cg, 16)
    quals = [(1, "<", 50)]
    agg, aggs = make_partial(cg, shards, quals, c2_aggs(cg))
    staged = [cg.Shard(rel) for rel, _, _ in shards]
    for i, sh in enumerate(staged):
        st = agg.scan_shard(sh, want_stats=(i % 2 == 1))
        if i % 2 == 1:
            assert st.rows_scanned == ROWS
            assert st.kernel_ms > 0
    assert_same_groups(agg.groups(), oracle_groups(oracle, shards, quals, aggs), aggs)


@pytest.mark.parametrize("null_mode", ["none", "all"])
def test_scan_relation_between_shard_scans(cg, oracle, null_mode):
    """cg_scan_relation stages through realign / rank kernels on the same stream in front of its own scans"""
    shards = make_shards(cg, 17, null_mode)
    quals = [(1, "<", 50)]
    agg, aggs = make_partial(cg, shards, quals, c2_aggs(cg))
    staged = [cg.Shard(rel) for rel, _, _ in shards]
    for i, ((rel, _, _), sh) in enumerate(zip(shards, staged)):
        if i % 2:
            agg.scan_relation(rel, want_stats=False)
        else:
            agg.scan_shard(sh, want_stats=False)
    shards[1][0].register()
    try:
        agg.scan_relation(shards[1][0], want_stats=False)          # pinned pages: the DMA path with its realign kernel
    finally:
        shards[1][0].unregister()
    want = oracle.Result(to_oracle_aggs(oracle, aggs))
    for rel in [s[0] for s in shards] + [shards[1][0]]:
        oracle_table(oracle, rel).scan(quals, [0], to_oracle_aggs(oracle, aggs), into=want)
    assert_same_groups(agg.groups(), want.groups(), aggs)


def test_two_partials_scanned_alternately(cg, oracle):
    shards = make_shards(cg, 18)
    q1, q2 = [(1, "<", 50)], [(1, ">=", 20)]
    a1, aggs1 = make_partial(cg, shards, q1, c2_aggs(cg))
    a2, aggs2 = make_partial(cg, shards, q2, [cg.sum_(2), cg.count_star(), cg.sum_(1)])
    staged = [cg.Shard(rel) for rel, _, _ in shards]
    for rep in range(2):
        for sh in staged:
            a1.scan_shard(sh, want_stats=False)
            a2.scan_shard(sh, want_stats=False)
    assert_same_groups(a1.groups(), oracle_groups(oracle, shards, q1, aggs1, times=2), aggs1)
    assert_same_groups(a2.groups(), oracle_groups(oracle, shards, q2, aggs2, times=2), aggs2)


def test_profile_counts_scan_launches_and_chain_time(cg):
    import time

    import torch
    from citus_b200 import capi
    shards = make_shards(cg, 19)
    agg, _ = make_partial(cg, shards, [(1, "<", 50)], c2_aggs(cg))
    staged = [cg.Shard(rel) for rel, _, _ in shards]
    scan_all(agg, staged)
    agg.ngroups()
    torch.cuda.synchronize()
    lib = capi.lib()
    capi.check(lib.cg_profile_begin())
    t0 = time.perf_counter()
    for _ in range(3):
        agg.reset()
        scan_all(agg, staged)
        agg.ngroups()
    torch.cuda.synchronize()
    wall_ms = (time.perf_counter() - t0) * 1e3
    n, total, longest = C.c_int32(), C.c_double(), C.c_double()
    capi.check(lib.cg_profile_collect(C.byref(n), C.byref(total), C.byref(longest)))
    assert n.value == 3 * len(staged)                   # one fast-kernel launch per shard scan
    assert total.value > 0 and longest.value > 0
    assert longest.value <= total.value <= wall_ms
