"""bit_and / bit_or / bool_and / bool_or (every) in the fused scan against the exact reference, on every kernel family.
The expected answers come from tests/reference.py: groups come from WHERE alone, and a row its FILTER does not find
TRUE is no input of that aggregate.  bool_and / bool_or
evaluate their predicate under three-valued logic (an UNKNOWN row is no input); every value is compared exactly."""
import dataclasses
import math
import os
import socket
import traceback

import numpy as np
import pytest

import reference as ref
from test_bool_bit_agg_host import bool_agg_case
from test_gpu_agg_filter import mixed_relation, scan_relation
from test_gpu_exact import gpu_run
from test_where_reference import constant_pools, random_tree
from gpu_harness import cg, kernel_family, FAMILIES  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

OPS = ("<", "<=", "=", ">=", ">", "<>")
SHAPES = [dict(group_cols=[]), dict(group_cols=[0]), dict(group_cols=[0, 1]), dict(group_cols=[2], expected_groups=4096, force_hash=True)]


def assert_exact(st, got, want, aggs, nrows):
    """counters, groups, and per aggregate the count and the exact value (bit_* / bool_* in minmax, bool as 0 / 1)"""
    assert st.rows_passed == want.rows_passed
    assert st.rows_removed_by_filter + (nrows - st.rows_scanned) == want.rows_removed
    if () in got and () not in want.groups:
        assert all(g["count"] == 0 for g in got[()])
        return
    assert set(got) == set(want.groups)
    for key, per in want.groups.items():
        for a, (spec, w) in enumerate(zip(aggs, per)):
            g = got[key][a]
            assert g["count"] == w.count, (key, a, spec.kind, g["count"], w.count)
            if w.count == 0:
                continue
            if spec.kind in (5, 6):
                assert g["minmax"] == w.value, (key, a, g["minmax"], w.value)
            elif spec.kind in (7, 8):
                assert g["minmax"] == int(w.value), (key, a, g["minmax"], w.value)
            elif spec.kind == 2 and not spec.is_float:
                assert g["sum"] == w.sum, (key, a)
            elif spec.kind == 2:
                assert w.float_sum_ok(g["fsum"]), (key, a)
            elif spec.kind in (3, 4):
                wantv = w.min if spec.kind == 3 else w.max
                if spec.is_float:
                    assert ref.float8_eq(float(np.int64(g["minmax"]).view(np.float64)), wantv), (key, a)
                else:
                    assert g["minmax"] == wantv, (key, a)


def check(cg, rel, cols, nulls, where, group_cols, aggs, n, float_cols=(), **kw):
    """the scan equals the reference; the WHERE counters equal those of the count(*)-only query"""
    want = ref.aggregate(cols, nulls, where, group_cols, aggs, float_cols)
    st, got, layout = gpu_run(cg, rel, where, group_cols, aggs, float_cols=float_cols, **kw)
    assert_exact(st, got, want, aggs, n)
    st0, _, _ = gpu_run(cg, rel, where, group_cols, [cg.count_star()], float_cols=float_cols, **kw)
    assert (st.rows_scanned, st.rows_removed_by_filter, st.chunk_groups_filtered) == \
        (st0.rows_scanned, st0.rows_removed_by_filter, st0.chunk_groups_filtered)
    return got, layout


# --------------------------------------------------------------------------- bool_agg.out
@pytest.mark.parametrize("family", FAMILIES)
def test_bool_agg_golden_queries(cg, kernel_family, family):
    """the six bool_agg.out queries over bool_test(id int4, val int4, flag bool (attlen 1), kind int4): WHERE flag,
    GROUP BY flag, GROUP BY kind, predicates such as bool_or(val > 2 OR id < 2); every(p) is bool_and(p)"""
    kernel_family(family)
    g, cols = bool_agg_case()
    rel = cg.Relation.write([4, 4, 1, 4], cols)
    flag = (2, "=", 1)
    three = [cg.bool_and(flag), cg.bool_or(flag), cg.bool_and(flag)]
    expr = [cg.bool_or(("or", (1, ">", 2), (0, "<", 2))), cg.bool_and((1, "<", 3))]
    bits = [cg.bit_and(1), cg.bit_or(1)]
    queries = [([], [], three), ([], [3], three), ([], [], expr), ([], [3], expr), ([flag], [], bits), ([], [2], bits)]
    for (sql, want_rows), (where, group, aggs) in zip(g["queries"], queries):
        got, _ = check(cg, rel, cols, None, where, group, aggs, 3)
        rows = []
        for key, per in got.items():
            cells = [("t" if k else "f") if group == [2] else str(k) for k in key]
            for a, x in zip(aggs, per):
                cells.append(("t" if x["minmax"] else "f") if a.kind in (7, 8) else str(x["minmax"]))
            rows.append(cells)
        assert sorted(rows) == sorted(want_rows), sql


# --------------------------------------------------------------------------- random predicate trees
@pytest.mark.parametrize("family", FAMILIES)
def test_random_predicate_trees_with_filters(cg, kernel_family, family):
    """random bool_and / bool_or argument trees and random FILTERs over int2 / int4 / int8 / float8 columns with
    NULL-bearing and all-NULL chunk groups, NaN and +-inf, next to bit_and / bit_or of each width: plain aggregate, one-
    and two-column direct-indexed tables and the hash table"""
    kernel_family(family)
    rng = np.random.default_rng(20261019)
    rel, cols, nulls, sr, cr = mixed_relation(cg, rng)
    fc = (5,)
    pools = constant_pools(ref.skip_minmax(cols, nulls, sr, cr, fc), [2, 4, 2, 4, 8, 8], fc)

    def atom():
        c = int(rng.integers(0, 6))
        return (c, OPS[int(rng.integers(0, 6))], pools[c][int(rng.integers(0, len(pools[c])))])

    def small_atom():                                            # atoms that are TRUE on some rows, FALSE on others
        c = int(rng.integers(2, 6))
        return (c, OPS[int(rng.integers(0, 6))], [0, 0, 0, 0, 0, 0.0][c])
    for trial in range(6):
        budget = 8
        aggs = [cg.count_star(), cg.bit_and(2), cg.bit_or(3), cg.bit_and(4), cg.bit_or(4)]
        for j in range(3):
            tree = random_tree(rng, small_atom if rng.random() < 0.6 else atom, min(3, budget))
            budget -= len(cg.flatten_where(tree)[0]) if isinstance(tree, tuple) else len(tree)
            flt = None
            if budget > 0 and rng.random() < 0.5:
                flt = random_tree(rng, small_atom, 1)
                budget -= 1
            aggs.append((cg.bool_and if j % 2 == 0 else cg.bool_or)(tree, filter=flt))
            if budget < 1:
                break
        if budget > 0:
            aggs[1] = dataclasses.replace(aggs[1], filter=(5, ">", 0.0))
        where = random_tree(rng, small_atom, 2) if trial % 2 else []
        for shape in SHAPES:
            check(cg, rel, cols, nulls, where, aggs=aggs, n=len(cols[0]), float_cols=fc, **shape)


@pytest.mark.parametrize("family", FAMILIES)
def test_unknown_groups_next_to_false_ones(cg, kernel_family, family):
    """a group whose every row is UNKNOWN (NULL result) next to a group with one FALSE row among UNKNOWN ones and a
    group with TRUE rows only; NaN atoms are never UNKNOWN; the plain aggregate over UNKNOWN rows only"""
    kernel_family(family)
    n = 12_000
    k = np.repeat(np.arange(4), n // 4)
    x = np.arange(n) % 100 + 1                                   # > 0 everywhere
    xn = np.zeros(n, np.uint8)
    xn[k == 0] = 1                                               # group 0: x NULL on every row
    xn[k == 1] = 1
    x[np.flatnonzero(k == 1)[1234]] = -5                         # group 1: one FALSE row, the rest NULL
    xn[np.flatnonzero(k == 1)[1234]] = 0
    f = np.where(k == 3, math.nan, 1.0)                           # group 3: NaN > 0 is TRUE in btree order
    cols, nulls = [k, x, f], [None, xn, None]
    rel = cg.Relation.write([8, 4, 8], cols, nulls, type_classes=[0, 0, 1], chunk_row_limit=1000)
    aggs = [cg.bool_and((1, ">", 0)), cg.bool_or((1, ">", 0)), cg.bool_or((1, "<", 0)), cg.bool_and((2, ">", 0.0)),
            cg.bool_and(("or", (1, ">", 0), (2, "<", 0.0))), cg.bit_or(1), cg.count_star()]
    for group in ([0], []):
        for force_hash in (False, True):
            got, _ = check(cg, rel, cols, nulls, [], group, aggs, n, float_cols=(2,), force_hash=force_hash, expected_groups=16)
            if group:
                assert [got[(0,)][a]["count"] for a in range(3)] == [0, 0, 0]
                assert [got[(1,)][a]["count"] for a in range(3)] == [1, 1, 1]
                assert [got[(1,)][a]["minmax"] for a in range(3)] == [0, 0, 1]
    got, _ = check(cg, rel, cols, nulls, [(0, "=", 0)], [], aggs, n, float_cols=(2,))
    assert [got[()][a]["count"] for a in range(3)] == [0, 0, 0]


# --------------------------------------------------------------------------- bit_and / bit_or of each width
@pytest.mark.parametrize("family", FAMILIES)
def test_bit_aggregates_of_every_width(cg, kernel_family, family):
    """int2 / int4 / int8 with negative values and the type limits, a group where AND reaches 0 and OR reaches -1, an
    all-NULL group, and one-value groups"""
    kernel_family(family)
    rng = np.random.default_rng(7)
    n = 16_000
    k = rng.integers(0, 5, n)
    lim = [(-2**15, 2**15 - 1), (-2**31, 2**31 - 1), (-2**63, 2**63 - 1)]
    cols = [k]
    nulls = [None]
    for lo, hi in lim:
        v = rng.integers(lo, hi, n, dtype=np.int64, endpoint=True)
        v[k == 1] = np.where(np.arange((k == 1).sum()) % 2, lo, hi)     # group 1: AND 0 (lo & hi), OR -1
        v[k == 2] = -3                                                # group 2: one value
        v[:4] = [lo, hi, 0, -1]
        z = (k == 3).astype(np.uint8)                                 # group 3: all NULL
        z[rng.random(n) < 0.05] = 1
        cols.append(v)
        nulls.append(z)
    rel = cg.Relation.write([8, 2, 4, 8], cols, nulls, chunk_row_limit=2000)
    aggs = [cg.bit_and(1), cg.bit_or(1), cg.bit_and(2), cg.bit_or(2), cg.bit_and(3), cg.bit_or(3), cg.count_star(),
            cg.bit_or(3, filter=(1, "<", 0))]
    for group in ([], [0]):
        for force_hash in (False, True):
            got, _ = check(cg, rel, cols, nulls, [], group, aggs, n, force_hash=force_hash, expected_groups=16)
            if group:
                assert [got[(1,)][a]["minmax"] for a in range(6)] == [0, -1] * 3
                assert [got[(3,)][a]["count"] for a in range(6)] == [0] * 6


# --------------------------------------------------------------------------- table kinds and kernel selection
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("nulls_on", [False, True])
def test_table_kinds(cg, kernel_family, family, nulls_on):
    """plain aggregate, small-domain (its generated kernel runs: cg_jit_launches), one- and two-column dense tables
    and the hash table, plain and nullable forms"""
    from citus_b200 import capi
    kernel_family(family)
    rng = np.random.default_rng(5)
    n = 40_000
    k1 = rng.integers(0, 6, n)
    k2 = rng.integers(0, 3, n)
    big = rng.integers(0, 50_000, n)
    v = rng.integers(-1000, 1000, n)
    w = rng.integers(0, 2, n)
    cols = [k1, k2, big, v, w]
    nulls = [None, None, None, (rng.random(n) < 0.1).astype(np.uint8) if nulls_on else None, None]
    rel = cg.Relation.write([2, 4, 8, 4, 1], cols, nulls, chunk_row_limit=4000)
    aggs = [cg.count_star(), cg.bool_or((3, ">", 900)), cg.bool_and((3, "<", 990)), cg.bit_or(3), cg.bit_and(3),
            cg.bool_or((4, "=", 1), filter=(3, ">", 0)), cg.sum_(3)]
    for group, extra in (([], {}), ([0], {}), ([0, 1], {}), ([2], {}), ([2], dict(force_hash=True, expected_groups=1 << 16))):
        j0 = capi.lib().cg_jit_launches()
        check(cg, rel, cols, nulls, [(2, "<", 45_000)], group, aggs, n, **extra)
        if group == [0] and family in ("jit", "jit_always"):
            assert capi.lib().cg_jit_launches() > j0           # the small-domain generated kernel took the plan
        if family in ("aot", "general"):
            assert capi.lib().cg_jit_launches() == j0


@pytest.mark.parametrize("family", FAMILIES)
def test_fast_kernel_shape_with_bit_or(cg, kernel_family, family):
    """count(*) + sum(bare int8 column) is the ahead-of-time specialised kernel's shape; with a bit_or or bool_or
    beside it the specialised kernel refuses the plan, and the answer stays exact"""
    kernel_family(family)
    rng = np.random.default_rng(13)
    n = 50_000
    cols = [rng.integers(0, 1000, n), rng.integers(0, 100, n), rng.integers(-10**9, 10**9, n)]
    rel = cg.Relation.write([8, 8, 8], cols, chunk_row_limit=5000)
    for aggs in ([cg.sum_(2), cg.count_star(), cg.bit_or(2)], [cg.sum_(2), cg.count_star(), cg.bool_or((2, ">", 0))],
                 [cg.count_star(), cg.bit_and(1)]):
        for group in ([], [0]):
            check(cg, rel, cols, None, [(1, "<", 50)], group, aggs, n)


@pytest.mark.parametrize("family", FAMILIES)
def test_count_bounded_sum_and_bit_or_packing_on_and_off(cg, kernel_family, family):
    kernel_family(family)
    rng = np.random.default_rng(17)
    n = 60_000
    cols = [rng.integers(0, 3000, n), rng.integers(0, 100, n), rng.integers(-10**6, 10**6, n)]
    rel = cg.Relation.write([8, 8, 8], cols, chunk_row_limit=5000)
    aggs = [cg.sum_(2), cg.count_star(), cg.bit_or(2)]
    want = ref.aggregate(cols, None, [(1, "<", 50)], [0], aggs)
    d = cg.make_desc([(1, "<", 50)], [0], aggs)
    kmin, kmax, bounds, rows = cg.relation_bounds(rel, d)
    a2 = [dataclasses.replace(a, term_abs_bound=b) for a, b in zip(aggs, bounds)]
    assert a2[0].term_abs_bound > 0 and a2[2].term_abs_bound == 0
    d = cg.make_desc([(1, "<", 50)], [0], a2)
    for packing in (True, False):
        part = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, rows)
        part.set_packing(packing)
        st = part.scan_shard(cg.Shard(rel))
        got = {(k,): per for k, per in part.groups().items()}
        assert_exact(st, got, want, a2, n)
        part.free()


# --------------------------------------------------------------------------- staging
@pytest.mark.parametrize("family", FAMILIES)
def test_argument_only_columns_through_every_staging_path(cg, kernel_family, family):
    """a column read only by a bool_or argument is staged by the shard path, by cg_scan_relation from pageable pages
    and from registered pages (DMA)"""
    kernel_family(family)
    rng = np.random.default_rng(23)
    n = 30_000
    cols = [rng.integers(0, 4, n), np.sort(rng.integers(0, 10**6, n)), rng.integers(-50, 50, n), rng.integers(0, 10**9, n)]
    rel = cg.Relation.write([8, 8, 8, 8], cols, chunk_row_limit=5000)
    where = [(1, "<", 400_000)]
    aggs = [cg.count_star(), cg.bool_or((2, ">", 45)), cg.bool_and((3, ">", 1000)), cg.bit_or(1)]
    want = ref.aggregate(cols, None, where, [0], aggs)
    st, got, _ = gpu_run(cg, rel, where, [0], aggs)
    assert_exact(st, got, want, aggs, n)
    for dma in (False, True):
        for group in ([], [0]):
            st, got = scan_relation(cg, rel, where, group, aggs, dma)
            assert_exact(st, got, ref.aggregate(cols, None, where, group, aggs), aggs, n)
            assert st.h2d_bytes > 0 and st.chunk_groups_filtered > 0


# --------------------------------------------------------------------------- combines
def test_layout_export_merge_and_fetch_merge_values_round_trips(cg):
    """word ops of each kind; export_device -> merge_rows into a fresh partial and fetch -> merge_values equal one
    scan over all rows (dense and hash tables)"""
    import torch
    from citus_b200 import capi
    L = capi.lib()
    rng = np.random.default_rng(43)
    n = 30_000
    k = rng.integers(0, 6, n)
    v = rng.integers(-10**12, 10**12, n)
    f = rng.normal(size=n)
    z = (rng.random(n) < 0.2).astype(np.uint8)
    cols, nulls = [k, v, f], [None, z, None]
    halves = [slice(0, n // 2), slice(n // 2, n)]
    rels = [cg.Relation.write([8, 8, 8], [c[h] for c in cols], [None, z[h], None], type_classes=[0, 0, 1]) for h in halves]
    aggs = [cg.bit_and(1), cg.bit_or(1, filter=(0, "<", 4)), cg.bool_and((1, ">", -9 * 10**11)), cg.bool_or(("and", (2, ">", 2.0), (1, "<", 0))),
            cg.count_star(), cg.bool_or((1, ">", 0), filter=(0, "=", 5))]
    want = ref.aggregate(cols, nulls, [], [0], aggs, (2,))
    for force_hash in (False, True):
        d = cg.make_desc([], [0], aggs, float_cols=(2,), expected_groups=16)
        kmin, kmax = (0, 5) if not force_hash else (0, -1)
        final = cg.GpuColumnarAgg(d, rels[0].column_descs(), kmin, kmax, n)
        via_values = cg.GpuColumnarAgg(d, rels[0].column_descs(), kmin, kmax, n)
        nw, ops, _, _ = final.layout()
        assert ops == [0, capi.CG_WORD_AND, 0, capi.CG_WORD_OR, 0, capi.CG_WORD_AND, 0, capi.CG_WORD_OR, 0, capi.CG_WORD_OR, 0]
        for rel in rels:
            part = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, n)
            part.scan_shard(cg.Shard(rel))
            g = part.ngroups()
            keys = torch.empty(g, dtype=torch.int64, device="cuda")
            kn = torch.empty(g, dtype=torch.uint8, device="cuda")
            words = torch.empty(g * nw, dtype=torch.int64, device="cuda")
            assert part.export_device(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), g) == g
            final.merge_rows(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), g)
            fr = part.fetch()
            capi.check(L.cg_partial_merge_values(via_values.h, fr["n"], fr["keys"].ctypes.data, fr["key_nulls"].ctypes.data,
                                                 np.ascontiguousarray(fr["sum_hi"]).ctypes.data, np.ascontiguousarray(fr["sum_lo"]).ctypes.data,
                                                 np.ascontiguousarray(fr["count"]).ctypes.data, np.ascontiguousarray(fr["minmax"]).ctypes.data,
                                                 np.ascontiguousarray(fr["fsum"]).ctypes.data))
            part.free()
        for combined in (final, via_values):
            got = {(kk,): per for kk, per in combined.groups().items()}
            st = type("S", (), dict(rows_passed=n, rows_removed_by_filter=0, rows_scanned=n))
            assert_exact(st, got, want, aggs, n)
            combined.free()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _combine_worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.cuda.set_device(rank)
        from citus_b200 import columnar as cg, distributed as cgd
        cg.init(rank)
        cgd.init(rank, world)
        rng = np.random.default_rng(29)
        n = 40_000
        k = rng.integers(0, 2000, n)
        v = rng.integers(-10**9, 10**9, n)
        cols = [k, v, rng.integers(0, 100, n)]
        halves = [slice(0, n // 2), slice(n // 2, n)]
        rel = cg.Relation.write([8, 8, 8], [c[halves[rank]] for c in cols], chunk_row_limit=5000)
        aggs = [cg.count_star(), cg.bit_and(1), cg.bit_or(1), cg.bool_and((2, "<", 98)), cg.bool_or((1, ">", 999_000_000))]
        want = ref.aggregate(cols, None, [], [0], aggs)
        for mode in (1, 0):
            cg.set_option("peer_window", mode)
            for kmin, kmax in ((0, 1999), (0, -1)):
                d = cg.make_desc([], [0], aggs, expected_groups=4096)
                agg = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, n)
                agg.scan_shard(cg.Shard(rel), want_stats=False)
                cgd.combine_partials(agg, dst=0)
                if rank == 0:
                    got = {(kk,): per for kk, per in agg.groups().items()}
                    st = type("S", (), dict(rows_passed=n, rows_removed_by_filter=0, rows_scanned=n))
                    assert_exact(st, got, want, aggs, n)
                agg.free()
                cgd.barrier()
        cgd.destroy()
        out.put((rank, "ok"))
    except Exception:          # noqa
        out.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_two_gpu_combine(cg):
    """cg_comm_combine of bit / bool partials (their words are not all ADD: row gather + merge) over the peer window
    and over NCCL, dense and hash tables"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_combine_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(results) == [(0, "ok"), (1, "ok")], results
