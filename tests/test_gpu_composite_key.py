"""Composite GROUP BY keys (CgScanDesc.composite_key) in the fused scan against the exact reference, on every kernel
family: one to four key columns of every integer-like type (bool, int1, int2, int4, int8, char(1), numeric(12, 2)),
negative values and NULLs in every key column, in the small-domain, direct-indexed and hash table kinds.  The expected
answers come from tests/reference.py, whose groups are keyed by the
tuple of key values with None for NULL -- the shape GpuColumnarAgg.groups() decodes composite codes into."""
import ctypes
import dataclasses
import os
import socket
import traceback

import numpy as np
import pytest

import reference as ref
from test_gpu_bool_bit_agg import assert_exact
from gpu_harness import cg, kernel_family, FAMILIES  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

BPCHAR1, NUMERIC2 = 3, 2 | (2 << 8)
ATTLENS = [1, 1, 2, 4, 8, -1, -1, 8, 8]
TYPES = [0, 0, 0, 0, 0, BPCHAR1, NUMERIC2, 0, 1]
FLOAT_COLS = (8,)
# key columns -> the table kind they give with the aggregates below
GROUPINGS = [([0, 1], "small"), ([2, 3], "dense"), ([5, 0], "dense"), ([1, 2, 3], "dense"), ([4, 3], "hash"), ([6], "hash"),
             ([0, 5, 6, 2], "hash")]


def make_rows(seed, n):
    """bool, int1, int2, int4, int8 (wide values), char(1), numeric(12, 2) (scaled), an int8 and a float8 argument.  NULLs
    in every key column, but only in the second half of the rows: the first half's chunk groups are NULL-free, so the
    NULL-free and the nullable forms of every kernel family both run"""
    rng = np.random.default_rng(seed)
    wide = rng.integers(-2**40, 2**40, 200)
    money = rng.integers(-10**9, 10**9, 50)
    cols = [rng.integers(0, 2, n), rng.integers(-2, 3, n), rng.integers(-300, 301, n), rng.integers(-8, 8, n),
            wide[rng.integers(0, 200, n)], rng.choice([0x41, 0x42, 0x43, 0x5A, 0xE9], n), money[rng.integers(0, 50, n)],
            rng.integers(-10**6, 10**6, n), rng.normal(0, 100, n)]
    nulls = []
    for c in range(len(cols)):
        z = np.zeros(n, bool)
        if c != 7:
            z[n // 2:] = rng.random(n - n // 2) < 0.08
        nulls.append(z)
    return cols, nulls


def write(cg, oracle, cols, nulls):
    t = oracle.Table(ATTLENS, TYPES, stripe_row_limit=4000, chunk_row_limit=1000)
    t.insert(cols, [z.astype(np.uint8) for z in nulls])
    return cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), ATTLENS, TYPES)


_TABLES = {}


def table(cg, oracle, seed=2026, n=20_000):
    if (seed, n) not in _TABLES:
        cols, nulls = make_rows(seed, n)
        _TABLES[(seed, n)] = (write(cg, oracle, cols, nulls), cols, nulls, n)
    return _TABLES[(seed, n)]


_REFERENCE = {}


def reference(cols, nulls, where, group, aggs, key):
    k = (key, repr(where), tuple(group), repr(aggs))
    if k not in _REFERENCE:
        _REFERENCE[k] = ref.aggregate(cols, nulls, where, group, aggs, FLOAT_COLS)
    return _REFERENCE[k]


def composite(cg, rels, where, group, aggs, bounds=None, expected_groups=1 << 15):
    """(descriptor, key bounds, aggregates with proven term bounds, rows) over the union of `rels`"""
    aggs = [dataclasses.replace(a) for a in aggs]
    d0 = cg.make_desc(where, group, aggs, float_cols=FLOAT_COLS)
    union, proven, rows = None, [0] * len(aggs), 0
    for rel in rels:
        kb = cg.relation_key_bounds(rel, d0)
        union = kb if union is None else [(min(a[0], b[0]), max(a[1], b[1])) for a, b in zip(union, kb)]
        _, _, pr, r = cg.relation_bounds(rel, d0)
        proven = [max(x, y) for x, y in zip(proven, pr)]
        rows += r
    for a, b in zip(aggs, proven):
        a.term_abs_bound = b
    bounds = bounds or union
    d = cg.make_desc(where, group, aggs, float_cols=FLOAT_COLS, expected_groups=expected_groups, composite=True, key_bounds=bounds)
    return d, bounds, aggs, max(rows, 1)


def run(cg, rel, where, group, aggs, path="shard", bounds=None, packing=True):
    d, _, aggs, rows = composite(cg, [rel], where, group, aggs, bounds)
    agg = cg.GpuColumnarAgg(d, rel.column_descs(), 0, -1, rows)
    try:
        if not packing:
            agg.set_packing(False)
        if path == "shard":
            shard = cg.Shard(rel)
            st = agg.scan_shard(shard)
            shard.free()
        else:
            st = agg.scan_relation(rel)
        return st, agg.groups(), agg.layout(), aggs
    finally:
        agg.free()


def base_aggs(cg):
    return [cg.count_star(), cg.sum_(7), cg.min_(8, True), cg.max_(3), cg.count(2)]


# --------------------------------------------------------------------------- keys of every width, every table kind
@pytest.mark.parametrize("family", FAMILIES)
def test_keys_of_every_width_in_every_table_kind(cg, oracle, kernel_family, family):
    kernel_family(family)
    rel, cols, nulls, n = table(cg, oracle)
    for i, (group, kind) in enumerate(GROUPINGS):
        for where in ([], ("or", (3, "<", 0), ("and", (1, ">", -2), (7, ">=", 0)))):
            aggs = base_aggs(cg)
            want = reference(cols, nulls, where, group, aggs, "base")
            st, got, layout, _ = run(cg, rel, where, group, aggs, path="shard" if i % 2 == 0 else "e2e")
            assert layout[2] == (kind != "hash"), (group, layout)
            assert len(want.groups) > 1
            assert any(None in key for key in want.groups)
            assert_exact(st, got, want, aggs, n)


@pytest.mark.parametrize("family", FAMILIES)
def test_filter_bool_and_bit_or_over_composite_groups(cg, oracle, kernel_family, family):
    kernel_family(family)
    rel, cols, nulls, n = table(cg, oracle)
    aggs = [cg.count_star(filter=(7, ">", 0)), cg.sum_(7, filter=("or", (3, "<", -4), (2, ">", 100))),
            cg.bool_and((7, ">", -900_000)), cg.bool_or(("and", (3, ">", 5), (1, "=", 0))), cg.bit_or(2), cg.bit_and(3, filter=(0, "=", 1)),
            cg.max_(4, filter=(2, "<>", 7))]
    for group, _ in GROUPINGS:
        where = ("or", (7, "<", 500_000), (2, "=", 0))
        want = reference(cols, nulls, where, group, aggs, "filters")
        st, got, _, _ = run(cg, rel, where, group, aggs)
        assert_exact(st, got, want, aggs, n)


# --------------------------------------------------------------------------- wrong bounds never give a wrong group
@pytest.mark.parametrize("family", FAMILIES)
def test_bounds_narrower_than_the_data_are_einval(cg, oracle, kernel_family, family):
    from citus_b200 import capi
    kernel_family(family)
    rel, cols, nulls, n = table(cg, oracle)
    for group, kind in GROUPINGS:
        _, good, _, _ = composite(cg, [rel], [], group, base_aggs(cg))
        for g in range(len(group)):
            for lo_adj, hi_adj in ((1, 0), (0, -1)):
                bad = list(good)
                bad[g] = (good[g][0] + lo_adj, good[g][1] + hi_adj)
                with pytest.raises(capi.CitusGpuError) as e:
                    run(cg, rel, [], group, base_aggs(cg), bounds=bad)
                assert e.value.code == capi.CG_EINVAL, (group, g, kind)
        # a column bounded as all-NULL while it holds values
        bad = list(good)
        bad[0] = (1, 0)
        with pytest.raises(capi.CitusGpuError) as e:
            run(cg, rel, [], group, base_aggs(cg), bounds=bad)
        assert e.value.code == capi.CG_EINVAL


@pytest.mark.parametrize("family", FAMILIES)
def test_packing_on_and_off_agree(cg, oracle, kernel_family, family):
    kernel_family(family)
    rel, cols, nulls, n = table(cg, oracle)
    aggs = [cg.count_star(), cg.sum_(7)]
    for group, kind in GROUPINGS:
        want = reference(cols, nulls, [], group, aggs, "packing")
        st1, on, _, _ = run(cg, rel, [], group, aggs, packing=True)
        st0, off, _, _ = run(cg, rel, [], group, aggs, packing=False)
        assert on == off
        assert_exact(st1, on, want, aggs, n)


# --------------------------------------------------------------------------- several shards, the combine forms
@pytest.mark.parametrize("family", FAMILIES)
def test_shards_fold_into_one_partial_under_union_bounds(cg, oracle, kernel_family, family):
    from citus_b200 import capi
    kernel_family(family)
    parts = [make_rows(300 + s, 6000) for s in range(3)]
    rels = [write(cg, oracle, c, z) for c, z in parts]
    cols = [np.concatenate([p[0][c] for p in parts]) for c in range(len(ATTLENS))]
    nulls = [np.concatenate([p[1][c] for p in parts]) for c in range(len(ATTLENS))]
    aggs = base_aggs(cg)
    for group, _ in GROUPINGS:
        d, bounds, aggs_b, rows = composite(cg, rels, [], group, aggs)
        agg = cg.GpuColumnarAgg(d, rels[0].column_descs(), 0, -1, rows)
        try:
            for i, rel in enumerate(rels):
                if i == 1:
                    agg.scan_relation(rel)
                else:
                    agg.scan_shard(cg.Shard(rel))
            got = agg.groups()
            # a descriptor with other bounds does not scan into this partial
            own, _, _, _ = composite(cg, rels[:1], [], group, aggs_b)
            if list(own.key_col_min)[:len(group)] != list(d.key_col_min)[:len(group)] or \
                    list(own.key_col_max)[:len(group)] != list(d.key_col_max)[:len(group)]:
                with pytest.raises(capi.CitusGpuError) as e:
                    capi.check(capi.lib().cg_scan_relation(ctypes.byref(rels[0].view), ctypes.byref(own), agg.h, None))
                assert e.value.code == capi.CG_EINVAL
        finally:
            agg.free()
        want = ref.aggregate(cols, nulls, [], group, aggs, FLOAT_COLS)
        assert set(got) == set(want.groups)
        for key, per in want.groups.items():
            assert [g["count"] for g in got[key]] == [w.count for w in per], (group, key)
            assert got[key][1]["sum"] == per[1].sum, (group, key)
            assert per[3].count == 0 or got[key][3]["minmax"] == per[3].max, (group, key)


def test_export_merge_rows_and_encoded_merge_values_round_trip(cg, oracle):
    import torch
    rel, cols, nulls, n = table(cg, oracle)
    aggs = base_aggs(cg)
    for group, _ in GROUPINGS:
        d, _, aggs_b, rows = composite(cg, [rel], [], group, aggs)
        src = cg.GpuColumnarAgg(d, rel.column_descs(), 0, -1, rows)
        via_rows = cg.GpuColumnarAgg(d, rel.column_descs(), 0, -1, rows)
        via_values = cg.GpuColumnarAgg(d, rel.column_descs(), 0, -1, rows)
        try:
            src.scan_shard(cg.Shard(rel))
            want = src.groups()
            ng = src.ngroups()
            nw = src.layout()[0]
            keys = torch.zeros(ng, dtype=torch.int64, device="cuda")
            kn = torch.ones(ng, dtype=torch.uint8, device="cuda")
            words = torch.zeros(ng * nw, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()                                # the fills run on torch's stream, the export on the library's
            got_n = src.export_device(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), ng)
            assert got_n == ng
            assert int(kn.sum()) == 0                               # a composite partial has no NULL key: codes only
            via_rows.merge_rows(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), got_n)
            assert via_rows.groups() == want
            f = src.fetch()
            tuples = cg.group_key_decode(d, f["keys"])
            assert tuples == list(cg.group_key_decode(d, cg.group_key_encode(d, tuples)))
            via_values.merge_values(tuples, None, f["sum_hi"], f["sum_lo"], f["count"], f["minmax"], f["fsum"])
            got = via_values.groups()
            assert set(got) == set(want)
            for key in want:
                for a in range(len(aggs)):
                    assert (got[key][a]["count"], got[key][a]["sum"], got[key][a]["minmax"]) == \
                        (want[key][a]["count"], want[key][a]["sum"], want[key][a]["minmax"]), (group, key, a)
        finally:
            src.free(); via_rows.free(); via_values.free()


@pytest.mark.parametrize("family", FAMILIES)
def test_packed_two_column_form_still_refuses_a_null_key(cg, oracle, kernel_family, family):
    """composite_key = 0 keeps today's behaviour: a NULL in a packed two-column key is CG_EUNSUPPORTED"""
    from citus_b200 import capi
    kernel_family(family)
    rel, cols, nulls, n = table(cg, oracle)
    d = cg.make_desc([], [1, 2], [cg.count_star()])
    kmin, kmax, _, rows = cg.relation_bounds(rel, d)
    agg = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, rows)
    try:
        with pytest.raises(capi.CitusGpuError) as e:
            agg.scan_shard(cg.Shard(rel))
            agg.groups()
        assert e.value.code == capi.CG_EUNSUPPORTED
    finally:
        agg.free()


# --------------------------------------------------------------------------- two GPUs
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.cuda.set_device(rank)
        from citus_b200 import capi, columnar as cg, distributed as cgd
        from oracle import oracle as orc
        orc.build()
        cg.init(rank)
        cgd.init(rank, world)
        parts = [make_rows(700 + r, 8000) for r in range(world)]
        rel = write(cg, orc, *parts[rank])
        cols = [np.concatenate([p[0][c] for p in parts]) for c in range(len(ATTLENS))]
        nulls = [np.concatenate([p[1][c] for p in parts]) for c in range(len(ATTLENS))]
        for pw in (1, 0):
            cg.set_option("peer_window", pw)
            # dense with additive words (reduced in place), and hashed (rows gathered and merged on the root)
            for group, aggs in (([2, 3], [cg.count_star(), cg.sum_(7)]), ([0, 5, 6, 2], [cg.count_star(), cg.sum_(7), cg.max_(3)])):
                d, bounds, aggs_b, rows = composite(cg, [rel], [], group, aggs)
                lo = cgd.allreduce([b[0] for b in bounds], "min")
                hi = cgd.allreduce([b[1] for b in bounds], "max")
                d, _, _, _ = composite(cg, [rel], [], group, aggs_b, bounds=list(zip(lo, hi)))
                agg = cg.GpuColumnarAgg(d, rel.column_descs(), 0, -1, rows * world)
                agg.scan_shard(cg.Shard(rel), want_stats=False)
                cgd.combine_partials(agg, dst=0)
                if rank == 0:
                    want = ref.aggregate(cols, nulls, [], group, aggs, FLOAT_COLS)
                    got = agg.groups()
                    assert set(got) == set(want.groups), (pw, group)
                    for key, per in want.groups.items():
                        assert [g["count"] for g in got[key]] == [w.count for w in per], (pw, group, key)
                        assert got[key][1]["sum"] == per[1].sum, (pw, group, key)
                agg.free()
                # bounds that differ between the ranks but give the same domain: the codes disagree, the combine refuses
                shifted = [(a + rank, b + rank) for a, b in zip(lo, hi)]
                d, _, _, _ = composite(cg, [rel], [], group, aggs_b, bounds=shifted)
                agg = cg.GpuColumnarAgg(d, rel.column_descs(), 0, -1, rows * world)
                try:
                    cgd.combine_partials(agg, dst=0)
                    raise AssertionError("mismatched key codecs were combined")
                except capi.CitusGpuError as e:
                    assert e.code == capi.CG_EINVAL and "do not share one layout" in str(e), str(e)
                agg.free()
        cgd.destroy()
        out.put((rank, "ok"))
    except Exception:          # noqa
        out.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_two_gpu_combine_of_composite_partials():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    from citus_b200 import build
    build.build()
    world = 2
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, out)) for r in range(world)]
    for p in procs:
        p.start()
    results = [out.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(results) == [(0, "ok"), (1, "ok")], results


# --------------------------------------------------------------------------- the table machinery really serves composite keys
@pytest.mark.parametrize("kind", ["dense", "hash"])
def test_packing_engages_and_its_overflow_is_detected(cg, kind):
    """count(*) + a bounded sum share one packed word per group in composite dense and hash tables too: a group that
    receives >= 2^C rows between drains is reported as CG_ERETRY_UNPACKED (so packing was on), and the rescan with
    packing off is exact"""
    from citus_b200 import capi
    rng = np.random.default_rng(31)
    n = 400_000
    k0 = rng.integers(0, 5000, n)
    k1 = rng.integers(-3, 4, n)
    k0[:150_000], k1[:150_000] = 7, 2                           # one hot group: 150 000 rows > 2^16
    if kind == "hash":
        k0 = k0 * (1 << 30)                                     # the same groups over a domain too large to index
    v = rng.integers(-10**9, 10**9, n)
    rel = cg.Relation.write([8, 2, 8], [k0, k1, v])
    aggs = [cg.sum_(2), cg.count_star()]
    d0 = cg.make_desc([], [0, 1], aggs)
    kb = cg.relation_key_bounds(rel, d0)
    _, _, proven, rows = cg.relation_bounds(rel, d0)
    aggs[0].term_abs_bound = proven[0]
    d = cg.make_desc([], [0, 1], aggs, composite=True, key_bounds=kb, expected_groups=1 << 16)
    agg = cg.GpuColumnarAgg(d, rel.column_descs(), 0, -1, rows)
    try:
        assert agg.layout()[2] == (kind == "dense")
        shard = cg.Shard(rel)
        agg.scan_shard(shard, want_stats=False)
        with pytest.raises(capi.CitusGpuError) as e:
            agg.groups()
        assert e.value.code == capi.CG_ERETRY_UNPACKED
        agg.reset()
        agg.set_packing(False)
        agg.scan_shard(shard, want_stats=False)
        got = agg.groups()
    finally:
        agg.free()
    want = ref.aggregate([k0, k1, v], None, [], [0, 1], aggs)
    assert set(got) == set(want.groups)
    for key, per in want.groups.items():
        assert (got[key][0]["sum"], got[key][1]["count"]) == (per[0].sum, per[1].count), key


@pytest.mark.parametrize("family", FAMILIES)
def test_small_composite_domains_run_the_shared_memory_kernels(cg, oracle, kernel_family, family):
    """the small-domain grouping runs the shared-memory kernels: cg_scan_small_kernel for the ahead-of-time family,
    the generated kernel's shared-memory kind (1) for the generated families; the general family is the interpretive
    cg_scan_kernel by definition"""
    import torch
    from test_composite_key_host import compile_check
    kernel_family(family)
    rel, cols, nulls, n = table(cg, oracle)
    group = [g for g, k in GROUPINGS if k == "small"][0]
    aggs = base_aggs(cg)
    d, _, aggs_b, rows = composite(cg, [rel], [], group, aggs)
    if family in ("jit", "jit_always"):
        for nullable in (0, (1 << len(ATTLENS)) - 1):
            rc, kind, _ = compile_check(d, rel.column_descs(), rows=rows, nullable=nullable)
            assert (rc, kind) == (0, 1)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        st, got, _, _ = run(cg, rel, [], group, aggs)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    want_kernel = {"jit": "cg_jit_scan", "jit_always": "cg_jit_scan", "aot": "cg_scan_small_kernel", "general": "cg_scan_kernel"}[family]
    assert any(want_kernel in name for name in names), sorted(names)
    if family == "aot":
        assert not any("cg_scan_kernel" in name for name in names)
    assert_exact(st, got, reference(cols, nulls, [], group, aggs, "base"), aggs, n)


def test_a_null_key_flag_is_refused_by_a_composite_partial(cg, oracle):
    """codes encode their NULLs: a merged row with key_nulls != 0 would land in the unused NULL entry, so it is refused"""
    import torch
    from citus_b200 import capi
    rel, cols, nulls, n = table(cg, oracle)
    d, _, aggs, rows = composite(cg, [rel], [], [2, 3], base_aggs(cg))
    src = cg.GpuColumnarAgg(d, rel.column_descs(), 0, -1, rows)
    dst = cg.GpuColumnarAgg(d, rel.column_descs(), 0, -1, rows)
    try:
        src.scan_shard(cg.Shard(rel))
        f = src.fetch()
        kn = np.zeros(f["n"], np.uint8)
        kn[3] = 1
        with pytest.raises(capi.CitusGpuError) as e:
            dst.merge_values(f["keys"], kn, f["sum_hi"], f["sum_lo"], f["count"], f["minmax"], f["fsum"])
        assert e.value.code == capi.CG_EINVAL
        dst.reset()
        ng, nw = src.ngroups(), src.layout()[0]
        keys = torch.zeros(ng, dtype=torch.int64, device="cuda")
        dkn = torch.zeros(ng, dtype=torch.uint8, device="cuda")
        words = torch.zeros(ng * nw, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()                                    # the fills run on torch's stream, the export on the library's
        src.export_device(keys.data_ptr(), dkn.data_ptr(), words.data_ptr(), ng)
        dkn[5] = 1
        torch.cuda.synchronize()
        with pytest.raises(capi.CitusGpuError) as e:
            dst.merge_rows(keys.data_ptr(), dkn.data_ptr(), words.data_ptr(), ng)
        assert e.value.code == capi.CG_EINVAL
    finally:
        src.free(); dst.free()
