"""var_pop / var_samp / stddev_pop / stddev_samp in the fused scan against the exact reference, on every kernel family.
The GPU keeps the exact state (N, sum(x), sum(x^2)) of CG_AGG_VARIANCE; tests/reference.py computes the same
state from the rows and the final functions from their definition.  Every word is compared exactly, and the final text
through cg_numeric_var_out."""
import dataclasses
import json
import os

import numpy as np
import pytest

import reference as ref
from gpu_harness import cg, kernel_family, FAMILIES  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
NUMERIC2 = 2 | (2 << 8)
VARIANCE = 9


def keyed(d, group_cols, got):
    out = {}
    for k, per in got.items():
        if not group_cols:
            key = ()
        elif d.composite_key:
            key = k
        elif len(group_cols) == 1:
            key = (k,)
        else:
            key = ref.unpack_two_column_key(k)
        out[key] = per
    return out


def run(cg, rels, where, group_cols, aggs, bounds=None, use_bounds=True, force_hash=False, composite=False, e2e=False,
        expected_groups=0):
    """one partial over one or several relations (shards); returns (stats of the last scan, groups keyed like the
    reference, layout).  bounds: term_abs_bound per aggregate (default: cg_relation_bounds of the first relation)"""
    rels = rels if isinstance(rels, list) else [rels]
    aggs = [dataclasses.replace(a) for a in aggs]
    kb = None
    d = cg.make_desc(where, group_cols, aggs, expected_groups=expected_groups)
    if composite:
        kb = [(min(b[0] for b in bs), max(b[1] for b in bs)) for bs in zip(*[cg.relation_key_bounds(r, d) for r in rels])]
        d = cg.make_desc(where, group_cols, aggs, expected_groups=expected_groups, composite=True, key_bounds=kb)
    kmin, kmax, proven, rows = cg.relation_bounds(rels[0], d)
    for r in rels[1:]:
        k2min, k2max, _, rows2 = cg.relation_bounds(r, d)
        kmin, kmax, rows = min(kmin, k2min), max(kmax, k2max), rows + rows2
    for i, a in enumerate(aggs):
        a.term_abs_bound = (bounds[i] if bounds else proven[i]) if use_bounds else 0
    d = cg.make_desc(where, group_cols, aggs, expected_groups=expected_groups, composite=composite, key_bounds=kb)
    if force_hash:
        kmin, kmax = 0, -1
    agg = cg.GpuColumnarAgg(d, rels[0].column_descs(), kmin, kmax, max(rows, 1))
    try:
        for r in rels:
            if e2e:
                if e2e == "dma":
                    r.register()
                try:
                    st = agg.scan_relation(r)
                finally:
                    if e2e == "dma":
                        r.unregister()
            else:
                shard = cg.Shard(r)
                st = agg.scan_shard(shard)
                shard.free()
        got = agg.groups()
        layout = agg.layout()
    finally:
        agg.free()
    return st, keyed(d, group_cols, got), layout


def assert_exact(cg, got, want, aggs, scales=None):
    """every group; per aggregate the count, sum and (variance) sum(x^2), and the four final texts"""
    if () in got and () not in want.groups:
        assert all(g["count"] == 0 for g in got[()])
        return
    assert set(got) == set(want.groups)
    for key, per in want.groups.items():
        for a, (spec, w) in enumerate(zip(aggs, per)):
            g = got[key][a]
            assert g["count"] == w.count, (key, a, g["count"], w.count)
            if spec.kind in (ref.SUM, VARIANCE) and w.count:
                assert g["sum"] == w.sum, (key, a)
            if spec.kind == VARIANCE:
                assert g["sumsq"] == (w.sumsq if w.count else 0), (key, a, g["sumsq"], w.sumsq)
                scale = scales[a] if scales else 0
                for final in range(4):
                    assert cg.numeric_var_out(final, g["count"], g["sum"], g["sumsq"], scale) == \
                        ref.var_out(final, w.count, w.sum, w.sumsq, scale), (key, a, final)


def var_words(nlimbs_sum, qlimbs):
    return nlimbs_sum + qlimbs + 1


# --------------------------------------------------------------------------- data
def mixed(cg, seed=7, n=12_000, stripe_rows=4000, chunk_rows=1000):
    """k1 int2 0..4, k2 int4 0..2 (NOT NULL keys), x int2 / y int4 / z int8 at their types' edges with NULLs (an all-NULL
    chunk in z), kn int2 -1..2 with NULLs (a composite key column)"""
    rng = np.random.default_rng(seed)
    k1, k2 = rng.integers(0, 5, n), rng.integers(0, 3, n)
    x, y, z = rng.integers(-2**15, 2**15, n), rng.integers(-2**31, 2**31, n), rng.integers(-2**62, 2**62, n)
    kn = rng.integers(-1, 3, n)
    x[:2], y[:2], z[:2] = [-2**15, 2**15 - 1], [-2**31, 2**31 - 1], [-2**62, 2**62 - 1]
    cols = [k1, k2, x, y, z, kn]
    nulls = [None, None] + [(rng.random(n) < r).astype(np.uint8) for r in (0.05, 0.0, 0.1, 0.1)]
    nulls[4][chunk_rows:2 * chunk_rows] = 1
    rel = cg.Relation.write([2, 4, 2, 4, 8, 2], cols, nulls, stripe_row_limit=stripe_rows, chunk_row_limit=chunk_rows)
    return rel, cols, nulls


SHAPES = [dict(group_cols=[]), dict(group_cols=[0]), dict(group_cols=[0, 1]), dict(group_cols=[1], force_hash=True, expected_groups=64),
          dict(group_cols=[0, 5], composite=True)]


@pytest.mark.parametrize("family", FAMILIES)
def test_every_key_form_with_nulls_where_and_filter(cg, kernel_family, family):
    kernel_family(family)
    rel, cols, nulls = mixed(cg)
    aggs = [cg.count_star(), cg.variance(2), cg.variance(3, filter=("or", (0, "<", 2), (2, ">", 100))), cg.variance(4),
            cg.sum_(3), cg.variance(2, filter=(5, ">=", 1))]
    for where in ([], [(1, "<", 2)], ("or", (2, ">", 0), (4, "<", 0))):
        for shape in SHAPES:
            want = ref.aggregate(cols, nulls, where, shape["group_cols"], aggs)
            for use_bounds in (True, False):
                _, got, _ = run(cg, rel, where, aggs=aggs, use_bounds=use_bounds, **shape)
                assert_exact(cg, got, want, aggs)


@pytest.mark.parametrize("family", FAMILIES)
def test_one_two_and_four_limb_forms(cg, kernel_family, family):
    """the sum(x^2) form follows term_abs_bound B and max_rows R: one word when B^2 R < 2^63, two limbs when B < 2^32,
    four limbs otherwise -- with x = INT64_MIN (x^2 = 2^126) and INT64_MAX in the four-limb form"""
    kernel_family(family)
    rng = np.random.default_rng(3)
    n = 5000
    k = rng.integers(0, 3, n)
    small = rng.integers(-1000, 1001, n)
    mid = rng.integers(-2**31, 2**31, n)
    wide = rng.integers(INT64_MIN, INT64_MAX, n, endpoint=True)
    wide[:6] = [INT64_MIN, INT64_MAX, INT64_MIN, INT64_MIN, INT64_MAX, -1]
    cols = [k, small, mid, wide]
    rel = cg.Relation.write([8, 8, 8, 8], cols, stripe_row_limit=2000, chunk_row_limit=1000)
    for c, bound, words in ((1, 1000, var_words(1, 1)), (2, 2**31, var_words(1, 2)), (3, 0, var_words(2, 4)),
                            (2, 0, var_words(2, 4)), (2, 2**40, var_words(1, 4))):
        aggs = [cg.count_star(), cg.variance(c)]
        for group in ([], [0]):
            want = ref.aggregate(cols, None, [], group, aggs)
            _, got, layout = run(cg, rel, [], group, aggs, bounds=[0, bound])
            assert layout[0] == 1 + words, (c, bound, layout)
            assert_exact(cg, got, want, aggs)


@pytest.mark.parametrize("family", FAMILIES)
def test_numeric_column_compressed_shards_and_several_shards(cg, oracle, kernel_family, family):
    """numeric(15, 2) values (scaled by 10^2) and int4 values: lz4 and zstd shards, and three shards into one partial"""
    kernel_family(family)
    rng = np.random.default_rng(5)
    parts = []
    for i, comp in enumerate(("lz4", "zstd", "none")):
        n = 4000 + 1000 * i
        m = rng.integers(-10**15 + 1, 10**15, n)
        m[:2] = [10**15 - 1, -10**15 + 1]
        cols = [rng.integers(0, 4, n), m, rng.integers(-2**31, 2**31, n)]
        nulls = [np.zeros(n, np.uint8), (rng.random(n) < 0.05).astype(np.uint8), np.zeros(n, np.uint8)]
        t = oracle.Table([4, -1, 4], [0, NUMERIC2, 0], stripe_row_limit=2000, chunk_row_limit=1000)
        t.insert(cols, nulls)
        numeric = cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), [4, -1, 4], [0, NUMERIC2, 0])
        cg.set_writer_compression(comp)
        try:
            plain = cg.Relation.write([4, 8, 4], cols, nulls, stripe_row_limit=2000, chunk_row_limit=1000)
        finally:
            cg.set_writer_compression("none")
        parts.append((numeric, plain, cols, nulls))
    aggs = [cg.count_star(), cg.variance(1), cg.variance(2, filter=(0, "<>", 1))]
    for rels, cs in (([p[0] for p in parts], None), ([p[1] for p in parts], None)):
        for i, p in enumerate(parts):
            want = ref.aggregate(p[2], p[3], [], [0], aggs)
            _, got, _ = run(cg, rels[i], [], [0], aggs)
            assert_exact(cg, got, want, aggs, scales=[0, 2, 0] if rels[i] is p[0] else None)
        cols = [np.concatenate([p[2][c] for p in parts]) for c in range(3)]
        nulls = [np.concatenate([p[3][c] for p in parts]) for c in range(3)]
        want = ref.aggregate(cols, nulls, [], [0], aggs)
        _, got, _ = run(cg, rels, [], [0], aggs)
        assert_exact(cg, got, want, aggs)


@pytest.mark.parametrize("family", FAMILIES)
def test_scan_relation_end_to_end(cg, kernel_family, family):
    kernel_family(family)
    rel, cols, nulls = mixed(cg, seed=9)
    aggs = [cg.variance(4), cg.count_star(), cg.variance(2, filter=(1, "=", 0))]
    for e2e in ("pageable", "dma"):
        for shape in SHAPES[:3]:
            want = ref.aggregate(cols, nulls, [(0, "<>", 3)], shape["group_cols"], aggs)
            _, got, _ = run(cg, rel, [(0, "<>", 3)], aggs=aggs, e2e=e2e, **shape)
            assert_exact(cg, got, want, aggs)


def test_contestant_golden_on_the_gpu(cg, kernel_family):
    """SELECT avg(rating), stddev_samp(rating) FROM contestant (columnar_query.out): 433.746119785032"""
    with open(os.path.join(HERE, "golden", "variance.json")) as f:
        g = json.load(f)["contestant"]
    rel = cg.Relation.write([4], [np.array(g["rating"])])
    for family in FAMILIES:
        kernel_family(family)
        _, got, _ = run(cg, rel, [], [], [cg.variance(0), cg.sum_(0)])
        v = got[()][0]
        assert cg.numeric_var_out(ref.STDDEV_SAMP, v["count"], v["sum"], v["sumsq"], 0) == g["stddev_samp"]
        assert cg.numeric_div_out(got[()][1]["sum"], 0, got[()][1]["count"]) == g["avg"]


# --------------------------------------------------------------------------- words: export, merge, limits
def test_export_merge_rows_round_trip_and_the_carry_chain(cg):
    """the words of a scanned partial merged twice into another partial give twice its state; merged rows whose limb
    words add past 2^64 in every limb give the exact sum(x^2) (limb l's carry goes to limb l + 1)"""
    import torch
    from citus_b200 import capi
    rng = np.random.default_rng(1)
    n = 3000
    cols = [rng.integers(0, 4, n), rng.integers(INT64_MIN, INT64_MAX, n, endpoint=True)]
    rel = cg.Relation.write([8, 8], cols)
    aggs = [cg.variance(1), cg.count_star()]
    d = cg.make_desc([], [0], aggs)
    a = cg.GpuColumnarAgg(d, rel.column_descs(), 0, 3, n)
    b = cg.GpuColumnarAgg(d, rel.column_descs(), 0, 3, 4 * n)
    try:
        shard = cg.Shard(rel)
        a.scan_shard(shard)
        shard.free()
        nw, ops, _, _ = a.layout()
        assert nw == 1 + var_words(2, 4) and set(ops) == {capi.CG_WORD_ADD}
        keys = torch.zeros(8, dtype=torch.int64, device="cuda")
        kn = torch.zeros(8, dtype=torch.uint8, device="cuda")
        words = torch.zeros(8 * nw, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()                   # the fills run on torch's stream, the library's kernels on its own
        rows = a.export_device(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), 8)
        assert rows == 4
        b.merge_rows(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), rows)
        b.merge_rows(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), rows)
        ga, gb = a.groups(), b.groups()
        want = ref.aggregate(cols, None, [], [0], aggs)
        assert_exact(cg, {(k,): v for k, v in ga.items()}, want, aggs)
        for k in ga:
            assert gb[k][0]["count"] == 2 * ga[k][0]["count"] and gb[k][0]["sum"] == 2 * ga[k][0]["sum"]
            assert gb[k][0]["sumsq"] == 2 * ga[k][0]["sumsq"]
        # hand-made rows: words [rows, sum lo, sum hi, q0, q1, q2, q3, NULL inputs]
        top = 2**64 - 1
        hand = [[3, top - 4, 7, top - 2, top - 6, top, 2**40, 0], [5, 2**63 + 9, -3, top, top, top - 1, 5, 1],
                [2, top, 2**20, 2**63, top - 3, top, 2**50, 0]]
        c = cg.GpuColumnarAgg(d, rel.column_descs(), 0, 3, 0)
        try:
            t = torch.tensor([[w - 2**64 if w >= 2**63 else w for w in r] for r in hand], dtype=torch.int64, device="cuda")
            k3 = torch.full((3,), 1, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            c.merge_rows(k3.data_ptr(), kn.data_ptr(), t.data_ptr(), 3)
            g = c.groups()[1]
            assert g[0]["count"] == sum(r[0] - r[7] for r in hand) and g[1]["count"] == 10
            assert g[0]["sum"] == sum(r[1] + (r[2] << 32) for r in hand)
            assert g[0]["sumsq"] == sum(r[3] + (r[4] << 32) + (r[5] << 64) + (r[6] << 96) for r in hand)
            assert all(sum(r[l] for r in hand) >= 2**64 for l in (3, 4, 5))
        finally:
            c.free()
    finally:
        a.free()
        b.free()


def test_groups_of_2_32_rows_and_host_row_merges_are_refused(cg):
    import torch
    from citus_b200 import capi
    rel = cg.Relation.write([8, 8], [np.zeros(1, np.int64), np.zeros(1, np.int64)])
    # (bound, max_rows) -> (sum(x) words, sum(x^2) words).  The last case refuses through the sum(x^2) limbs alone: its
    # sum(x) is one word (2^31 * 1000 < 2^63), its sum(x^2) two limbs (2^62 * 1000 >= 2^63)
    for bound, max_rows, limbs in ((0, 1 << 62, (2, 4)), (1000, 1 << 62, (2, 2)), (2**31, 1000, (1, 2))):
        aggs = [dataclasses.replace(cg.variance(1), term_abs_bound=bound), cg.count_star()]
        d = cg.make_desc([], [0], aggs)
        p = cg.GpuColumnarAgg(d, rel.column_descs(), 0, 3, max_rows)
        try:
            nw, _, _, _ = p.layout()
            assert nw == 1 + var_words(*limbs)
            keys = torch.full((1,), 2, dtype=torch.int64, device="cuda")
            kn = torch.zeros(1, dtype=torch.uint8, device="cuda")
            big = torch.zeros((1, nw), dtype=torch.int64, device="cuda")
            big[0, 0] = 2**32
            torch.cuda.synchronize()
            p.merge_rows(keys.data_ptr(), kn.data_ptr(), big.data_ptr(), 1)
            with pytest.raises(capi.CitusGpuError) as e:
                p.groups()
            assert e.value.code == capi.CG_EUNSUPPORTED
            with pytest.raises(capi.CitusGpuError) as e:
                p.merge_values([1], [0], [0, 0], [0, 0], [1, 1], [0, 0], [0.0, 0.0])
            assert e.value.code == capi.CG_EUNSUPPORTED
        finally:
            p.free()


@pytest.mark.parametrize("family", FAMILIES)
def test_bound_violated_by_the_data_is_an_error(cg, kernel_family, family):
    """a row over term_abs_bound fails the scan with CG_EINVAL in every sum(x^2) form: one word, two limbs (B < 2^32,
    B^2 R >= 2^63) and four limbs (B >= 2^32); a bound the data respects gives the exact state"""
    from citus_b200 import capi
    kernel_family(family)
    n = 3000
    i = np.arange(n)
    sign = np.where(i % 2 == 0, 1, -1)
    cols = [i % 3, i - 1500, sign * (2**32 + i), sign * (2**41 - i)]
    rel = cg.Relation.write([8, 8, 8, 8], cols)
    # (column, violated bound, respected bound, sum(x) words, sum(x^2) words)
    cases = ((1, 10, 1500, 1, 1), (1, 1400, 1500, 1, 1), (2, 2**32 - 1, None, 1, 2), (3, 2**40, 2**41, 1, 4))
    for group in ([], [0]):
        kmin, kmax = (0, 2) if group else (0, -1)
        for c, bad, good, sl, ql in cases:
            aggs = [dataclasses.replace(cg.variance(c), term_abs_bound=bad), cg.count_star()]
            p = cg.GpuColumnarAgg(cg.make_desc([], group, aggs), rel.column_descs(), kmin, kmax, n)
            try:
                assert p.layout()[0] == 1 + var_words(sl, ql), (c, bad)
                with pytest.raises(capi.CitusGpuError) as e:
                    shard = cg.Shard(rel)
                    try:
                        p.scan_shard(shard)
                    finally:
                        shard.free()
                    p.groups()
                assert e.value.code == capi.CG_EINVAL, (c, bad)
            finally:
                p.free()
            if good is None:
                continue
            aggs = [cg.variance(c), cg.count_star()]
            _, got, layout = run(cg, rel, [], group, aggs, bounds=[good, 0])
            assert layout[0] == 1 + var_words(sl, ql)
            assert_exact(cg, got, ref.aggregate(cols, None, [], group, aggs), aggs)
