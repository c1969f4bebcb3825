"""GPU parity tests: the CUDA path (through the C-ABI) against the CPU oracle on the same
inputs, and against the reference's golden vectors.  Bit-exact for COUNT / integer SUM /
MIN / MAX / counters / partition indexes; float SUM within the error bound of any summation
order around the exact sum (tests/reference.py), or 1e-12 relative where only the oracle's
answer is at hand."""
import ctypes as C
import datetime

import numpy as np
import pytest

import reference as ref
from gpu_harness import cg, kernel_family  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

FLOAT_RTOL = 1e-12


def pgdate(s):
    y, m, d = map(int, s.split("-"))
    return (datetime.date(y, m, d) - datetime.date(2000, 1, 1)).days


def oracle_table(oracle, rel, chunk_row_limit=10000):
    descs = rel.column_descs()
    return oracle.Table.attach(rel.pages(), rel.stripes_bytes(), rel.nodes_bytes(), [l for l, _ in descs],
                               [t for _, t in descs], chunk_row_limit=chunk_row_limit)


def to_oracle_aggs(oracle, aggs):
    return [oracle.Agg(a.kind, list(a.factors), a.is_float) for a in aggs]


def assert_same_groups(got, want, aggs, float_rtol=FLOAT_RTOL, float_sum_ok=None):
    """float_sum_ok(key, aggregate, got): the reference's error bound for a float sum; else float_rtol to the oracle's"""
    assert set(got.keys()) == set(want.keys())
    for k in want:
        for a, spec in enumerate(aggs):
            g, w = got[k][a], want[k][a]
            kind = spec.kind
            if kind in (0, 1):                                  # count(*), count(x)
                assert g["count"] == w["count"], (k, a)
            elif kind == 2:                                     # sum
                assert g["count"] == w["count"], (k, a)
                if w["count"] == 0:
                    continue
                if spec.is_float and float_sum_ok is not None:
                    assert float_sum_ok(k, a, g["fsum"]), (k, a, g["fsum"], w["fsum"])
                elif spec.is_float:
                    assert g["fsum"] == pytest.approx(w["fsum"], rel=float_rtol, abs=1e-300), (k, a)
                else:
                    assert g["sum"] == w["sum"], (k, a)
            else:                                               # min / max
                assert g["count"] == w["count"], (k, a)
                if w["count"] == 0:
                    continue
                if spec.is_float:
                    got_f = np.int64(g["minmax"]).view(np.float64)
                    assert got_f == (w["fmin"] if kind == 3 else w["fmax"]), (k, a)
                else:
                    assert g["minmax"] == (w["min"] if kind == 3 else w["max"]), (k, a)


def run_both(cg, oracle, rel, quals=(), group_cols=(), aggs=(), chunk_row_limit=10000, force_hash=False,
             pushdown=True, float_cols=(), use_bounds=True, e2e=False, expected_groups=0):
    d = cg.make_desc(quals, group_cols, aggs, qual_pushdown=pushdown, float_cols=float_cols,
                     expected_groups=expected_groups)
    kmin, kmax, bounds, rows = cg.relation_bounds(rel, d)
    if use_bounds:
        for i, a in enumerate(aggs):
            a.term_abs_bound = bounds[i]
        d = cg.make_desc(quals, group_cols, aggs, qual_pushdown=pushdown, float_cols=float_cols,
                         expected_groups=expected_groups)
    if force_hash:
        kmin, kmax = 0, -1
    agg = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, max(rows, 1))
    if e2e:
        if e2e == "dma":
            rel.register()                       # pinned pages: copy-engine de-framing + GPU realign
        st = agg.scan_relation(rel)
        if e2e == "dma":
            assert st.h2d_bytes > 0
            rel.unregister()
    else:
        shard = cg.Shard(rel)
        st = agg.scan_shard(shard)
        shard.free()
    t = oracle_table(oracle, rel, chunk_row_limit)
    is_tree = isinstance(quals, tuple) and len(quals) > 0 and quals[0] in ("and", "or")
    r = t.scan(quals if is_tree else list(quals), list(group_cols), to_oracle_aggs(oracle, aggs), qual_pushdown=pushdown)
    assert st.rows_scanned == r.rows_scanned
    assert st.rows_removed_by_filter == r.rows_removed_by_filter
    assert st.chunk_groups_filtered == r.chunk_groups_filtered
    assert st.rows_passed == r.rows_passed
    got = agg.groups()
    want = r.groups()
    if not group_cols:
        want = {0: want.get(0, [dict(sum=0, count=0, min=0, max=0, fsum=0.0, fmin=0.0, fmax=0.0)] * len(aggs))}
        got = {0: list(got.values())[0]}
    assert_same_groups(got, want, aggs, float_sum_ok=reference_float_sums(t, quals, group_cols, aggs, float_cols))
    agg.free()
    return st, got


def reference_float_sums(t, quals, group_cols, aggs, float_cols):
    """float sums checked against the exact reference over the decoded relation (None: the query has none)"""
    if not any(a.kind == 2 and a.is_float for a in aggs):
        return None
    vals, nulls = t.decode_all()
    want = ref.aggregate(vals, nulls, quals, group_cols, aggs, float_cols).groups

    def ok(key, a, got):
        if not group_cols:
            rk = ()
        elif len(group_cols) == 1:
            rk = (key,)
        else:
            rk = ref.unpack_two_column_key(key)
        return want[rk][a].float_sum_ok(got)
    return ok


# --------------------------------------------------------------------------- C1 shape
@pytest.mark.parametrize("sorted_b", [False, True])
def test_c1_sum_where_four_shards(cg, oracle, sorted_b):
    """BASELINE config 1 at 1/10 scale: t(a,b,c,d int8) hash-distributed on d into 4 shards,
    SELECT sum(a) WHERE b < k; workers produce partial sums, the coordinator sums them."""
    n = 1_000_000
    rng = np.random.default_rng(20260921)
    a = rng.integers(-2**31, 2**31, n)
    b = rng.integers(0, 10**6, n)
    if sorted_b:
        b = np.sort(b)
    c = rng.integers(-2**62, 2**62, n)
    d = np.arange(n)
    mins, maxs = oracle.synthetic_intervals(4)
    shard_of, _ = oracle.partition_rows(d, None, 8, "h", mins, maxs)
    aggs = [cg.sum_(0), cg.count_star()]
    total = 0
    total_cnt = 0
    want_total = 0
    for s in range(4):
        sel = shard_of == s
        rel = cg.Relation.write([8, 8, 8, 8], [a[sel], b[sel], c[sel], d[sel]])
        st, got = run_both(cg, oracle, rel, quals=[(1, "<", 250000)], aggs=aggs)
        if sorted_b:
            assert st.chunk_groups_filtered > 0
        total += got[0][0]["sum"]
        total_cnt += got[0][1]["count"]
        want_total += int(a[sel][b[sel] < 250000].sum())
    assert total == want_total == int(a[b < 250000].sum())
    assert total_cnt == int((b < 250000).sum())


def test_plain_aggregate_int128_and_empty_input(cg, oracle):
    big = np.full(5000, 2**62, dtype=np.int64)
    rel = cg.Relation.write([8, 8], [big, np.arange(5000)], chunk_row_limit=1000)
    st, got = run_both(cg, oracle, rel, aggs=[cg.sum_(0), cg.min_(0), cg.max_(1)], chunk_row_limit=1000)
    assert got[0][0]["sum"] == 5000 * 2**62
    st, got = run_both(cg, oracle, rel, quals=[(1, "<", 0)], aggs=[cg.sum_(0), cg.count_star(), cg.count(0)],
                       chunk_row_limit=1000)
    assert got[0][0]["count"] == 0 and got[0][1]["count"] == 0       # sum over no rows is NULL
    rel = cg.Relation.write([8], [np.zeros(0, np.int64)])
    d = cg.make_desc(aggs=[cg.count_star(), cg.sum_(0)])
    agg = cg.GpuColumnarAgg(d, rel.column_descs())
    st = agg.scan_shard(cg.Shard(rel))
    assert st.rows_scanned == 0
    g = agg.groups()
    assert list(g.values())[0][0]["count"] == 0


# --------------------------------------------------------------------------- C2 shape
@pytest.mark.parametrize("force_hash", [False, True])
@pytest.mark.parametrize("null_ppm", [0, 50000])
def test_c2_filter_group_by(cg, oracle, force_hash, null_ppm):
    """BASELINE config 2 scaled down: 8 int8 columns, SELECT key, sum(v), count(*) WHERE f < 50 GROUP BY key"""
    cols = [(8, 0, 0, 5000, 0), (8, 0, 0, 100, 0), (8, 0, -10**9, 10**9, null_ppm)] + [(8, 0, 0, 1 << 40, 0)] * 5
    rel = cg.Relation.generate(cols, 345_678, seed=20260922)
    run_both(cg, oracle, rel, quals=[(1, "<", 50)], group_cols=[0], aggs=[cg.sum_(2), cg.count_star()],
             force_hash=force_hash, expected_groups=5000)
    # same through the end-to-end call on host buffers
    run_both(cg, oracle, rel, quals=[(1, "<", 50)], group_cols=[0], aggs=[cg.sum_(2), cg.count_star()],
             force_hash=force_hash, expected_groups=5000, e2e=True)
    run_both(cg, oracle, rel, quals=[(1, "<", 50)], group_cols=[0], aggs=[cg.sum_(2), cg.count_star()],
             force_hash=force_hash, expected_groups=5000, e2e="dma")


def test_group_by_wide_keys_null_keys_and_two_limb_sums(cg, oracle):
    rng = np.random.default_rng(4)
    n = 200_000
    pool = rng.integers(-2**63, 2**63 - 1, 3000)
    pool[0] = -2**63                                            # collides with the table's EMPTY sentinel
    key = pool[rng.integers(0, 3000, n)]
    keyn = (rng.random(n) < 0.01).astype(np.uint8)
    v = rng.integers(-2**62, 2**62, n)                          # sums overflow int64: needs the two-word form
    vn = (rng.random(n) < 0.3).astype(np.uint8)
    rel = cg.Relation.write([8, 8], [key, v], [keyn, vn], stripe_row_limit=50000, chunk_row_limit=7000)
    run_both(cg, oracle, rel, group_cols=[0], chunk_row_limit=7000, expected_groups=4000,
             aggs=[cg.sum_(1), cg.count(1), cg.count_star(), cg.min_(1), cg.max_(1)])


def test_hash_table_full_is_reported(cg):
    from citus_b200 import capi
    n = 100_000
    rel = cg.Relation.write([8], [np.arange(n) * 7919])
    d = cg.make_desc(group_cols=[0], aggs=[cg.count_star()], expected_groups=100)
    agg = cg.GpuColumnarAgg(d, rel.column_descs())                # 1024 slots for 100000 groups
    with pytest.raises(capi.CitusGpuError) as e:
        agg.scan_shard(cg.Shard(rel))
        agg.ngroups()
    assert e.value.code == capi.CG_ETABLEFULL


# --------------------------------------------------------------------------- goldens through the GPU
def _filter_quals(where):
    where = where.replace("WHERE", "").strip()
    if not where:
        return []
    if "BETWEEN" in where:
        lo, hi = where.split("BETWEEN")[1].split("AND")
        return [(0, ">=", int(lo)), (0, "<=", int(hi))]
    col, op, k = where.split()
    return [(0, op, int(k))]


def test_chunk_filtering_goldens(cg, oracle, expected):
    one = np.arange(1, 10001)
    rel1 = cg.Relation.write([4], [one], stripe_row_limit=2000, chunk_row_limit=1000)
    for where, want in expected["chunk_filtering"][:9]:
        st, _ = run_both(cg, oracle, rel1, quals=_filter_quals(where), aggs=[cg.count_star()], chunk_row_limit=1000)
        assert st.rows_removed_by_filter == want, where
    # the second INSERT starts a new stripe sequence: two images of 5 stripes each scanned into one partial
    for where, want in expected["chunk_filtering"][9:]:
        d = cg.make_desc(_filter_quals(where), aggs=[cg.count_star()])
        agg = cg.GpuColumnarAgg(d, rel1.column_descs())
        removed = 0
        for _ in range(2):
            removed += agg.scan_relation(rel1).rows_removed_by_filter
        assert removed == want, where
    for case in expected["simple_chunk_filtering"]:
        rel = cg.Relation.write([4], [np.arange(0, case["max"] + 1)])
        st, got = run_both(cg, oracle, rel, quals=[(0, ">", case["gt"])], aggs=[cg.count_star()])
        assert (st.chunk_groups_filtered, st.rows_removed_by_filter, got[0][0]["count"]) == \
            (case["groups_removed"], case["rows_removed"], case["actual_rows"])
    st, _ = run_both(cg, oracle, rel, quals=[(0, ">", 123456)], aggs=[cg.count_star()], pushdown=False)
    assert st.chunk_groups_filtered == 0


def _lineitem_rels(cg, oracle, li):
    mins, maxs = oracle.synthetic_intervals(2)
    idx, _ = oracle.partition_rows(li["l_orderkey"], None, 8, "h", mins, maxs)
    cols = ["l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus",
            "l_shipdate", "l_suppkey"]
    return [cg.Relation.write([8, 8, 8, 8, 1, 1, 4, 4], [li[c][idx == s] for c in cols],
                              stripe_row_limit=2000, chunk_row_limit=1000) for s in range(2)]


def test_tpch_q6_golden(cg, oracle, expected, lineitem):
    quals = [(6, ">=", pgdate("1994-01-01")), (6, "<", pgdate("1995-01-01")), (2, ">=", 5), (2, "<=", 7), (0, "<", 2400)]
    aggs = [cg.Agg(2, [(1, 0, 1), (2, 0, 1)])]
    total = 0
    for rel in _lineitem_rels(cg, oracle, lineitem):
        _, got = run_both(cg, oracle, rel, quals=quals, aggs=aggs, chunk_row_limit=1000)
        total += got[0][0]["sum"]                                # coordinator: sum(partial sums)
    assert cg.numeric_out(total, 4) == expected["tpch_q6"]


def test_tpch_q1_golden(cg, oracle, expected, lineitem):
    quals = [(6, "<=", pgdate("1998-09-02"))]
    aggs = [cg.sum_(0), cg.sum_(1), cg.Agg(2, [(1, 0, 1), (2, 100, -1)]),
            cg.Agg(2, [(1, 0, 1), (2, 100, -1), (3, 100, 1)]), cg.sum_(2), cg.count_star()]
    merged = {}
    for rel in _lineitem_rels(cg, oracle, lineitem):
        _, got = run_both(cg, oracle, rel, quals=quals, group_cols=[4, 5], aggs=aggs, chunk_row_limit=1000,
                          expected_groups=16)
        for k, per in got.items():
            acc = merged.setdefault(k, [dict(sum=0, count=0) for _ in aggs])
            for a in range(len(aggs)):
                acc[a]["sum"] += per[a]["sum"]
                acc[a]["count"] += per[a]["count"]
    rows = []
    for key, v in sorted(merged.items(), key=lambda kv: (kv[0] & 0xffffffff, kv[0] >> 32)):
        rows.append([chr(key & 0xff), chr((key >> 32) & 0xff),
                     cg.numeric_out(v[0]["sum"], 2), cg.numeric_out(v[1]["sum"], 2),
                     cg.numeric_out(v[2]["sum"], 4), cg.numeric_out(v[3]["sum"], 6),
                     cg.numeric_div_out(v[0]["sum"], 2, v[0]["count"]),
                     cg.numeric_div_out(v[1]["sum"], 2, v[1]["count"]),
                     cg.numeric_div_out(v[4]["sum"], 2, v[4]["count"]), str(v[5]["count"])])
    assert rows == expected["tpch_q1"]


def test_sum_int4_and_float_goldens(cg, oracle, expected, lineitem):
    total = 0
    for rel in _lineitem_rels(cg, oracle, lineitem):
        _, got = run_both(cg, oracle, rel, aggs=[cg.sum_(7)], chunk_row_limit=1000)
        total += got[0][0]["sum"]
    assert str(total) == expected["sum_l_suppkey"]
    f = np.array([float(r[0]) for r in expected["agg_type_data"]])
    dd = np.array([float(r[1]) for r in expected["agg_type_data"]])
    rel = cg.Relation.write([4, 8], [f, dd], type_classes=[1, 1])
    for col, exp in ((0, expected["agg_type_float"]), (1, expected["agg_type_double"])):
        aggs = [cg.min_(col, True), cg.max_(col, True), cg.sum_(col, True), cg.count(col)]
        _, got = run_both(cg, oracle, rel, aggs=aggs, float_cols=(0, 1))
        g = got[0]
        assert np.int64(g[0]["minmax"]).view(np.float64) == pytest.approx(float(exp[0]), rel=1e-12)
        assert np.int64(g[1]["minmax"]).view(np.float64) == pytest.approx(float(exp[1]), rel=1e-12)
        assert g[2]["fsum"] == pytest.approx(float(exp[2]), rel=1e-12)
        assert g[3]["count"] == int(exp[3])


# --------------------------------------------------------------------------- types, NULLs, ragged shapes
def test_mixed_widths_with_nulls(cg, oracle):
    rng = np.random.default_rng(8)
    n = 123_457
    c8 = rng.integers(-2**50, 2**50, n)
    c4 = rng.integers(-2**31, 2**31, n)
    c2 = rng.integers(-2**15, 2**15, n)
    c1 = rng.integers(-128, 128, n)
    f8 = rng.normal(size=n)
    f4 = rng.normal(size=n).astype(np.float32).astype(np.float64)
    nulls = [(rng.random(n) < p).astype(np.uint8) for p in (0.1, 0.5, 0.0, 0.9, 0.2, 0.05)]
    nulls[2] = None
    nulls[0][20000:31000] = 1                                   # a chunk group that is entirely NULL
    rel = cg.Relation.write([8, 4, 2, 1, 8, 4], [c8, c4, c2, c1, f8, f4], nulls, type_classes=[0, 0, 0, 0, 1, 1])
    aggs = [cg.sum_(0), cg.min_(1), cg.max_(1), cg.sum_(3), cg.count(3), cg.sum_(4, True), cg.min_(5, True), cg.max_(4, True)]
    run_both(cg, oracle, rel, quals=[(2, ">", -20000), (4, "<", 1.5)], aggs=aggs, float_cols=(4, 5))
    run_both(cg, oracle, rel, quals=[(5, ">=", -0.25)], group_cols=[3], aggs=aggs[:5] + [cg.count_star()], float_cols=(4, 5))
    run_both(cg, oracle, rel, quals=[(1, "<>", 0)], group_cols=[3], aggs=[cg.count_star(), cg.sum_(1)],
             float_cols=(4, 5), force_hash=True, expected_groups=300)
    # odd-length exists bitmaps put every value stream at an odd byte offset: the DMA path's realign kernel
    run_both(cg, oracle, rel, quals=[(2, ">", -20000), (4, "<", 1.5)], aggs=aggs, float_cols=(4, 5), e2e="dma")
    sorted_rel = cg.Relation.write([8, 4], [np.sort(c8), c4], [None, nulls[1]], stripe_row_limit=20000, chunk_row_limit=1111)
    run_both(cg, oracle, sorted_rel, quals=[(0, ">", 0)], group_cols=[], aggs=[cg.count_star(), cg.sum_(1), cg.min_(0)],
             chunk_row_limit=1111, e2e="dma")                   # chunk-group skipping + DMA spans


def test_ragged_chunks_and_max_chunk_size(cg, oracle):
    rng = np.random.default_rng(12)
    for n, stripe, chunk in ((1, 1000, 1000), (999, 1000, 1000), (1001, 1000, 1000), (250_001, 200_000, 100_000)):
        a = rng.integers(-1000, 1000, n)
        b = rng.integers(0, 10, n)
        nb = (rng.random(n) < 0.3).astype(np.uint8)
        rel = cg.Relation.write([8, 8], [a, b], [None, nb], stripe_row_limit=stripe, chunk_row_limit=chunk)
        run_both(cg, oracle, rel, quals=[(0, ">=", -500)], group_cols=[1], aggs=[cg.count_star(), cg.sum_(0)],
                 chunk_row_limit=chunk)
        run_both(cg, oracle, rel, aggs=[cg.count_star(), cg.sum_(0), cg.count(1)], chunk_row_limit=chunk, e2e=True)
        run_both(cg, oracle, rel, quals=[(0, "<", 900)], group_cols=[1], aggs=[cg.count_star(), cg.sum_(0)],
                 chunk_row_limit=chunk, e2e="dma")


# --------------------------------------------------------------------------- compressed chunks (K7)
def _compressed_relation(cg, oracle, comp, n, seed, stripe=150000, chunk=10000):
    """a table written by the oracle's writer (columnar_writer.c:590-654) with lz4 / pglz value streams:
    long overlapping matches, short matches, long literal runs, NULLs, narrow columns"""
    rng = np.random.default_rng(seed)
    cols = [
        (np.arange(n) % 7, 8, None),                                   # one long match with overlap
        (rng.integers(0, 100, n), 8, None),                            # short sequences
        (rng.integers(-2**62, 2**62, n), 8, None),                     # incompressible: lz4 = literal runs, pglz = stored raw
        (rng.integers(-10**9, 10**9, n), 8, (rng.random(n) < 0.1)),    # NULLs: the stream holds only non-NULL values
        (rng.integers(0, 20000, n) // 100, 4, None),
        (rng.integers(0, 3, n), 2, (rng.random(n) < 0.5)),
        (np.repeat(rng.integers(0, 100, (n + 499) // 500), 500)[:n], 1, None),
    ]
    t = oracle.Table([c[1] for c in cols], stripe_row_limit=stripe, chunk_row_limit=chunk, compression=comp)
    t.insert([c[0] for c in cols], [None if c[2] is None else c[2].astype(np.uint8) for c in cols])
    rel = cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), [c[1] for c in cols])
    kinds = {nd.compression_type for nd in t.nodes()}
    return t, rel, kinds


@pytest.fixture
def lz4_kernel(cg, request):
    """"lanes" = a lane per stream (cg_lz4_lane_kernel), "groups" = eight lanes per stream (cg_decompress_kernel)"""
    cg.set_option("lz4_lanes", {"lanes": 1, "groups": 0, "auto": 2}[request.param])
    yield request.param
    cg.set_option("lz4_lanes", -1)          # back to the library's default


@pytest.mark.parametrize("path", ["shard", "e2e", "dma"])
@pytest.mark.parametrize("comp,lz4_kernel", [("lz4", "lanes"), ("lz4", "groups"), ("lz4", "auto"), ("pglz", "auto"), ("zstd", "auto")],
                         indirect=["lz4_kernel"])
def test_compressed_chunks(cg, oracle, comp, path, lz4_kernel):
    if comp == "lz4" and not oracle.lib().orc_have_lz4():
        pytest.skip("liblz4 missing")
    if comp == "zstd" and not oracle.lib().orc_have_zstd():
        pytest.skip("libzstd missing")
    code = {"lz4": oracle.COMP_LZ4, "pglz": oracle.COMP_PGLZ, "zstd": oracle.COMP_ZSTD}[comp]
    for n, stripe, chunk in ((123_457, 50_000, 10_000), (2_001, 1_000, 1_000)):
        t, rel, kinds = _compressed_relation(cg, oracle, code, n, seed=n, stripe=stripe, chunk=chunk)
        assert code in kinds
        if comp == "pglz":
            assert oracle.COMP_NONE in kinds        # the incompressible column is stored raw: mixed relation
        e2e = {"shard": False, "e2e": True, "dma": "dma"}[path]
        run_both(cg, oracle, rel, quals=[(1, "<", 50)], group_cols=[0],
                 aggs=[cg.count_star(), cg.sum_(2), cg.sum_(3), cg.count(3), cg.min_(4), cg.max_(6)],
                 chunk_row_limit=chunk, e2e=e2e)
        run_both(cg, oracle, rel, quals=[(4, ">=", 20), (6, "<", 90)], group_cols=[5],
                 aggs=[cg.count_star(), cg.sum_(1), cg.sum_(6)], chunk_row_limit=chunk, e2e=e2e)
        run_both(cg, oracle, rel, aggs=[cg.count_star(), cg.sum_(2), cg.count(5), cg.sum_(0)], chunk_row_limit=chunk, e2e=e2e)


@pytest.mark.parametrize("lz4_kernel", ["lanes", "groups"], indirect=True)
def test_lz4_matches_beyond_the_window(cg, oracle, lz4_kernel):
    """value streams whose matches reach back 1.6 KB, 40 KB and (int2) 8 KB -- beyond the 2 KB windows of both
    LZ4 decoders -- next to streams of one long overlapping match"""
    if not oracle.lib().orc_have_lz4():
        pytest.skip("liblz4 missing")
    rng = np.random.default_rng(11)
    n = 70_001
    base200, base5000 = rng.integers(-2**40, 2**40, 200), rng.integers(-2**40, 2**40, 5000)
    cols = [
        (base200[np.arange(n) % 200], 8, None),                          # period 1600 bytes (inside the window)
        (base5000[np.arange(n) % 255], 8, None),                         # period 2040 bytes (just beyond the reach of 2000)
        (base5000[np.arange(n) % 5000], 8, None),                        # period 40000 bytes
        (rng.integers(-30000, 30000, 4_000).astype(np.int64)[np.arange(n) % 4_000], 2, None),     # period 8000 bytes
        (np.zeros(n, np.int64), 8, None),                                # one match over the whole stream
        (rng.integers(0, 50, n), 8, (rng.random(n) < 0.3)),
    ]
    cols = cols[:1] + cols[2:] + cols[1:2]          # the extra column goes last: the queries below address columns 0..4
    t = oracle.Table([c[1] for c in cols], stripe_row_limit=30_000, chunk_row_limit=10_000, compression=oracle.COMP_LZ4)
    t.insert([c[0] for c in cols], [None if c[2] is None else c[2].astype(np.uint8) for c in cols])
    rel = cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), [c[1] for c in cols])
    for e2e in (False, "dma"):
        run_both(cg, oracle, rel, quals=[(4, "<", 25)], group_cols=[4],
                 aggs=[cg.count_star(), cg.sum_(0), cg.sum_(1), cg.sum_(2), cg.sum_(3), cg.min_(1), cg.max_(0)],
                 chunk_row_limit=10_000, e2e=e2e)
        run_both(cg, oracle, rel, aggs=[cg.count_star(), cg.sum_(0), cg.sum_(1), cg.sum_(2), cg.count(4), cg.sum_(5)], chunk_row_limit=10_000, e2e=e2e)


@pytest.mark.parametrize("comp,lz4_kernel", [("lz4", "lanes"), ("lz4", "groups"), ("pglz", "lanes"), ("zstd", "lanes")],
                         indirect=["lz4_kernel"])
def test_corrupt_compressed_stream_is_reported(cg, oracle, comp, lz4_kernel):
    from citus_b200 import capi
    if comp == "lz4" and not oracle.lib().orc_have_lz4():
        pytest.skip("liblz4 missing")
    if comp == "zstd" and not oracle.lib().orc_have_zstd():
        pytest.skip("libzstd missing")
    code = {"lz4": oracle.COMP_LZ4, "pglz": oracle.COMP_PGLZ, "zstd": oracle.COMP_ZSTD}[comp]
    t = oracle.Table([8], compression=code)
    t.insert([np.arange(30000) % 11])
    nodes = t.nodes_array().copy()
    assert nodes.shape[0] % 80 == 0
    vl = nodes[40:48].view(np.uint64)
    vl[0] -= 1                                             # truncated stream: "cannot decompress the buffer"
    bad = cg.Relation.from_image(t.pages(), t.stripes_array(), nodes, [8])
    with pytest.raises(capi.CitusGpuError) as e:
        cg.Shard(bad)
    assert e.value.code == capi.CG_ECORRUPT
    d = cg.make_desc(aggs=[cg.count_star(), cg.sum_(0)])
    agg = cg.GpuColumnarAgg(d, bad.column_descs())
    with pytest.raises(capi.CitusGpuError) as e:
        agg.scan_relation(bad)
        agg.groups()
    assert e.value.code == capi.CG_ECORRUPT
    agg.free()


def test_unsupported_inputs_are_refused(cg, oracle):
    from citus_b200 import capi
    t = oracle.Table([8])
    t.insert([np.arange(50000) % 7])
    nodes = t.nodes_array().copy()
    nodes[4:8].view(np.int32)[0] = 7                                            # no such CompressionType
    rel = cg.Relation.from_image(t.pages(), t.stripes_array(), nodes, [8])
    with pytest.raises(capi.CitusGpuError) as e:
        cg.Shard(rel)
    assert e.value.code == capi.CG_ECORRUPT
    rel = cg.Relation.write([8], [np.arange(10)])
    with pytest.raises(capi.CitusGpuError):
        cg.GpuColumnarAgg(cg.make_desc(aggs=[cg.sum_(3)]), rel.column_descs())     # column out of range
    corrupt = rel.pages().copy()
    corrupt[2 * 8192 + 12: 2 * 8192 + 14] = 0                                    # pd_lower of the first data page
    bad = cg.Relation.from_image(corrupt, rel.stripes_bytes(), rel.nodes_bytes(), [8])
    with pytest.raises(capi.CitusGpuError) as e:
        cg.Shard(bad)
    assert e.value.code == capi.CG_ECORRUPT


# --------------------------------------------------------------------------- combine (K5)
def test_combine_partials_of_four_shards(cg, oracle):
    import torch
    cols = [(8, 0, 0, 3000, 0), (8, 0, 0, 100, 0), (8, 0, -10**12, 10**12, 20000)]
    aggs = [cg.sum_(2), cg.count_star(), cg.min_(2), cg.max_(2)]
    for force_hash in (False, True):
        d = cg.make_desc([(1, "<", 50)], [0], aggs, expected_groups=4000)
        rels = [cg.Relation.generate(cols, 100_000 + s, seed=77, first_row=s * 10**6) for s in range(4)]
        kmin, kmax = (0, 2999) if not force_hash else (0, -1)
        final = cg.GpuColumnarAgg(d, rels[0].column_descs(), kmin, kmax, 10**6)
        want = None
        for rel in rels:
            part = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, 10**6)      # one worker task
            part.scan_shard(cg.Shard(rel))
            nw, ops, dense, cap = part.layout()
            n = part.ngroups()
            keys = torch.empty(n, dtype=torch.int64, device="cuda")
            kn = torch.empty(n, dtype=torch.uint8, device="cuda")
            words = torch.empty(n * nw, dtype=torch.int64, device="cuda")
            assert part.export_device(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), n) == n
            final.merge_rows(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), n)   # coordinator combine
            r = oracle_table(oracle, rel).scan([(1, "<", 50)], [0], to_oracle_aggs(oracle, aggs))
            if want is None:
                want = r
            else:
                want.combine(r)
        assert_same_groups(final.groups(), want.groups(), aggs)


# --------------------------------------------------------------------------- hash repartition (K6)
def _partition(cg, keys, nulls, key_len, method, mins, maxs):
    import torch
    dk = torch.from_numpy(np.ascontiguousarray(keys, np.int64)).cuda()
    dn = torch.from_numpy(np.ascontiguousarray(nulls, np.uint8)).cuda() if nulls is not None else None
    idx = torch.empty(len(keys), dtype=torch.int32, device="cuda")
    cnt = torch.empty(len(mins), dtype=torch.int64, device="cuda")
    cg.worker_partition_query_result(dk.data_ptr(), dn.data_ptr() if dn is not None else None, len(keys), key_len,
                                     method, mins, maxs, idx.data_ptr(), cnt.data_ptr())
    torch.cuda.synchronize()
    return idx, cnt, dk


def test_partition_goldens(cg, oracle, expected):
    i = np.arange(1, 11)
    idx, cnt, _ = _partition(cg, i, None, 4, "hash", expected["squares_hash_mins"], expected["squares_hash_maxs"])
    idx = idx.cpu().numpy()
    for p in range(4):
        assert i[idx == p].tolist() == expected["squares_hash_members"][p]
    i = np.arange(1, 1000001)
    idx, cnt, _ = _partition(cg, i, None, 4, "hash", expected["squares_hash_mins"], expected["squares_hash_maxs"])
    assert cnt.cpu().tolist() == [r[1] for r in expected["doubles_hash_text"]]
    idx, cnt, _ = _partition(cg, i, None, 4, "range", [0, 250001, 500001, 750001], [250000, 500000, 750000, 1000000])
    assert cnt.cpu().tolist() == [r[1] for r in expected["doubles_range_binary"]]
    # bytes_written of the COPY text / binary files (partitioned_intermediate_results.out: 21/14/5/9 and 93/57/39/75)
    import torch
    i = np.arange(1, 11)
    di, dsq = torch.from_numpy(i).cuda(), torch.from_numpy(i * i).cuda()
    idx, cnt, _ = _partition(cg, i, None, 4, "hash", expected["squares_hash_mins"], expected["squares_hash_maxs"])
    rows, nbytes = cg.partition_copy_bytes(idx.data_ptr(), 10, 4, [di.data_ptr(), dsq.data_ptr()], [4, 4], binary=False)
    assert [[p, int(rows[p]), int(nbytes[p])] for p in range(4)] == expected["squares_hash_text"]
    idx, cnt, _ = _partition(cg, i * i, None, 4, "range", [0, 21, 41, 61], [20, 40, 60, 100])
    rows, nbytes = cg.partition_copy_bytes(idx.data_ptr(), 10, 4, [di.data_ptr(), dsq.data_ptr()], [4, 4], binary=True)
    assert [[p, int(rows[p]), int(nbytes[p])] for p in range(4)] == expected["squares_range_binary"]
    i = np.arange(1, 1000001)
    di, d2 = torch.from_numpy(i).cuda(), torch.from_numpy(i * 2).cuda()
    idx, cnt, _ = _partition(cg, i, None, 4, "hash", expected["squares_hash_mins"], expected["squares_hash_maxs"])
    rows, nbytes = cg.partition_copy_bytes(idx.data_ptr(), len(i), 4, [di.data_ptr(), d2.data_ptr()], [4, 4], binary=False)
    assert [[p, int(rows[p]), int(nbytes[p])] for p in range(4)] == expected["doubles_hash_text"]
    idx, cnt, _ = _partition(cg, i, None, 4, "range", [0, 250001, 500001, 750001], [250000, 500000, 750000, 1000000])
    rows, nbytes = cg.partition_copy_bytes(idx.data_ptr(), len(i), 4, [di.data_ptr(), d2.data_ptr()], [4, 4], binary=True)
    assert [[p, int(rows[p]), int(nbytes[p])] for p in range(4)] == expected["doubles_range_binary"]
    # edge keys that hash to INT32_MAX / INT32_MIN (distributed_planning.out:12-33)
    mins, maxs = oracle.synthetic_intervals(32)
    idx, cnt, _ = _partition(cg, np.array([2608474032, 963809240]), None, 8, "hash", mins, maxs)
    assert idx.cpu().tolist() == [31, 0]


def test_partition_parity_and_scatter(cg, oracle):
    import torch
    rng = np.random.default_rng(6)
    n = 1_234_567
    keys = rng.integers(-2**63, 2**63 - 1, n)
    nulls = (rng.random(n) < 0.01).astype(np.uint8)
    payload = rng.integers(-2**40, 2**40, n)
    for P in (1, 3, 32, 257):
        mins, maxs = oracle.synthetic_intervals(P)
        idx, cnt, dk = _partition(cg, keys, nulls, 8, "hash", mins, maxs)
        want_idx, want_rows = oracle.partition_rows(keys, nulls, 8, "h", mins, maxs)
        assert np.array_equal(idx.cpu().numpy(), want_idx)
        assert np.array_equal(cnt.cpu().numpy(), want_rows)
        dp = torch.from_numpy(payload).cuda()
        # the UDF's return rows: COPY text and binary byte counts with NULLs, negative and 19-digit values
        dn = torch.from_numpy(nulls).cuda()
        for binary in (False, True):
            rows, nbytes = cg.partition_copy_bytes(idx.data_ptr(), n, P, [dk.data_ptr(), dp.data_ptr()], [8, 8], binary,
                                                   d_null_ptrs=[dn.data_ptr(), None])
            assert np.array_equal(rows, want_rows)
            for p in (0, P // 2, P - 1):
                want_bytes = oracle.copy_file_bytes([keys, payload], [8, 8], want_idx, p, binary, colnulls=[nulls, None])
                if binary and want_rows[p] == 0:
                    want_bytes = 0                      # lazy start-up: the receiver of an empty partition never starts
                assert int(nbytes[p]) == want_bytes, (P, p, binary)
        ok = torch.empty_like(dk)
        op = torch.empty_like(dp)
        offs = cg.partition_scatter(idx.data_ptr(), n, P, [dk.data_ptr(), dp.data_ptr()], [ok.data_ptr(), op.data_ptr()])
        assert np.array_equal(np.diff(offs), want_rows)
        ok, op = ok.cpu().numpy(), op.cpu().numpy()
        for p in (0, P // 2, P - 1):
            sel = want_idx == p                                   # stable: input order inside a partition
            assert np.array_equal(ok[offs[p]:offs[p + 1]], keys[sel])
            assert np.array_equal(op[offs[p]:offs[p + 1]], payload[sel])
    # a hash that falls in no interval is an error, like the reference's ereport
    from citus_b200 import capi
    with pytest.raises(capi.CitusGpuError):
        _partition(cg, np.arange(100), None, 8, "hash", [0], [10])


# --------------------------------------------------------------------------- optimistic packing
def test_packed_accumulators_overflow_is_detected_and_retry_is_exact(cg, oracle):
    """count(*) + bounded sum share one 64-bit word per group; a group that receives >= 2^C
    rows between drains must be reported (CG_ERETRY_UNPACKED), never answered wrongly."""
    from citus_b200 import capi
    rng = np.random.default_rng(21)
    n = 400_000
    key = rng.integers(0, 100_000, n)                           # domain too large for the shared-memory kernel
    key[:150_000] = 7                                           # one hot group: 150 000 rows > 2^16
    v = rng.integers(-10**9, 10**9, n)
    rel = cg.Relation.write([8, 8], [key, v])
    aggs = [cg.sum_(1), cg.count_star()]
    d = cg.make_desc(group_cols=[0], aggs=aggs)
    kmin, kmax, bounds, rows = cg.relation_bounds(rel, d)
    aggs[0].term_abs_bound = bounds[0]
    d = cg.make_desc(group_cols=[0], aggs=aggs)
    agg = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, rows)
    shard = cg.Shard(rel)
    agg.scan_shard(shard, want_stats=False)
    with pytest.raises(capi.CitusGpuError) as e:
        agg.groups()
    assert e.value.code == capi.CG_ERETRY_UNPACKED
    agg.reset()
    agg.set_packing(False)
    agg.scan_shard(shard, want_stats=False)
    want = oracle_table(oracle, rel).scan([], [0], to_oracle_aggs(oracle, aggs)).groups()
    assert_same_groups(agg.groups(), want, aggs)
    # moderate skew below the threshold stays on the packed path and is exact
    key2 = rng.integers(0, 100_000, n)
    key2[:60_000] = 7
    rel2 = cg.Relation.write([8, 8], [key2, v])
    agg2 = cg.GpuColumnarAgg(d, rel2.column_descs(), kmin, kmax, rows)
    for _ in range(3):                                          # drained between launches: 3 x 60 400 rows is fine
        agg2.scan_shard(cg.Shard(rel2), want_stats=False)
        agg2.ngroups()
    want = oracle.Result(to_oracle_aggs(oracle, aggs))
    for _ in range(3):
        oracle_table(oracle, rel2).scan([], [0], to_oracle_aggs(oracle, aggs), into=want)
    assert_same_groups(agg2.groups(), want.groups(), aggs)


# --------------------------------------------------------------------------- merge-side join (K8)
def test_join_count_sum_matches_row_at_a_time_join(cg, oracle):
    import torch
    rng = np.random.default_rng(21)
    for nb, npr, domain in ((1, 1, 1), (1000, 0, 10), (50_000, 70_000, 5_000), (300_000, 250_000, 1 << 28)):
        bk = rng.integers(0, domain, nb)
        pk = rng.integers(0, domain, npr)
        if nb > 10:
            bk[:5] = [-2**63, 2**63 - 1, 0, -1, -2**63]           # the table's EMPTY sentinel is a legal key
        if npr > 10:
            pk[:4] = [-2**63, 2**63 - 1, -1, 7]
        bx = rng.integers(-2**62, 2**62, nb)
        py = rng.integers(-2**62, 2**62, npr)
        bn = (rng.random(nb) < 0.05).astype(np.uint8)
        pn = (rng.random(npr) < 0.05).astype(np.uint8)
        want = oracle.join_count_sum(bk, bx, pk, py, bn, pn)
        d = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (bk, bx, pk, py, bn, pn)]
        got = cg.join_count_sum(d[0].data_ptr(), d[1].data_ptr(), nb, d[2].data_ptr(), d[3].data_ptr(), npr,
                                d_build_nulls=d[4].data_ptr(), d_probe_nulls=d[5].data_ptr())
        assert got == want, (nb, npr, domain)


# --------------------------------------------------------------------------- NULL-bearing chunk groups on the fast paths
@pytest.mark.parametrize("family", ["jit", "jit_always", "aot", "general"])
@pytest.mark.parametrize("path", ["shard", "e2e", "dma"])
def test_c2_with_nulls_on_every_kernel_family(cg, oracle, kernel_family, family, path):
    """SURVEY 8(d): C2 with 5 % NULLs in v (and, second pass, NULLs in the key and the filter column too).
    count(*) counts the row, sum(v) skips it (strict transition function), a NULL filter input drops the
    row, a NULL key is its own group -- bit-exact against the oracle on every kernel family and staging path"""
    from citus_b200 import capi
    kernel_family(family)
    for nulls in ((0, 0, 50000), (20000, 30000, 50000)):
        cols = [(8, 0, 0, 3000, nulls[0]), (8, 0, 0, 100, nulls[1]), (8, 0, -10**9, 10**9, nulls[2])] + [(8, 0, 0, 1 << 40, 0)] * 2
        rel = cg.Relation.generate(cols, 123_457, seed=77 + nulls[0], stripe_row_limit=30000, chunk_row_limit=5000)
        aggs = [cg.sum_(2), cg.count_star(), cg.count(2)]
        jit0 = capi.lib().cg_jit_launches()
        for force_hash in (False, True):
            run_both(cg, oracle, rel, [(1, "<", 50)], [0], aggs, chunk_row_limit=5000, force_hash=force_hash,
                     e2e=False if path == "shard" else path)
        if family in ("jit", "jit_always"):
            assert capi.lib().cg_jit_launches() > jit0       # the NULL-bearing chunk groups ran on the generated kernel
        else:
            assert capi.lib().cg_jit_launches() == jit0


@pytest.mark.parametrize("family", ["jit", "general"])
def test_nulls_in_plain_and_small_domain_aggregates(cg, oracle, kernel_family, family):
    """NULL inputs in a plain aggregate (thread registers) and in a tiny key domain (shared-memory cells),
    mixed widths, min/max/count(x), a NULL group key on the small-domain table"""
    kernel_family(family)
    cols = [(8, 0, -1000, 1000, 100000), (4, 0, 0, 100, 50000), (2, 0, 0, 5, 150000), (1, 0, -50, 50, 300000),
            (8, 0, -2**40, 2**40, 10000)]
    rel = cg.Relation.generate(cols, 77_777, seed=5, stripe_row_limit=20000, chunk_row_limit=3000)
    aggs = [cg.sum_(0), cg.count_star(), cg.count(3), cg.min_(4), cg.max_(0), cg.sum_(3)]
    run_both(cg, oracle, rel, [(1, "<", 70)], [], aggs, chunk_row_limit=3000)
    run_both(cg, oracle, rel, [(1, "<", 70)], [2], aggs, chunk_row_limit=3000)
    run_both(cg, oracle, rel, [(1, ">=", 10)], [2], aggs, chunk_row_limit=3000, e2e=True)


# --------------------------------------------------------------------------- WHERE trees (R10)
@pytest.mark.parametrize("family", ["jit", "general"])
def test_or_clause_goldens_through_the_gpu(cg, oracle, expected, kernel_family, family):
    """expected/columnar_chunk_filtering.out pushdown_test: Rows Removed by Filter, Columnar Chunk Groups
    Removed by Filter and sum(a) of the three OR queries"""
    kernel_family(family)
    a = np.arange(1, 200001)
    rel = cg.Relation.write([4, 4], [a, np.zeros_like(a)], [None, np.ones(a.shape[0], np.uint8)],
                            stripe_row_limit=2000, chunk_row_limit=1000)
    trees = {
        "a = 204356 or a = 104356 or a = 76556": ("or", (0, "=", 204356), (0, "=", 104356), (0, "=", 76556)),
        "a = 194356 or a = 104356 or a = 76556": ("or", (0, "=", 194356), (0, "=", 104356), (0, "=", 76556)),
        "(a > 1000 and a < 10000) or (a > 20000 and a < 50000)":
            ("or", ("and", (0, ">", 1000), (0, "<", 10000)), ("and", (0, ">", 20000), (0, "<", 50000))),
    }
    for g in expected["pushdown_or"]:
        for e2e in (False, True):
            st, got = run_both(cg, oracle, rel, trees[g["where"]], [], [cg.sum_(0)], chunk_row_limit=1000, e2e=e2e)
            assert st.chunk_groups_filtered == g["groups_removed"]
            assert st.rows_removed_by_filter == g["rows_removed"]
            assert got[0][0]["sum"] == g["sum"]


@pytest.mark.parametrize("family", ["jit", "general"])
def test_where_trees_with_nulls_and_groups(cg, oracle, kernel_family, family):
    """three-valued logic under OR: FALSE OR NULL drops the row, TRUE OR NULL keeps it; trees over several
    columns, float atoms, GROUP BY on a direct-indexed and a hash table"""
    kernel_family(family)
    rng = np.random.default_rng(21)
    n = 60_000
    k = rng.integers(0, 500, n)
    x = rng.integers(-100, 100, n)
    y = rng.integers(0, 1000, n)
    f = rng.normal(size=n)
    nx = (rng.random(n) < 0.2).astype(np.uint8)
    ny = (rng.random(n) < 0.1).astype(np.uint8)
    rel = cg.Relation.write([8, 4, 8, 8], [k, x, y, f], [None, nx, ny, None], type_classes=[0, 0, 0, 1],
                            stripe_row_limit=20000, chunk_row_limit=4000)
    where = ("and", ("or", (1, "<", -50), (2, ">", 900), ("and", (3, ">", 0.5), (1, "<>", 7))), (0, "<", 450))
    aggs = [cg.sum_(2), cg.count_star(), cg.count(1), cg.max_(1)]
    for force_hash in (False, True):
        run_both(cg, oracle, rel, where, [0], aggs, chunk_row_limit=4000, force_hash=force_hash, float_cols=(3,))
    run_both(cg, oracle, rel, where, [], aggs, chunk_row_limit=4000, float_cols=(3,), e2e=True)


# --------------------------------------------------------------------------- R18: the partition files themselves
def test_copy_serializer_writes_the_reference_files(cg, oracle, expected):
    """cg_partition_copy_serialize: the COPY text / binary bytes of every partition file -- golden sizes
    (21/14/5/9 and 93/57/39/75) and byte-for-byte the oracle's row-at-a-time files, incl. NULLs, negative
    numbers, empty partitions (lazy start-up vs generate_empty_results) and 200 000 rows over 32 partitions"""
    import torch

    def files_of(idx_t, n, P, cols, lens, binary, nulls=None, gen_empty=False):
        dcols = [torch.from_numpy(np.ascontiguousarray(c, np.int64)).cuda() for c in cols]
        dn = None if nulls is None else [None if x is None else torch.from_numpy(np.ascontiguousarray(x, np.uint8)).cuda() for x in nulls]
        rows, nbytes = cg.partition_copy_bytes(idx_t.data_ptr(), n, P, [c.data_ptr() for c in dcols], lens, binary=binary,
                                               d_null_ptrs=None if dn is None else [None if x is None else x.data_ptr() for x in dn],
                                               generate_empty_results=gen_empty)
        total = int(nbytes.sum())
        out = torch.zeros(max(total, 1) + 64, dtype=torch.uint8, device="cuda")
        offs = cg.partition_copy_serialize(idx_t.data_ptr(), n, P, [c.data_ptr() for c in dcols], lens, binary, out.data_ptr(), total,
                                           d_null_ptrs=None if dn is None else [None if x is None else x.data_ptr() for x in dn],
                                           generate_empty_results=gen_empty)
        assert np.array_equal(np.diff(offs), nbytes)
        host = out.cpu().numpy().tobytes()
        assert host[total:total + 64] == b"\0" * 64                      # nothing written past the files
        return [host[offs[p]:offs[p + 1]] for p in range(P)], rows, nbytes

    i = np.arange(1, 11)
    idx, cnt, _ = _partition(cg, i, None, 4, "hash", expected["squares_hash_mins"], expected["squares_hash_maxs"])
    files, rows, nbytes = files_of(idx, 10, 4, [i, i * i], [4, 4], False)
    assert [[p, int(rows[p]), len(files[p])] for p in range(4)] == expected["squares_hash_text"]
    assert files == oracle.copy_files(idx.cpu().numpy(), [i, i * i], [4, 4], 4, False)
    idx, cnt, _ = _partition(cg, i * i, None, 4, "range", [0, 21, 41, 61], [20, 40, 60, 100])
    files, rows, nbytes = files_of(idx, 10, 4, [i, i * i], [4, 4], True)
    assert [[p, int(rows[p]), len(files[p])] for p in range(4)] == expected["squares_range_binary"]
    assert files == oracle.copy_files(idx.cpu().numpy(), [i, i * i], [4, 4], 4, True)
    # larger, with NULLs, negative values, 8-byte and 2-byte binary fields, partitions that receive nothing
    rng = np.random.default_rng(8)
    n, P = 200_000, 32
    k = rng.integers(-2**40, 2**40, n)
    a = rng.integers(-30000, 30000, n)
    b = rng.integers(-2**62, 2**62, n)
    na = (rng.random(n) < 0.1).astype(np.uint8)
    mins, maxs = oracle.synthetic_intervals(P)
    idx, cnt, _ = _partition(cg, k, None, 8, "hash", mins, maxs)
    hidx = idx.cpu().numpy()
    for binary in (False, True):
        files, rows, nbytes = files_of(idx, n, P, [k, a, b], [8, 2, 8], binary, nulls=[None, na, None])
        assert files == oracle.copy_files(hidx, [k, a, b], [8, 2, 8], P, binary, nulls=[None, na, None])
    few = np.array([5, 6, 7])
    idx, cnt, _ = _partition(cg, few, None, 8, "range", [0, 100, 200], [99, 199, 299])
    for gen_empty in (False, True):
        files, rows, nbytes = files_of(idx, 3, 3, [few], [8], True, gen_empty=gen_empty)
        assert files == oracle.copy_files(idx.cpu().numpy(), [few], [8], 3, True, generate_empty_results=gen_empty)
        assert len(files[1]) == (21 if gen_empty else 0)


# --------------------------------------------------------------------------- (f)-4: varlena numeric / char(1) columns
NUM2 = 2 | (2 << 8)          # numeric with scale 2 (decimal(15,2)); 3 = char(1)


def _lineitem_varlena_rels(cg, oracle, li, short_headers, compression):
    """the reference's own lineitem column types (test/regress/sql/multi_create_table.sql:12-28): decimal(15,2) for
    quantity / extendedprice / discount / tax, char(1) for the flags -- written as varlena datums by the oracle's writer"""
    mins, maxs = oracle.synthetic_intervals(2)
    idx, _ = oracle.partition_rows(li["l_orderkey"], None, 8, "h", mins, maxs)
    cols = ["l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus", "l_shipdate", "l_suppkey"]
    attlen = [-1, -1, -1, -1, -1, -1, 4, 4]
    atttype = [NUM2, NUM2, NUM2, NUM2, 3, 3, 0, 0]
    rels = []
    oracle.lib().orc_set_short_varlena_headers(1 if short_headers else 0)
    try:
        for s in range(2):
            t = oracle.Table(attlen, atttype, stripe_row_limit=2000, chunk_row_limit=1000, compression=compression)
            t.insert([li[c][idx == s] for c in cols])
            rels.append(cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), attlen, atttype))
    finally:
        oracle.lib().orc_set_short_varlena_headers(0)
    return rels


@pytest.mark.parametrize("path", ["shard", "e2e", "dma"])
@pytest.mark.parametrize("compression", ["none", "lz4"])
@pytest.mark.parametrize("short_headers", [False, True])
def test_tpch_goldens_on_varlena_numeric_and_char_columns(cg, oracle, expected, lineitem, short_headers, compression, path):
    """TPC-H Q1 + Q6 (expected/multi_tpch_query1.out, multi_tpch_query6.out) over decimal(15,2) / char(1) columns stored
    as varlena value streams (4-byte and packed 1-byte headers, plain and lz4-compressed): decoded on the GPU
    (cg_varlena_decode_kernel) into the fixed-width form the fused kernels scan"""
    if compression == "lz4" and not oracle.lib().orc_have_lz4():
        pytest.skip("liblz4 missing")
    comp = {"none": oracle.COMP_NONE, "lz4": oracle.COMP_LZ4}[compression]
    e2e = False if path == "shard" else (True if path == "e2e" else "dma")
    rels = _lineitem_varlena_rels(cg, oracle, lineitem, short_headers, comp)
    quals = [(6, ">=", pgdate("1994-01-01")), (6, "<", pgdate("1995-01-01")), (2, ">=", 5), (2, "<=", 7), (0, "<", 2400)]
    aggs = [cg.Agg(2, [(1, 0, 1), (2, 0, 1)])]
    total = 0
    for rel in rels:
        _, got = run_both(cg, oracle, rel, quals=quals, aggs=aggs, chunk_row_limit=1000, e2e=e2e)
        total += got[0][0]["sum"]
    assert cg.numeric_out(total, 4) == expected["tpch_q6"]
    quals = [(6, "<=", pgdate("1998-09-02"))]
    aggs = [cg.sum_(0), cg.sum_(1), cg.Agg(2, [(1, 0, 1), (2, 100, -1)]),
            cg.Agg(2, [(1, 0, 1), (2, 100, -1), (3, 100, 1)]), cg.sum_(2), cg.count_star()]
    merged = {}
    for rel in rels:
        _, got = run_both(cg, oracle, rel, quals=quals, group_cols=[4, 5], aggs=aggs, chunk_row_limit=1000, expected_groups=16, e2e=e2e)
        for k, per in got.items():
            acc = merged.setdefault(k, [dict(sum=0, count=0) for _ in aggs])
            for a in range(len(aggs)):
                acc[a]["sum"] += per[a]["sum"]
                acc[a]["count"] += per[a]["count"]
    rows = []
    for key, v in sorted(merged.items(), key=lambda kv: (kv[0] & 0xffffffff, kv[0] >> 32)):
        rows.append([chr(key & 0xff), chr((key >> 32) & 0xff), cg.numeric_out(v[0]["sum"], 2), cg.numeric_out(v[1]["sum"], 2),
                     cg.numeric_out(v[2]["sum"], 4), cg.numeric_out(v[3]["sum"], 6), cg.numeric_div_out(v[0]["sum"], 2, v[0]["count"]),
                     cg.numeric_div_out(v[1]["sum"], 2, v[1]["count"]), cg.numeric_div_out(v[4]["sum"], 2, v[4]["count"]), str(v[5]["count"])])
    assert rows == expected["tpch_q1"]


def test_varlena_columns_with_nulls_wide_values_and_bad_scale(cg, oracle):
    """NULLs in varlena columns (rank directory over the decoded array), values up to 10^17, negative numbers, zero; a value
    with more fractional digits than the declared scale is refused (CG_EUNSUPPORTED), never rounded"""
    from citus_b200 import capi
    rng = np.random.default_rng(4)
    n = 25_000
    a = rng.integers(-10**17, 10**17, n)
    a[:6] = [0, 1, -1, 10**17, -10**17, 99]
    b = rng.integers(0, 50, n)
    f = rng.integers(65, 70, n)
    na = (rng.random(n) < 0.15).astype(np.uint8)
    nf = (rng.random(n) < 0.05).astype(np.uint8)
    NUM4 = 2 | (4 << 8)
    for short in (False, True):
        oracle.lib().orc_set_short_varlena_headers(1 if short else 0)
        try:
            t = oracle.Table([-1, 8, -1], [NUM4, 0, 3], stripe_row_limit=6000, chunk_row_limit=1500)
            t.insert([a, b, f], nulls=[na, None, nf])
        finally:
            oracle.lib().orc_set_short_varlena_headers(0)
        rel = cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), [-1, 8, -1], [NUM4, 0, 3])
        aggs = [cg.sum_(0), cg.count_star(), cg.count(0), cg.min_(0), cg.max_(0), cg.count(2)]
        run_both(cg, oracle, rel, [(1, "<", 40)], [2], aggs, chunk_row_limit=1500)
        run_both(cg, oracle, rel, [(0, ">", 0)], [], aggs, chunk_row_limit=1500, e2e=True)
    # the same bytes declared as numeric with scale 2: values like 0.0123 are not representable -> refused
    rel = cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), [-1, 8, -1], [NUM2, 0, 3])
    d = cg.make_desc([], [], [cg.sum_(0)])
    agg = cg.GpuColumnarAgg(d, rel.column_descs(), 0, -1, n)
    with pytest.raises(capi.CitusGpuError) as ei:
        agg.scan_relation(rel)
        agg.groups()
    assert ei.value.code == capi.CG_EUNSUPPORTED


def test_join_rows_matches_a_row_at_a_time_join(cg, oracle):
    """cg_join_rows: the merge-side join emitting (key, b.payload, p.payload) rows -- the multiset of rows equals a
    nested-loop join on the host (duplicates on both sides, NULL keys join nothing, the key equal to the table's EMPTY
    sentinel, an empty side, capacity handling).  600 000 probe rows are 2344 blocks of 256: the offsets of the second
    scan chunk of 2048 blocks carry the first chunk's rows"""
    import torch
    from collections import Counter
    from citus_b200 import capi
    rng = np.random.default_rng(12)
    nb = 30_000
    for npr, pkeys in ((50_000, 6000), (600_000, 60_000)):
        bk = rng.integers(0, 5000, nb); bk[:3] = -2**63
        pk = rng.integers(0, pkeys, npr); pk[:2] = -2**63
        bx = rng.integers(-2**40, 2**40, nb)
        py = rng.integers(-2**40, 2**40, npr)
        bn = (rng.random(nb) < 0.05).astype(np.uint8)
        pn = (rng.random(npr) < 0.05).astype(np.uint8)
        d = [torch.from_numpy(x).cuda() for x in (bk, bx, pk, py)]
        dbn, dpn = torch.from_numpy(bn).cuda(), torch.from_numpy(pn).cuda()
        n = cg.join_rows(d[0].data_ptr(), d[1].data_ptr(), nb, d[2].data_ptr(), d[3].data_ptr(), npr,
                         d_build_nulls=dbn.data_ptr(), d_probe_nulls=dpn.data_ptr())
        joined, jsum = cg.join_count_sum(d[0].data_ptr(), d[1].data_ptr(), nb, d[2].data_ptr(), d[3].data_ptr(), npr,
                                         d_build_nulls=dbn.data_ptr(), d_probe_nulls=dpn.data_ptr())
        wj, ws = oracle.join_count_sum(bk, bx, pk, py, bn, pn)
        assert n == joined == wj and jsum == ws
        out = [torch.empty(n, dtype=torch.int64, device="cuda") for _ in range(3)]
        n2 = cg.join_rows(d[0].data_ptr(), d[1].data_ptr(), nb, d[2].data_ptr(), d[3].data_ptr(), npr, capacity=n,
                          d_out=[o.data_ptr() for o in out], d_build_nulls=dbn.data_ptr(), d_probe_nulls=dpn.data_ptr())
        assert n2 == n
        got = Counter(zip(*(o.cpu().tolist() for o in out)))
        by_key = {}
        for k, x, z in zip(bk.tolist(), bx.tolist(), bn.tolist()):
            if not z:
                by_key.setdefault(k, []).append(x)
        want = Counter()
        for k, y, z in zip(pk.tolist(), py.tolist(), pn.tolist()):
            if not z:
                for x in by_key.get(k, ()):
                    want[(k, x, y)] += 1
        assert got == want
        # the emitted rows add up to the aggregate form's sum
        assert int((out[1].cpu().numpy().astype(object) + out[2].cpu().numpy().astype(object)).sum()) == ws
        with pytest.raises(capi.CitusGpuError):
            cg.join_rows(d[0].data_ptr(), d[1].data_ptr(), nb, d[2].data_ptr(), d[3].data_ptr(), npr, capacity=n - 1,
                         d_out=[o.data_ptr() for o in out], d_build_nulls=dbn.data_ptr(), d_probe_nulls=dpn.data_ptr())
        assert cg.join_rows(d[0].data_ptr(), d[1].data_ptr(), 0, d[2].data_ptr(), d[3].data_ptr(), npr) == 0


@pytest.mark.parametrize("tma", [1, 0])
def test_dma_realign_kernels_agree(cg, oracle, tma):
    """pinned pages -> whole-page DMA -> de-framing on the GPU, with the Hopper bulk-copy pipeline (cp.async.bulk + mbarrier) and
    with the plain-load kernel: ragged chunk sizes so that buffers start at every byte alignment and straddle page headers"""
    cg.set_option("realign_tma", tma)
    try:
        cols = [(8, 0, 0, 500, 0), (4, 0, 0, 100, 20000), (2, 0, -1000, 1000, 0), (1, 0, -50, 50, 100000), (8, 0, -10**9, 10**9, 50000)]
        for rows, chunk in ((54_321, 1777), (100_003, 10_000), (999, 1000)):
            rel = cg.Relation.generate(cols, rows, seed=rows, stripe_row_limit=chunk * 7, chunk_row_limit=chunk)
            aggs = [cg.sum_(4), cg.count_star(), cg.min_(2), cg.max_(3), cg.count(1)]
            run_both(cg, oracle, rel, [(1, "<", 70)], [0], aggs, chunk_row_limit=chunk, e2e="dma")
    finally:
        cg.set_option("realign_tma", 1)
