"""The row-emitting scan (cg_scan_shard_rows) against the oracle's decode of the same image and the vectorised WHERE
reference (tests/scan_rows_reference.py): every emitted value, null byte, the row count and the row order, for every
column type the scan decodes, NULLs in WHERE and in projected-only columns, every codec, several stripes, chunk row
limits and chunk-group tails at the bitmap word edges, a shard whose tile-offset scan takes several chunks, the
capacity protocol, the refusals, the aggregate scan's cached chunk-group selection, and the two places the rows go: the
COPY files of worker_partition_query_result and a repartition join through the one-GPU exchange."""
import ctypes as C
import math

import numpy as np
import pytest

import join_agg_reference as jref
import reference as ref
import scan_rows_reference as srr
from gpu_harness import cg  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

BPCHAR1, NUMERIC2 = 3, 2 | (2 << 8)
# bool, int1, int2, int4, int8, char(1), numeric(12, 2), float4, float8
ATTLENS = [1, 1, 2, 4, 8, -1, -1, 4, 8]
TYPES = [0, 0, 0, 0, 0, BPCHAR1, NUMERIC2, 1, 1]
FLOAT_COLS = (7, 8)
SCALES = {6: 2}
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
SENTINEL = 0x5A5A5A5A5A5A5A5A


def make_rows(rng, n, null_rate=0.06):
    """values at every type's edges; NULLs in every column but the int8 one, none in the first 3000 rows (NULL-free
    chunk groups next to NULL-bearing ones)"""
    f4 = np.array([-1.5, -0.0, 0.0, 2.25, 1e30, -1e-30, math.inf, -math.inf, math.nan], np.float32)
    f8 = rng.normal(0, 1e3, n)
    sp = rng.random(n) < 0.05
    f8[sp] = np.array([math.nan, math.inf, -math.inf, -0.0, 0.0])[rng.integers(0, 5, int(sp.sum()))]
    i8 = rng.integers(-2**62, 2**62, n)
    i8[:4] = [INT64_MIN, INT64_MAX, -1, 0]
    cols = [rng.integers(0, 2, n), rng.integers(-128, 128, n), rng.integers(-2**15, 2**15, n), rng.integers(-2**31, 2**31, n),
            i8, rng.choice([0x20, 0x41, 0x5A, 0x7F, 0x80, 0xE9, 0xFF], n), rng.integers(-10**11, 10**11, n),
            f4[rng.integers(0, len(f4), n)].astype(np.float64), f8]
    nulls = []
    for c in range(len(cols)):
        z = (rng.random(n) < null_rate).astype(np.uint8)
        z[:3000] = 0
        if c == 4:
            z[:] = 0
        nulls.append(z)
    return cols, nulls


def write(cg, oracle, cols, nulls, stripe_rows, chunk_rows, compression=0, attlens=ATTLENS, types=TYPES):
    t = oracle.Table(attlens, types, stripe_row_limit=stripe_rows, chunk_row_limit=chunk_rows, compression=compression)
    t.insert(cols, nulls)
    rel = cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), attlens, types)
    return rel, t


def scan_rows(cg, shard, where, atts, float_cols=FLOAT_COLS, pushdown=True):
    """(rows, stats, values, nulls) through the count call and the write call, outputs pre-filled with sentinels"""
    import torch
    d = cg.make_desc(where if where is not None else (), (), (), qual_pushdown=pushdown, float_cols=float_cols)
    n, st0 = shard.scan_rows(d, atts)
    cols = [torch.full((n + 1,), SENTINEL, dtype=torch.int64, device="cuda") for _ in atts]
    nul = [torch.full((n + 1,), 7, dtype=torch.uint8, device="cuda") for _ in atts]
    n2, st = shard.scan_rows(d, atts, [c.data_ptr() for c in cols], [x.data_ptr() for x in nul], n)
    torch.cuda.synchronize()
    assert n2 == n and st0.rows_passed == st.rows_passed == n
    assert st0.chunk_groups_filtered == st.chunk_groups_filtered and st0.rows_scanned == st.rows_scanned
    vals = [c.cpu().numpy() for c in cols]
    nuls = [x.cpu().numpy() for x in nul]
    assert all(v[n] == SENTINEL for v in vals) and all(x[n] == 7 for x in nuls), "a row past the count was written"
    return n, st, [v[:n] for v in vals], [x[:n] for x in nuls]


def _canonical(v, att, float4_cols):
    """float4 NaNs widen to a NaN whose payload the conversion chooses: compare them as one NaN"""
    if att not in float4_cols:
        return v
    f = v.view(np.float64)
    return np.where(np.isnan(f), np.int64(0x7FF8000000000000), v)


def check(cg, shard, dec_vals, dec_nulls, where, atts, stripe_rows, chunk_rows, float_cols=FLOAT_COLS, scales=SCALES,
          float4_cols=(7,), pushdown=True):
    n, st, got_v, got_n = scan_rows(cg, shard, where, atts, float_cols, pushdown)
    want_v, want_n = srr.expected_rows(dec_vals, dec_nulls, where, atts, float_cols, scales)
    assert n == len(want_v[0]), (where, n, len(want_v[0]))
    for i, a in enumerate(atts):
        assert np.array_equal(got_n[i], want_n[i]), (where, a)
        assert np.array_equal(_canonical(got_v[i], a, float4_cols), _canonical(want_v[i], a, float4_cols)), (where, a)
    total = len(dec_vals[0])
    mask = ref.selected_chunk_mask(dec_vals, dec_nulls, where, stripe_rows, chunk_rows, float_cols=float_cols,
                                   qual_pushdown=pushdown)
    assert st.chunk_groups_filtered == ref.chunks_filtered(mask), where
    assert st.chunk_groups_scanned == sum(k for s in mask for k in s)
    assert st.rows_scanned == ref.rows_kept(mask, total, stripe_rows, chunk_rows), where
    assert st.rows_passed == n and st.rows_removed_by_filter == st.rows_scanned - n
    return n, st


def where_forms(cg):
    Col = cg.Col
    return [
        None,                                                                     # no WHERE: every row
        [(4, ">=", INT64_MIN)],                                                   # passes everything
        [(1, ">", 127)],                                                          # passes nothing (every chunk skipped)
        [(2, "<", 0), (3, ">", 0)],
        ("or", ("and", (0, "=", 1), (5, ">", 0x7F)), ("and", (6, "<=", -10**10), (8, ">", 0.0))),
        ("or", (7, "=", math.nan), (8, "<", -500.0)),
        [(5, "in", (0x41, 0xE9, None)), (1, "not in", (0, 1, 2))],
        ("or", (3, "is null"), (6, "is null")),
        [(2, "is not null"), (4, "in", (INT64_MIN, INT64_MAX, 0))],
        ("or", (2, "<", Col(3)), (6, ">", Col(4))),
        [(7, "<=", Col(8)), (0, "<>", Col(1))],
        ("and", ("or", (1, "<", -100), (1, ">", 100)), (8, "is not null"), (7, "<>", -0.0)),
    ]


@pytest.fixture(scope="module")
def typed(cg, oracle):
    rng = np.random.default_rng(20261019)
    cols, nulls = make_rows(rng, 20_000)
    rel, t = write(cg, oracle, cols, nulls, 6000, 1000)
    vals, dn = t.decode_all()
    return rel, vals, dn


ALL_ATTS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 4, 8]     # every type, two attributes twice


@pytest.mark.parametrize("form", range(12))
def test_types_and_where_forms(cg, typed, form):
    rel, vals, dn = typed
    shard = cg.Shard(rel)
    where = where_forms(cg)[form]
    n, _ = check(cg, shard, vals, dn, where, ALL_ATTS, 6000, 1000)
    if form in (0, 1):
        assert n == 20_000
    if form == 2:
        assert n == 0
    shard.free()


def test_pushdown_off_and_projection_only_nulls(cg, typed):
    """no skipping with enable_qual_pushdown off; projected columns whose NULLs the WHERE never reads"""
    rel, vals, dn = typed
    shard = cg.Shard(rel)
    check(cg, shard, vals, dn, [(4, "<", 0)], [8, 7, 6, 5, 3, 0], 6000, 1000, pushdown=False)
    check(cg, shard, vals, dn, [(4, "<", 0)], [8, 7, 6, 5, 3, 0], 6000, 1000)
    shard.free()


@pytest.mark.parametrize("compression", ["pglz", "lz4", "zstd"])
def test_codecs(cg, oracle, compression):
    kind = {"pglz": 1, "lz4": 2, "zstd": 3}[compression]
    if kind == 2 and not oracle.lib().orc_have_lz4() or kind == 3 and not oracle.lib().orc_have_zstd():
        pytest.skip(f"the oracle was built without {compression}")
    rng = np.random.default_rng(7 + kind)
    cols, nulls = make_rows(rng, 9000)
    cols[4] = rng.integers(-50, 50, 9000)                 # compressible values
    rel, t = write(cg, oracle, cols, nulls, 4000, 1000, compression=kind)
    vals, dn = t.decode_all()
    shard = cg.Shard(rel)
    for where in (None, [(4, "<", 0)], ("or", (3, "is null"), (5, "in", (0x41, 0xFF)))):
        check(cg, shard, vals, dn, where, ALL_ATTS, 4000, 1000)
    shard.free()


@pytest.mark.parametrize("chunk_rows", [1000, 1001, 1024, 100_000])
@pytest.mark.parametrize("tail", [1, 63, 64, 65])
def test_chunk_limits_and_tails(cg, oracle, chunk_rows, tail):
    """every stripe's last chunk group has `tail` rows (stripe_row_limit = 2 chunks + tail), the last stripe is short"""
    stripe_rows = 2 * chunk_rows + tail
    n = 3 * stripe_rows + 777
    rng = np.random.default_rng(chunk_rows * 100 + tail)
    attlens, types = [8, 4, 8], [0, 0, 1]
    cols = [rng.integers(-1000, 1000, n), rng.integers(-5, 5, n), rng.normal(size=n)]
    nulls = [np.zeros(n, np.uint8), (rng.random(n) < 0.1).astype(np.uint8), (rng.random(n) < 0.03).astype(np.uint8)]
    rel, t = write(cg, oracle, cols, nulls, stripe_rows, chunk_rows, attlens=attlens, types=types)
    vals, dn = t.decode_all()
    shard = cg.Shard(rel)
    for where in (None, [(0, "<", 0)], ("or", (1, "is null"), (2, ">", 1.0)), [(0, "=", 999)]):
        check(cg, shard, vals, dn, where, [2, 0, 1], stripe_rows, chunk_rows, float_cols=(2,), scales={}, float4_cols=())
    shard.free()


def test_large_shard_several_scan_chunks(cg, oracle):
    """~50 M rows: about 24 000 tiles, so the tile-offset scan runs over several of its chunks"""
    n = 50_000_000
    cols = [(8, 0, -10**6, 10**6, 0), (8, 0, 0, 1 << 40, 20000)]
    rel = cg.Relation.generate(cols, n, seed=20261019, stripe_row_limit=150_000, chunk_row_limit=10_000)
    t = oracle.Table.attach(rel.pages(), rel.stripes_bytes(), rel.nodes_bytes(), [8, 8], chunk_row_limit=10_000)
    vals, dn = t.decode_all()
    shard = cg.Shard(rel)
    for where in ([(0, "<", -8 * 10**5)], None):
        n_got, st, gv, gn = scan_rows(cg, shard, where, [1, 0], float_cols=())
        keep = srr.where_mask(where, vals, dn)
        assert n_got == int(keep.sum())
        assert np.array_equal(gv[1], vals[0][keep]) and np.array_equal(gn[0], dn[1][keep])
        assert np.array_equal(gv[0], np.where(dn[1] == 1, 0, vals[1])[keep])
        assert st.rows_scanned == n and st.kernel_ms > 0
    shard.free()


def _raw_call(cg, shard, desc, atts, capacity, cols, nulls):
    from citus_b200 import capi
    a = (C.c_int32 * len(atts))(*atts)
    cp = None if cols is None else (C.c_void_p * len(cols))(*cols)
    npp = None if nulls is None else (C.c_void_p * len(nulls))(*nulls)
    n = C.c_int64(-1)
    rc = capi.lib().cg_scan_shard_rows(shard.h, C.byref(desc), a, len(atts), capacity, cp, npp, C.byref(n), None)
    return rc, n.value


def test_capacity(cg, typed):
    import torch
    from citus_b200 import capi
    rel, vals, dn = typed
    shard = cg.Shard(rel)
    where = [(3, ">", 0)]
    d = cg.make_desc(where, float_cols=FLOAT_COLS)
    atts = [3, 8]
    rc, n = _raw_call(cg, shard, d, atts, 0, None, None)
    assert rc == 0 and n == int(srr.where_mask(where, vals, dn, FLOAT_COLS).sum()) and n > 0
    cols = [torch.full((n,), SENTINEL, dtype=torch.int64, device="cuda") for _ in atts]
    nul = [torch.full((n,), 7, dtype=torch.uint8, device="cuda") for _ in atts]
    ptrs, nptrs = [c.data_ptr() for c in cols], [x.data_ptr() for x in nul]
    rc, got = _raw_call(cg, shard, d, atts, n - 1, ptrs, nptrs)
    torch.cuda.synchronize()
    assert rc == capi.CG_EINVAL and got == n
    assert all((c.cpu().numpy() == SENTINEL).all() for c in cols) and all((x.cpu().numpy() == 7).all() for x in nul)
    rc, got = _raw_call(cg, shard, d, atts, n, ptrs, nptrs)
    torch.cuda.synchronize()
    assert rc == 0 and got == n
    want_v, want_n = srr.expected_rows(vals, dn, where, atts, FLOAT_COLS)
    for i in range(2):
        assert np.array_equal(cols[i].cpu().numpy(), want_v[i]) and np.array_equal(nul[i].cpu().numpy(), want_n[i])
    shard.free()


def test_refusals(cg, typed):
    import torch
    from citus_b200 import capi
    rel, vals, dn = typed
    shard = cg.Shard(rel)
    buf = torch.zeros(30_000, dtype=torch.int64, device="cuda")
    nb = torch.zeros(30_000, dtype=torch.uint8, device="cuda")
    plain = cg.make_desc([(4, "<", 0)])
    for desc in (cg.make_desc([(4, "<", 0)], (), [cg.count_star()]),        # aggregates
                 cg.make_desc([(4, "<", 0)], [1], ())):                       # group columns
        assert _raw_call(cg, shard, desc, [4], 30_000, [buf.data_ptr()], None)[0] == capi.CG_EINVAL
    assert _raw_call(cg, shard, plain, [4] * 17, 30_000, [buf.data_ptr()] * 17, None)[0] == capi.CG_EINVAL
    assert _raw_call(cg, shard, plain, [4] * 16, 30_000, [buf.data_ptr()] * 16, None)[0] == 0
    assert _raw_call(cg, shard, plain, [9], 30_000, [buf.data_ptr()], None)[0] == capi.CG_EINVAL      # out of range
    assert _raw_call(cg, shard, plain, [3], 30_000, [buf.data_ptr()], None)[0] == capi.CG_EINVAL      # NULLs, no array
    assert _raw_call(cg, shard, plain, [3], 30_000, [buf.data_ptr()], [None])[0] == capi.CG_EINVAL
    assert _raw_call(cg, shard, plain, [3], 30_000, [buf.data_ptr()], [nb.data_ptr()])[0] == 0
    assert _raw_call(cg, shard, plain, [3], 0, None, None)[0] == 0                                    # counting needs none
    part = cg.Shard(rel, columns=[4, 8])
    assert _raw_call(cg, part, plain, [2], 30_000, [buf.data_ptr()], [nb.data_ptr()])[0] == capi.CG_EINVAL  # not staged
    assert _raw_call(cg, part, cg.make_desc([(2, "<", 0)]), [4], 30_000, [buf.data_ptr()], None)[0] == capi.CG_EINVAL
    part.free()
    shard.free()


def test_aggregate_cache_survives_row_scans(cg, typed):
    """cg_scan_shard's cached chunk-group selection is untouched by row scans with other WHEREs in between"""
    rel, vals, dn = typed
    shard = cg.Shard(rel)
    aggs = [cg.count_star(), cg.sum_(3), cg.min_(2)]
    where_a = [(4, "<", 0), (2, "is not null")]
    d = cg.make_desc(where_a, [0], aggs)

    def agg_scan(sh):
        a = cg.GpuColumnarAgg(d, rel.column_descs(), 0, 1, 20_000)
        st = a.scan_shard(sh)
        g = a.groups()
        a.free()
        return g, (st.rows_scanned, st.rows_passed, st.chunk_groups_filtered)

    fresh_shard = cg.Shard(rel)
    want = agg_scan(fresh_shard)
    fresh_shard.free()
    assert agg_scan(shard) == want
    for where in ([(4, ">", 0)], ("or", (3, "is null"), (1, "in", (5, 6))), None):
        check(cg, shard, vals, dn, where, [4, 3], 6000, 1000)
        assert agg_scan(shard) == want
    shard.free()


def test_map_task_copy_files(cg, oracle, typed):
    """worker_partition_query_result over a columnar shard with nothing on the host: rows -> cg_partition_index ->
    cg_partition_copy_serialize equal the oracle's COPY files of the oracle-filtered rows, text and binary, NULLs in the
    payload"""
    import torch
    rel, vals, dn = typed
    shard = cg.Shard(rel)
    where = ("or", (2, "<", 0), (6, "is null"))
    atts, lens = [4, 3, 2, 6], [8, 4, 2, 8]
    n, _, _, _ = scan_rows(cg, shard, where, atts)
    cols = [torch.empty(n, dtype=torch.int64, device="cuda") for _ in atts]
    nul = [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in atts]
    got, _ = shard.scan_rows(cg.make_desc(where, float_cols=FLOAT_COLS), atts, [c.data_ptr() for c in cols],
                             [x.data_ptr() for x in nul], n)
    assert got == n
    P = 8
    mins, maxs = oracle.synthetic_intervals(P)
    idx = torch.empty(n, dtype=torch.int32, device="cuda")
    cnt = torch.empty(P, dtype=torch.int64, device="cuda")
    cg.worker_partition_query_result(cols[0].data_ptr(), nul[0].data_ptr(), n, 8, "hash", mins, maxs, idx.data_ptr(),
                                     cnt.data_ptr())
    want_v, want_n = srr.expected_rows(vals, dn, where, atts, FLOAT_COLS, SCALES)
    want_idx, want_rows = oracle.partition_rows(want_v[0], want_n[0], 8, "h", mins, maxs)
    assert np.array_equal(idx.cpu().numpy(), want_idx) and np.array_equal(cnt.cpu().numpy(), want_rows)
    for binary in (False, True):
        out = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
        offs = cg.partition_copy_serialize(idx.data_ptr(), n, P, [c.data_ptr() for c in cols], lens, binary, out.data_ptr(),
                                           out.numel(), d_null_ptrs=[x.data_ptr() for x in nul])
        host = out.cpu().numpy().tobytes()
        want = oracle.copy_files(want_idx, want_v, lens, P, binary, nulls=want_n)
        assert [host[offs[p]:offs[p + 1]] for p in range(P)] == want, binary
    shard.free()


@pytest.fixture(scope="module")
def comm(cg):
    from citus_b200 import distributed
    distributed.init(0, 1)
    yield distributed
    distributed.destroy()


def test_repartition_join(cg, oracle, comm):
    """two shards' map queries (WHERE with key IS NOT NULL) -> the one-rank exchange -> cg_join_aggregate, against the
    join reference and the exact aggregate reference over the oracle-filtered rows"""
    import torch
    from citus_b200 import capi
    rng = np.random.default_rng(31)
    attlens, types = [8, 4, 8], [0, 0, 0]
    sides = []
    for s, n in enumerate((30_000, 25_000)):
        cols = [rng.integers(-3000, 3000, n), rng.integers(-100, 100, n), rng.integers(-2**40, 2**40, n)]
        nulls = [(rng.random(n) < 0.05).astype(np.uint8), (rng.random(n) < 0.1).astype(np.uint8), np.zeros(n, np.uint8)]
        rel, t = write(cg, oracle, cols, nulls, 10_000, 1000, attlens=attlens, types=types)
        vals, dn = t.decode_all()
        where = [(0, "is not null"), (1, ">" if s == 0 else "<", -20 if s == 0 else 50)]
        shard = cg.Shard(rel)
        m, _ = shard.scan_rows(cg.make_desc(where), [0, 2])
        out = [torch.empty(m, dtype=torch.int64, device="cuda") for _ in range(2)]
        # the key column has NULLs in the chunk groups scanned, so it needs a null array even though WHERE drops them
        nul = [torch.full((m,), 7, dtype=torch.uint8, device="cuda") for _ in range(2)]
        got, _ = shard.scan_rows(cg.make_desc(where), [0, 2], [o.data_ptr() for o in out], [x.data_ptr() for x in nul], m)
        assert got == m
        want_v, want_n = srr.expected_rows(vals, dn, where, [0, 2])
        assert not want_n[0].any() and not want_n[1].any()
        assert all((x.cpu().numpy() == 0).all() for x in nul)
        assert np.array_equal(out[0].cpu().numpy(), want_v[0]) and np.array_equal(out[1].cpu().numpy(), want_v[1])
        sides.append((shard, out, m, want_v))
    P = 8
    mins = np.ascontiguousarray(oracle.synthetic_intervals(P)[0], np.int32)
    maxs = np.ascontiguousarray(oracle.synthetic_intervals(P)[1], np.int32)
    lib = capi.lib()
    counts = []
    for slot, (_, out, m, _) in enumerate(sides):
        cp = (C.c_void_p * 2)(*[o.data_ptr() for o in out])
        recv = C.c_int64(-1)
        assert lib.cg_comm_repartition_exchange(slot, cp, None, m, 2, 8, P, mins.ctypes.data, maxs.ctypes.data,
                                                C.byref(recv)) == 0
        assert recv.value == m
        assert lib.cg_comm_exchange_wait(slot) == 0
    ptrs = []
    for slot in range(2):
        p = (C.c_void_p * 8)()
        cnt = np.zeros(P, np.int64)
        assert lib.cg_comm_exchange_result(slot, p, None, cnt.ctypes.data, None, None, None) == 0
        ptrs.append(p)
        counts.append(np.concatenate([[0], np.cumsum(cnt)]))
    aggs = [cg.count_star(), cg.sum_(1), cg.sum_(3), cg.min_(3)]
    desc = cg.make_desc((), (), aggs)
    part = cg.GpuColumnarAgg(desc, [(8, 0)] * 4, 0, -1, 0)
    for q in range(P):
        ob, op = counts[0], counts[1]
        nb, npr = int(ob[q + 1] - ob[q]), int(op[q + 1] - op[q])
        if nb == 0 or npr == 0:
            continue
        b = [ptrs[0][c] + 8 * int(ob[q]) for c in range(2)]
        p = [ptrs[1][c] + 8 * int(op[q]) for c in range(2)]
        part.join_aggregate(b, 0, nb, p, 0, npr)
    got = list(part.groups().values())
    jc, jn = jref.join(sides[0][3], None, 0, sides[1][3], None, 0)
    want = ref.aggregate(jc, jn, None, [], aggs)
    w = want.groups[()]
    assert len(got) == 1 and got[0][0]["count"] == w[0].count
    assert got[0][1]["sum"] == w[1].sum and got[0][2]["sum"] == w[2].sum and got[0][3]["minmax"] == w[3].min
    part.free()
    for shard, _, _, _ in sides:
        shard.free()
