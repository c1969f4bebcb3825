"""The fast scan kernel's narrow (bit-packed, frame-of-reference) images against an exact reference.

  * the images themselves, read back word for word, against narrow_reference.pack: every width 0..32, a width that
    changes from chunk group to chunk group, bases at INT64_MIN and streams ending at INT64_MAX, a column one of whose
    chunk groups spans 2^32 (no images anywhere), a column with NULLs in some chunk groups, and chunk groups of 1, 63,
    64, 65, 127, 128 and 1000 rows, some of them between stripes; staged subsets in another order; lz4 and zstd;
  * every width as a qual column, as a group key and as a sum argument, against reference.aggregate;
  * every narrow instance of cg_scan_fast_kernel (quals x mode x sums x packing x row pairs per lane x paired updates)
    against reference.aggregate and, bit for bit, against the same data staged without images, with bytes_scanned
    proving which path ran;
  * shards with images, without them, with NULL chunk groups and staged plain, back to back into one partial;
  * cg_scan_relation's transient staging, which builds no images."""
import dataclasses
from dataclasses import dataclass

import numpy as np
import pytest

import narrow_reference as nr
import reference as ref

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
GLOBAL, DENSE, HASH = "global", "dense", "hash"


@pytest.fixture(scope="module")
def cg():
    import torch
    assert torch.cuda.is_available(), "these tests need an H100"
    from citus_b200 import build
    build.build()
    from citus_b200 import columnar
    columnar.init(0)
    yield columnar
    columnar.set_option("narrow_images", 1)
    columnar.set_writer_compression("none")


@dataclass
class RelData:
    rel: object
    cols: list
    nulls: list
    stripe: int
    chunk: int

    @property
    def n(self):
        return len(self.cols[0])

    @property
    def layout(self):
        return ref.chunk_layout(self.n, self.stripe, self.chunk)

    def narrow_layout(self, staged=None):
        return nr.narrow_layout(self.cols, self.nulls, self.layout, list(range(len(self.cols))) if staged is None else staged)

    def prefix(self, nstripes):
        rows = sum(r for s in self.layout[:nstripes] for _, r in s)
        return RelData(self.rel.prefix(nstripes), [c[:rows] for c in self.cols],
                       [None if x is None else x[:rows] for x in self.nulls], self.stripe, self.chunk)


def write(cg, cols, nulls, stripe, chunk, compression="none"):
    cg.set_writer_compression(compression)
    try:
        rel = cg.Relation.write([8] * len(cols), cols, nulls=nulls, stripe_row_limit=stripe, chunk_row_limit=chunk)
    finally:
        cg.set_writer_compression("none")
    return RelData(rel, cols, nulls, stripe, chunk)


def stage(cg, rd, images=True, columns=None):
    cg.set_option("narrow_images", 1 if images else 0)
    try:
        return cg.Shard(rd.rel, columns)
    finally:
        cg.set_option("narrow_images", 1)


def fill(col, first, rows, base, span, rng):
    """rows [first, first + rows) in [base, base + span], both ends present, at random rows, when there are two rows or
    more (so that every warp of the min / max reduction holds an extreme somewhere)"""
    col[first:first + rows] = np.int64(base) + rng.integers(0, span + 1, rows, dtype=np.int64) if span else base
    if rows >= 2:
        i, j = rng.choice(rows, 2, replace=False)
        col[first + i], col[first + j] = base, base + span


# --------------------------------------------------------------------------- query helpers
def query_atts(where, group, aggs):
    return sorted({a[0] for a in where} | set(group) | {f[0] for a in aggs for f in a.factors})


def renumber(where, group, aggs):
    """the query over its own columns only, renumbered 0..n-1 (the reference then converts just those)"""
    m = {a: i for i, a in enumerate(query_atts(where, group, aggs))}
    return ([(m[c], op, k) for c, op, k in where], [m[c] for c in group],
            [dataclasses.replace(a, factors=[(m[c], x, y) for c, x, y in a.factors]) for a in aggs])


def reference(rds, where, group, aggs):
    atts = query_atts(where, group, aggs)
    w, g, a = renumber(where, group, aggs)
    cols = [np.concatenate([rd.cols[c] for rd in rds]) for c in atts]
    nulls = [None if all(rd.nulls[c] is None for rd in rds) else
             np.concatenate([np.zeros(rd.n, np.uint8) if rd.nulls[c] is None else rd.nulls[c] for rd in rds]) for c in atts]
    return ref.aggregate(cols, nulls, w, g, a)


def chunk_mask(rd, where, group, aggs):
    """SelectedChunkMask of the relation for this WHERE list, one flag per chunk group"""
    atts = query_atts(where, group, aggs)
    w, _, _ = renumber(where, group, aggs)
    mask = ref.selected_chunk_mask([rd.cols[c] for c in atts], [rd.nulls[c] for c in atts], w, rd.stripe, rd.chunk)
    return [k for s in mask for k in s]


def run(cg, shards, rds, where, group, aggs, mode, packing=True, want_stats=True):
    """one partial over the shards, scanned back to back: (stats per shard, groups keyed like the reference, layout)"""
    aggs = [dataclasses.replace(a) for a in aggs]
    d = cg.make_desc(where, group, aggs)
    kmin = kmax = None
    bounds = [0] * len(aggs)
    for rd in rds:
        a, b, bs, _ = cg.relation_bounds(rd.rel, d)
        if a <= b:
            kmin = a if kmin is None else min(kmin, a)
            kmax = b if kmax is None else max(kmax, b)
        bounds = [max(x, y) for x, y in zip(bounds, bs)]
    for a, b in zip(aggs, bounds):
        a.term_abs_bound = b
    nrows = sum(rd.n for rd in rds)
    d = cg.make_desc(where, group, aggs, expected_groups=nrows if mode == HASH else 0)
    if mode != DENSE or kmin is None:
        kmin, kmax = 0, -1
    agg = cg.GpuColumnarAgg(d, rds[0].rel.column_descs(), kmin, kmax, nrows)
    try:
        if not packing:
            agg.set_packing(False)
        stats = [agg.scan_shard(sh, want_stats) for sh in shards]
        got = agg.groups()
        layout = agg.layout()
    finally:
        agg.free()
    keyed = {(k,) if group else (): per for k, per in got.items()}
    return stats, keyed, layout


def assert_answer(got, want, aggs):
    if not want.groups:             # a plain aggregate over no rows: one row of zero counts, or none
        assert all(g["count"] == 0 for per in got.values() for g in per)
        return
    assert set(got) == set(want.groups)
    for key, per in want.groups.items():
        for i, (spec, st) in enumerate(zip(aggs, per)):
            assert got[key][i]["count"] == st.count, (key, i)
            if spec.kind == ref.SUM and st.count:
                assert got[key][i]["sum"] == st.sum, (key, i)


def check_query(cg, shards, rds, layouts, where, group, aggs, mode, narrow=True, packing=True):
    """the exact answer (or CG_EUNSUPPORTED where an argument leaves int64), the chunk-group counters from the rows, and
    bytes_scanned: the narrow streams when narrow, the plain columns otherwise.  Returns (stats, groups)."""
    from citus_b200 import capi
    want = reference(rds, where, group, aggs)
    if ref.overflows(want):
        with pytest.raises(capi.CitusGpuError) as e:
            run(cg, shards, rds, where, group, aggs, mode, packing)
        assert e.value.code == capi.CG_EUNSUPPORTED
        return None, None
    stats, got, _ = run(cg, shards, rds, where, group, aggs, mode, packing)
    assert_answer(got, want, aggs)
    atts = query_atts(where, group, aggs)
    assert sum(st.rows_passed for st in stats) == want.rows_passed
    for st, rd, lay in zip(stats, rds, layouts):
        mask = chunk_mask(rd, where, group, aggs)
        kept_rows = sum(r for (_, r), k in zip([g for s in rd.layout for g in s], mask) if k)
        assert (st.rows_scanned, st.chunk_groups_scanned, st.chunk_groups_filtered) == \
               (kept_rows, sum(mask), len(mask) - sum(mask))
        assert st.bytes_scanned == lay.scan_bytes(atts, mask, narrow and lay.narrow_plan(atts))
    return stats, got


# --------------------------------------------------------------------------- 1. the images, word for word
NWIDTH = 33                                    # attribute w < 33 has width w in every chunk group of two rows or more
VARYING, AT_MIN, AT_MAX, SPAN33, NULLY = 33, 34, 35, 36, 37
NATTS = 38
VARYING_WIDTHS = [0, 1, 17, 32, 5, 31, 2, 13]
# (stripe_row_limit, rows) at 1000-row chunk groups: 1000|1|1000|1|64, 1000|63|1000|63|65 and 1000|128|127
LAYOUTS = [(1001, 2 * 1001 + 64), (1063, 2 * 1063 + 65), (1128, 1128 + 127)]


def width_columns(nrows, groups, seed):
    rng = np.random.default_rng(seed)
    cols = [np.zeros(nrows, np.int64) for _ in range(NATTS)]
    nulls = [None] * NATTS
    nulls[NULLY] = np.zeros(nrows, np.uint8)
    for w in range(NWIDTH):
        # even widths far out in int64 (two-limb sums), odd ones near zero; every chunk group its own base
        far = int(rng.integers(-(1 << 62), 1 << 62)) if w % 2 == 0 else int(rng.integers(-10**6, 10**6))
        for f, m in groups:
            fill(cols[w], f, m, far + int(rng.integers(0, 1000)), (1 << w) - 1, rng)
    for g, (f, m) in enumerate(groups):
        vw = VARYING_WIDTHS[g % len(VARYING_WIDTHS)]
        fill(cols[VARYING], f, m, int(rng.integers(-(1 << 40), 1 << 40)), (1 << vw) - 1, rng)
        fill(cols[AT_MIN], f, m, I64_MIN, (1 << 32) - 1, rng)
        fill(cols[AT_MAX], f, m, I64_MAX - (1 << 32) + 1, (1 << 32) - 1, rng)
        fill(cols[SPAN33], f, m, 12345, (1 << 32) if g == 0 else 1000, rng)
        fill(cols[NULLY], f, m, -5000, (1 << 20) - 1, rng)
        if g % 2:
            nulls[NULLY][f:f + m] = rng.random(m) < 0.1
            nulls[NULLY][f] = 1
    return cols, nulls


_width_rels = {}


def width_rels(cg, compression):
    if compression not in _width_rels:
        out = []
        for i, (stripe, nrows) in enumerate(LAYOUTS):
            groups = [g for s in ref.chunk_layout(nrows, stripe, 1000) for g in s]
            cols, nulls = width_columns(nrows, groups, 100 + i)
            out.append(write(cg, cols, nulls, stripe, 1000, compression))
        _width_rels[compression] = out
    return _width_rels[compression]


def check_images(cg, sh, rd, lay, atts):
    from citus_b200 import capi
    for g, (f, m) in enumerate(lay.groups):
        for a in atts:
            base, width, words = sh.narrow_image(g, a)
            im = lay.image[(g, a)]
            if im is None:
                assert (width, words.size) == (nr.NONE, 0), (g, a)
                continue
            wb, ww, wwords = nr.pack(rd.cols[a][f:f + m])
            assert (base, width) == (wb, ww) == im, (g, a)
            assert np.array_equal(words, wwords), (g, a, width, np.flatnonzero(words != wwords)[:4])
    for a in atts:
        assert capi.lib().cg_shard_narrow_column(sh.h, a) == lay.col_narrow[a], a
    assert capi.lib().cg_shard_narrow_bytes(sh.h) == lay.narrow_bytes


@pytest.mark.parametrize("compression", ["none", "lz4", "zstd"])
def test_images_word_for_word(cg, compression):
    from citus_b200 import capi
    seen = set()
    for rd in width_rels(cg, compression):
        lay = rd.narrow_layout()
        assert lay.col_narrow == {a: a != SPAN33 for a in range(NATTS)}
        for g, (_, m) in enumerate(lay.groups):
            for w in range(NWIDTH):
                assert lay.image[(g, w)][1] == (w if m > 1 else 0)
            seen.add(m)
        sh = stage(cg, rd)
        plain = stage(cg, rd, images=False)
        check_images(cg, sh, rd, lay, range(NATTS))
        # the arena is the same; the images add exactly the streams and their descriptors
        assert sh.device_bytes - plain.device_bytes == lay.narrow_bytes > 0
        assert capi.lib().cg_shard_narrow_bytes(plain.h) == 0
        assert all(capi.lib().cg_shard_narrow_column(plain.h, a) == 0 for a in range(NATTS))
        assert all(plain.narrow_image(g, a)[1] == nr.NONE for g in range(len(lay.groups)) for a in (0, 32, AT_MIN))
        # staged subsets in another order: the slot differs from the attribute, the images per attribute do not
        for cols in ([5, 2, 0], [SPAN33, 17, NULLY, VARYING, 0, AT_MIN, 32, AT_MAX]):
            sub = stage(cg, rd, columns=cols)
            check_images(cg, sub, rd, rd.narrow_layout(cols), cols)
            with pytest.raises(capi.CitusGpuError) as e:
                sub.narrow_image(0, 1)                      # not staged
            assert e.value.code == capi.CG_EINVAL
            sub.free()
        for bad in ((len(lay.groups), 0), (-1, 0), (0, NATTS)):
            with pytest.raises(capi.CitusGpuError):
                sh.narrow_image(*bad)
        sh.free()
        plain.free()
    assert {1, 63, 64, 65, 127, 128, 1000} <= seen


# --------------------------------------------------------------------------- 2. every width in every role
@pytest.fixture(scope="module")
def width_shards(cg):
    rds = width_rels(cg, "none")
    shards = [stage(cg, rd) for rd in rds]
    return rds, shards, [rd.narrow_layout() for rd in rds]


@pytest.mark.parametrize("w", range(NWIDTH))
def test_every_width_in_every_role(cg, width_shards, w):
    rds, shards, lays = width_shards
    other, key = (w + 11) % NWIDTH, (w + 3) % NWIDTH
    vals = np.concatenate([rd.cols[w] for rd in rds])
    mid = int(vals.min()) + (int(vals.max()) - int(vals.min())) // 2
    v = int(vals[1234])
    omid = int(np.median(np.concatenate([rd.cols[other] for rd in rds])))
    aggs_w = [cg.count_star(), cg.sum_(other)]
    for where in ([(w, "<", mid)], [(w, ">=", mid)], [(w, "=", v)], [(w, "<>", v)]):
        check_query(cg, shards, rds, lays, where, [], aggs_w, GLOBAL)
        check_query(cg, shards, rds, lays, where, [key], aggs_w, HASH)
    for mode in (DENSE, HASH):
        check_query(cg, shards, rds, lays, [], [w], aggs_w, mode)
    check_query(cg, shards, rds, lays, [(other, ">=", omid)], [], [cg.count_star(), cg.sum_(w)], GLOBAL)
    check_query(cg, shards, rds, lays, [], [key], [cg.sum_(w), cg.count_star()], HASH)
    check_query(cg, shards, rds, lays, [], [], [cg.sum_(w), cg.sum_(VARYING), cg.sum_(AT_MIN)], GLOBAL)


# --------------------------------------------------------------------------- 3. every narrow instance
Q0, Q1, KEY, HKEY, S0, S1, S2, B0, B1, B2 = range(10)
SMALL_SUMS, BIG_SUMS = [S0, S1, S2], [B0, B1, B2]


def instance_columns(nrows, groups, seed):
    """q0 [0, 1000), q1 +-70000, a dense key of 2100 values, a hash key whose chunk groups sit at INT64_MIN (the hash
    table's EMPTY value), at INT64_MAX and around zero, single-limb sums of widths 19, 5 and 32, and two-limb sums near
    INT64_MAX and INT64_MIN (and one of width 13 at 2^40)"""
    rng = np.random.default_rng(seed)
    cols = [np.zeros(nrows, np.int64) for _ in range(10)]
    for g, (f, m) in enumerate(groups):
        fill(cols[Q0], f, m, 0, 999, rng)
        fill(cols[Q1], f, m, -70000, 140000, rng)
        fill(cols[KEY], f, m, -700, 2099, rng)
        fill(cols[HKEY], f, m, [I64_MIN, I64_MAX - 1999, -1000][g % 3], 1999, rng)
        fill(cols[S0], f, m, -(1 << 18), (1 << 19) - 1, rng)
        fill(cols[S1], f, m, 0, 31, rng)
        fill(cols[S2], f, m, -(1 << 31), (1 << 32) - 1, rng)
        fill(cols[B0], f, m, I64_MAX - (1 << 31) + 1, (1 << 31) - 1, rng)
        fill(cols[B1], f, m, I64_MIN, (1 << 32) - 1, rng)
        fill(cols[B2], f, m, 1 << 40, (1 << 13) - 1, rng)
    return cols, [None] * 10


QUALS = {
    0: [[]],
    1: [[(Q0, "<", 300)],
        [(Q0, ">=", 100), (Q0, "<", 900)],            # one column constrained twice
        [(Q0, "<>", 7)],
        [(Q0, ">=", 600), (Q0, "<", 200)],             # an empty range that no chunk group's min / max refutes
        [(Q0, "<", I64_MIN)]],                         # empty, and every chunk group is skipped
    2: [[(Q0, "<", 500), (Q1, ">=", 0)],
        [(Q0, ">=", 100), (Q0, "<=", 800), (Q1, "<>", 5)],
        [(Q0, "<>", 3), (Q1, "<", -1000)],
        [(Q0, "<", 900), (Q1, ">=", 50), (Q1, "<", 0)]],
}


def narrow_instances():
    """(nq, mode, ns, pack, U, paired) of every instance launch_fast_variant launches on narrow images: plans of one to
    three columns; PACK in the grouped modes with a single-limb sum; U = 2 row pairs per lane up to two columns;
    paired updates for hash tables with single-limb sums only"""
    out = []
    for nq in range(3):
        for mode in (GLOBAL, DENSE, HASH):
            for ns in range(4):
                nc = nq + (mode != GLOBAL) + ns
                if not 1 <= nc <= 3:
                    continue
                u = 2 if nc <= 2 else 1
                out.append((nq, mode, ns, False, u, mode == HASH and ns > 0))
                if mode != GLOBAL and ns > 0:
                    out.append((nq, mode, ns, True, u, False))
                if mode == HASH and ns > 0:
                    out.append((nq, mode, ns, False, u, False))
    return out


@pytest.fixture(scope="module")
def instance_data(cg):
    nrows, stripe = 14_037, 6000                       # chunk groups of 6000, 6000 and 2037 rows, one per stripe
    groups = [g for s in ref.chunk_layout(nrows, stripe, stripe) for g in s]
    cols, nulls = instance_columns(nrows, groups, 7)
    full = write(cg, cols, nulls, stripe, stripe)
    rds = [full.prefix(1), full.prefix(2), full]       # launches of one, two and three chunk groups
    out = []
    for rd in rds:
        out.append((rd, stage(cg, rd), stage(cg, rd, images=False), rd.narrow_layout()))
    return out


def test_every_narrow_instance(cg, instance_data):
    from citus_b200 import capi
    for rd, sh, plain, lay in instance_data:
        assert all(lay.col_narrow.values()) and capi.lib().cg_shard_narrow_bytes(sh.h) == lay.narrow_bytes
    covered = set()
    instances = narrow_instances()
    for t, (nq, mode, ns, pack, u, paired) in enumerate(instances):
        two_limbs = mode == HASH and ns > 0 and not pack and not paired
        sums = (BIG_SUMS if two_limbs else SMALL_SUMS)[:ns]
        group = [] if mode == GLOBAL else [HKEY if mode == HASH else KEY]
        aggs = [cg.count_star()] + [cg.sum_(c) for c in sums]
        for v, where in enumerate(QUALS[nq]):
            targets = instance_data if nq == 0 else [instance_data[(t + v) % 3]]
            for rd, sh, plain, lay in targets:
                stats, got = check_query(cg, [sh], [rd], [lay], where, group, aggs, mode, packing=pack)
                # the same rows staged without images: the plain fast kernel, bit for bit
                pstats, pgot, _ = run(cg, [plain], [rd], where, group, aggs, mode, packing=pack)
                assert pgot == got
                a, b = stats[0], pstats[0]
                assert (a.rows_scanned, a.rows_removed_by_filter, a.chunk_groups_scanned, a.chunk_groups_filtered) == \
                       (b.rows_scanned, b.rows_removed_by_filter, b.chunk_groups_scanned, b.chunk_groups_filtered)
                atts = query_atts(where, group, aggs)
                assert b.bytes_scanned == lay.scan_bytes(atts, chunk_mask(rd, where, group, aggs), narrow=False)
        covered.add((nq, mode, ns, pack, u, paired))
    assert covered == set(instances)
    # 8 plain-aggregate, 9 direct-indexed and 9 hash-table template instances; the hash tables' unpacked single-limb
    # shapes run both the paired and the unpaired update
    assert len({i[:4] for i in covered}) == 26 and len(covered) == 29


def test_hash_key_at_the_empty_value(cg, instance_data):
    """the hash key column's first chunk group holds INT64_MIN, the table's EMPTY value, and its second INT64_MAX"""
    rd, sh, plain, lay = instance_data[2]
    assert rd.cols[HKEY].min() == I64_MIN and rd.cols[HKEY].max() == I64_MAX
    _, got = check_query(cg, [sh], [rd], [lay], [], [HKEY], [cg.count_star(), cg.sum_(S2)], HASH)
    assert (I64_MIN,) in got and (I64_MAX,) in got


# --------------------------------------------------------------------------- 4. mixed shards in one partial
def mixed_rels(cg):
    """four relations of one schema (key, q, s): s with images; s spanning 2^33 in one chunk group (no images for s);
    s with NULLs in two chunk groups (narrow prefix, generated nullable rest); and one to be staged without images"""
    out = []
    for i in range(4):
        rng = np.random.default_rng(40 + i)
        nrows, stripe = 6321 + 97 * i, 2500
        groups = [g for s in ref.chunk_layout(nrows, stripe, 1000) for g in s]
        cols = [np.zeros(nrows, np.int64) for _ in range(3)]
        nulls = [None, None, None]
        for g, (f, m) in enumerate(groups):
            fill(cols[0], f, m, 100 * i, 1500, rng)
            fill(cols[1], f, m, 0, 99, rng)
            fill(cols[2], f, m, -10**6, 2 * 10**6, rng)
        if i == 1:
            g1 = groups[1]
            fill(cols[2], g1[0], g1[1], -(1 << 32), 1 << 33, rng)
        if i == 2:
            nulls[2] = np.zeros(nrows, np.uint8)
            for f, m in (groups[2], groups[4]):
                nulls[2][f:f + m] = rng.random(m) < 0.2
        out.append(write(cg, cols, nulls, stripe, 1000))
    return out


def test_mixed_shards_back_to_back(cg):
    from citus_b200 import capi
    rds = mixed_rels(cg)
    shards = [stage(cg, rd, images=i != 3) for i, rd in enumerate(rds)]
    assert [capi.lib().cg_shard_narrow_column(sh.h, 2) for sh in shards] == [1, 0, 1, 0]
    assert [capi.lib().cg_shard_narrow_column(sh.h, 0) for sh in shards] == [1, 1, 1, 0]
    for mode, group, where in ((DENSE, [0], [(1, "<", 60)]), (HASH, [0], [(1, "<", 60)]), (GLOBAL, [], [(1, ">=", 20)]),
                               (GLOBAL, [], [])):
        aggs = [cg.count_star(), cg.sum_(2)]
        want = reference(rds, where, group, aggs)
        # the first scan of a shard under a WHERE list uploads its chunk-group selection (a host sync); after that the
        # four launches of one query go out back to back, with no statistics read in between
        run(cg, shards, rds, where, group, aggs, mode)
        _, got, _ = run(cg, shards, rds, where, group, aggs, mode, want_stats=False)
        assert_answer(got, want, aggs)
        stats, got2, _ = run(cg, shards, rds, where, group, aggs, mode)
        assert got2 == got
        lays = [rd.narrow_layout() for rd in rds]
        lays[3] = nr.narrow_layout(rds[3].cols, rds[3].nulls, rds[3].layout, [0, 1, 2], candidate=[0, 0, 0])
        atts = query_atts(where, group, aggs)
        for st, rd, lay in zip(stats, rds, lays):
            assert st.bytes_scanned == lay.scan_bytes(atts, chunk_mask(rd, where, group, aggs), lay.narrow_plan(atts))


# --------------------------------------------------------------------------- 5. transient staging
def test_transient_staging_builds_no_images(cg, instance_data):
    rd, sh, plain, lay = instance_data[2]
    where, group, aggs = [(Q0, "<", 500)], [KEY], [cg.count_star(), cg.sum_(S2)]
    stats, got, _ = run(cg, [sh], [rd], where, group, aggs, DENSE)
    atts = query_atts(where, group, aggs)
    mask = chunk_mask(rd, where, group, aggs)
    assert lay.narrow_plan(atts) and stats[0].bytes_scanned == lay.scan_bytes(atts, mask, narrow=True)
    d_aggs = [dataclasses.replace(a) for a in aggs]
    d = cg.make_desc(where, group, d_aggs)
    kmin, kmax, bounds, rows = cg.relation_bounds(rd.rel, d)
    for a, b in zip(d_aggs, bounds):
        a.term_abs_bound = b
    d = cg.make_desc(where, group, d_aggs)
    rd.rel.register()
    try:
        agg = cg.GpuColumnarAgg(d, rd.rel.column_descs(), kmin, kmax, rows)
        st = agg.scan_relation(rd.rel)
        got2 = {(k,): per for k, per in agg.groups().items()}
        agg.free()
    finally:
        rd.rel.unregister()
    assert got2 == got
    assert st.bytes_scanned == lay.scan_bytes(atts, mask, narrow=False)
    assert_answer(got, reference([rd], where, group, aggs), aggs)
