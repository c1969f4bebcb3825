"""WHERE evaluation and chunk-group skipping on the GPU against the exact reference (tests/reference.py), which
evaluates every row and skips nothing, and whose skip mask is computed from the rows.  Every case runs on every
kernel family and checks three things: the rows passed and the groups equal the reference's; "Chunk Groups Removed
by Filter" equals reference.selected_chunk_mask's count; and with qual pushdown off only the counters change.  The
cases sit where kernels go wrong: integer constants at and beyond the edges of the column's type, constants equal to
a chunk's min or max, WHERE lists the fast kernel's range reduction has to merge or refuse, NULL-bearing chunk groups
under AND / OR trees, and varlena char(1) / numeric columns."""
import numpy as np
import pytest

import reference as ref
from test_gpu_exact import assert_matches_reference
from test_where_reference import HAND_DATUMS, INT64_MAX, INT64_MIN, LIMITS, OPS, constant_pools, image_with_datums, random_tree
from gpu_harness import cg, kernel_family, FAMILIES  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

BPCHAR1 = 3


class Table:
    """a relation together with the rows it was written from (what the reference reads)"""

    def __init__(self, rel, cols, nulls, stripe_rows, chunk_rows, float_cols=(), key=None):
        self.rel, self.cols, self.nulls, self.key = rel, cols, nulls, key
        self.stripe_rows, self.chunk_rows, self.float_cols = stripe_rows, chunk_rows, tuple(float_cols)
        self.n = len(cols[0])
        self.minmax = ref.skip_minmax(cols, nulls, stripe_rows, chunk_rows, float_cols)

    @classmethod
    def write(cls, cg, attlens, cols, nulls=None, float_cols=(), stripe_rows=3000, chunk_rows=1000, key=None):
        """key: names data that is the same in every kernel family (fixed seed), so the reference is computed once"""
        tc = [1 if c in float_cols else 0 for c in range(len(attlens))]
        rel = cg.Relation.write(attlens, cols, nulls, type_classes=tc, stripe_row_limit=stripe_rows, chunk_row_limit=chunk_rows)
        return cls(rel, cols, nulls, stripe_rows, chunk_rows, float_cols, key)

    @classmethod
    def oracle(cls, cg, oracle, attlens, types, cols, nulls=None, stripe_rows=3000, chunk_rows=1000, key=None):
        t = oracle.Table(attlens, types, stripe_row_limit=stripe_rows, chunk_row_limit=chunk_rows)
        t.insert(cols, nulls)
        rel = cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), attlens, types)
        return cls(rel, cols, nulls, stripe_rows, chunk_rows, [c for c, ty in enumerate(types) if ty == 1], key)


def gpu_scan(cg, tab, where, group_cols, aggs, pushdown=True, path="shard", force_hash=False):
    """one partial aggregate; returns (stats, groups keyed like the reference)"""
    d = cg.make_desc(where, group_cols, aggs, qual_pushdown=pushdown, float_cols=tab.float_cols, expected_groups=4096)
    kmin, kmax, _, rows = cg.relation_bounds(tab.rel, d)
    if force_hash:
        kmin, kmax = 0, -1
    agg = cg.GpuColumnarAgg(d, tab.rel.column_descs(), kmin, kmax, max(rows, 1))
    try:
        if path == "shard":
            shard = cg.Shard(tab.rel)
            st = agg.scan_shard(shard)
            shard.free()
        elif path == "e2e":
            st = agg.scan_relation(tab.rel)
        else:
            tab.rel.register()
            try:
                st = agg.scan_relation(tab.rel)
            finally:
                tab.rel.unregister()
        got = agg.groups()
    finally:
        agg.free()
    keyed = {}
    for k, per in got.items():
        if not group_cols:
            keyed[()] = per
        elif len(group_cols) == 1:
            keyed[(k,)] = per
        else:
            keyed[ref.unpack_two_column_key(k)] = per
    return st, keyed


_REFERENCE = {}


def _reference(tab, where, group_cols, aggs):
    """reference.aggregate, computed once per table and query across the kernel families"""
    key = (tab.key, repr(where), tuple(group_cols), repr(aggs))
    if tab.key is None or key not in _REFERENCE:
        _REFERENCE[key] = ref.aggregate(tab.cols, tab.nulls, where, group_cols, aggs, tab.float_cols)
    return _REFERENCE[key]


def check(cg, tab, where, group_cols, aggs, path="shard", force_hash=False, what=""):
    """the three checks of every case; `what` names the case in a failure"""
    try:
        want = _reference(tab, where, group_cols, aggs)
        assert not ref.overflows(want)
        mask = ref.selected_chunk_mask(tab.cols, tab.nulls, where, tab.stripe_rows, tab.chunk_rows, tab.float_cols,
                                       minmax=tab.minmax)
        st, got = gpu_scan(cg, tab, where, group_cols, aggs, True, path, force_hash)
        assert st.chunk_groups_filtered == ref.chunks_filtered(mask)
        assert st.rows_scanned == ref.rows_kept(mask, tab.n, tab.stripe_rows, tab.chunk_rows)
        assert_matches_reference(st, got, want, aggs, tab.n)
        st2, got2 = gpu_scan(cg, tab, where, group_cols, aggs, False, path, force_hash)
        assert (st2.chunk_groups_filtered, st2.rows_scanned, st2.rows_passed) == (0, tab.n, st.rows_passed)
        assert_matches_reference(st2, got2, want, aggs, tab.n)
        return st
    except AssertionError as e:
        raise AssertionError(f"{what} where={where} group={group_cols} path={path} hash={force_hash}: {e}") from e


# --------------------------------------------------------------------------- integer atoms at the edges
def _edge_ints(rng, n, attlen):
    lo, hi = LIMITS[attlen]
    v = rng.integers(lo, hi, n, endpoint=True)
    v[:4] = [lo, hi, lo + 1, hi - 1]
    v[n // 2:n // 2 + 2] = [lo, hi]
    return v


@pytest.mark.parametrize("family", FAMILIES)
def test_integer_atoms_at_the_edges_of_every_width(cg, kernel_family, family):
    """<, <=, =, >=, >, <> against INT64_MIN, INT64_MIN + 1, INT64_MAX - 1, INT64_MAX on int1 / int2 / int4 / int8
    columns that hold their own extremes, and on the narrow ones against constants just outside their range"""
    kernel_family(family)
    rng = np.random.default_rng(101)
    n = 6000
    cols = [_edge_ints(rng, n, w) for w in (1, 2, 4, 8)] + [rng.integers(-10**12, 10**12, n), rng.integers(0, 4, n)]
    tab = Table.write(cg, [1, 2, 4, 8, 8, 8], cols, key="edges")
    for c, w in enumerate((1, 2, 4, 8)):
        lo, hi = LIMITS[w]
        consts = [INT64_MIN, INT64_MIN + 1, INT64_MAX - 1, INT64_MAX]
        if w < 8:
            consts += [lo - 1, lo, hi, hi + 1, 2**32 + 5 if w == 4 else 40000]
        aggs = [cg.count_star(), cg.sum_(4), cg.min_(c), cg.max_(c)]
        for i, k in enumerate(consts):
            for j, op in enumerate(OPS):
                check(cg, tab, [(c, op, k)], [] if (i + j) % 2 else [5], aggs, what=f"int{w}")


# --------------------------------------------------------------------------- the fast kernel's range reduction
@pytest.mark.parametrize("family", FAMILIES)
def test_fast_kernel_range_reduction_merges_or_refuses(cg, kernel_family, family):
    """several conjuncts on one column, empty intersections, a lone <>, <> next to a range on the same column, quals
    on two and three columns, a qual column that is also the group key or a sum argument: the answer is the
    reference's, and under "jit" the specialised kernel runs exactly when the WHERE list reduces to <= 2 ranges"""
    from citus_b200 import capi
    kernel_family(family)
    rng = np.random.default_rng(103)
    n = 8000
    x = rng.integers(-50, 50, n)
    x[:2] = [INT64_MIN, INT64_MAX]
    y = rng.integers(-1000, 1000, n)
    z = rng.integers(0, 10, n)
    k = rng.integers(0, 300, n)
    v = rng.integers(-10**9, 10**9, n)
    tab = Table.write(cg, [8] * 5, [x, y, z, k, v], key="fast")
    plain = [cg.count_star(), cg.sum_(4)]
    cases = [  # (where, group, aggs, the specialised kernel takes it)
        ([(0, ">=", -10), (0, "<", 20)], [], plain, True),
        ([(0, ">", -10), (0, "<=", 20), (0, ">=", 0), (0, "<", 5)], [], plain, True),
        ([(0, "<", 5), (0, ">", 10)], [], plain, True),
        ([(0, "=", 7), (0, "=", 8)], [], plain, True),
        ([(0, "=", 7), (0, "=", 7)], [], plain, True),
        ([(0, "=", 7), (0, "<=", 7), (0, ">=", 7)], [], plain, True),
        ([(0, "<", INT64_MIN)], [], plain, True),
        ([(0, ">", INT64_MAX)], [], plain, True),
        ([(0, "<=", INT64_MIN)], [], plain, True),
        ([(0, ">=", INT64_MAX)], [], plain, True),
        ([(0, "<>", 3)], [], plain, True),
        ([(0, "<>", INT64_MIN)], [], plain, True),
        ([(0, ">", -10), (1, "<", 0)], [], plain, True),
        ([(0, ">", -10), (1, "<", 0), (1, ">", -500)], [3], plain, True),
        ([(0, "<>", 3), (1, "<>", 0)], [3], plain, True),
        ([(0, "<>", 3), (0, ">", -10)], [], plain, False),
        ([(0, ">", -10), (0, "<>", 3)], [], plain, False),
        ([(0, "<>", 3), (0, "<>", 4)], [], plain, False),
        ([(0, ">", -10), (1, "<", 0), (2, "=", 4)], [], plain, False),
        ([(0, ">", -10), (0, "<", 10)], [0], plain, False),
        ([(0, ">", -10), (0, "<", 10)], [], [cg.count_star(), cg.sum_(0)], False),
        ([(1, "<", 0)], [3], [cg.count_star(), cg.sum_(4), cg.sum_(1)], False),
    ]
    for where, group, aggs, fast in cases:
        jit0 = capi.lib().cg_jit_launches()
        check(cg, tab, where, group, aggs, force_hash=bool(group), what="fast plan")
        if family == "jit":
            assert (capi.lib().cg_jit_launches() == jit0) == fast, (where, group)


# --------------------------------------------------------------------------- skip boundaries
def _boundary_table(cg, rng):
    """sorted int8, constant-per-chunk int4, sorted float8, a column whose chunks are all NULL, hold a single
    non-NULL value, or hold values -- every chunk of its own range, so constants land exactly on min / max"""
    n, chunk = 9000, 1000
    s = np.sort(rng.integers(-10**6, 10**6, n))
    c = np.repeat(np.arange(n // chunk) * 5 - 20, chunk)
    f = np.sort(rng.normal(size=n)) * 100
    f[-3:] = [np.inf, np.nan, np.nan]
    sparse = rng.integers(-100, 100, n)
    ns = np.zeros(n, np.uint8)
    ns[chunk:2 * chunk] = 1                        # chunk 1: all NULL
    ns[3 * chunk:4 * chunk] = 1
    ns[3 * chunk + 500] = 0                        # chunk 3: one non-NULL value
    ns[5 * chunk:6 * chunk:3] = 1                  # chunk 5: NULL-bearing
    v = rng.integers(-10**6, 10**6, n)
    cols = [s, c, f, sparse, v, rng.integers(-3, 4, n)]
    return Table.write(cg, [8, 4, 8, 8, 8, 2], cols, [None, None, None, ns, None, None], float_cols=(2,),
                       stripe_rows=3000, chunk_rows=chunk, key="boundary")


@pytest.mark.parametrize("family", FAMILIES)
def test_skip_boundaries_on_chunk_min_and_max(cg, kernel_family, family):
    """constants equal to a chunk's min or max (and one past them) on sorted, constant-per-chunk and float columns and
    on all-NULL / single-value chunks, through the shard, end-to-end and DMA staging paths"""
    kernel_family(family)
    rng = np.random.default_rng(107)
    tab = _boundary_table(cg, rng)
    paths = ["shard", "e2e", "dma"]
    i = 0
    for col in (0, 1, 2, 3):
        consts = []
        for stripe in tab.minmax[col]:
            for mm in stripe:
                if mm is not None:
                    consts += [mm[0], mm[1]]
        consts = consts[::2] + consts[-1:] if col != 3 else consts
        if col != 2:
            consts += [consts[0] - 1, consts[-1] + 1]
        aggs = [cg.count_star(), cg.sum_(4), cg.count(3), cg.min_(col, col == 2), cg.max_(col, col == 2)]
        for k in consts:
            for op in OPS:
                check(cg, tab, [(col, op, k)], [5] if i % 3 == 0 else [], aggs, path=paths[i % 3], what="boundary")
                i += 1
    # OR / AND trees whose arms each refute some chunks but not the same ones
    mm0, mm1 = tab.minmax[0][0][1], tab.minmax[0][2][0]
    trees = [("or", (0, "<", mm0[0]), (0, ">", mm1[1])),
             ("or", (0, "=", mm0[1]), (0, "=", mm1[0]), (1, "=", -20)),
             ("and", ("or", (0, "<=", mm0[1]), (3, ">", 0)), (1, "<>", -15)),
             ("or", ("and", (3, ">=", -100), (3, "<=", 99)), (2, ">", 1e300))]
    for t, where in enumerate(trees):
        check(cg, tab, where, [5], [cg.count_star(), cg.sum_(4), cg.min_(3)], path=paths[t % 3], what="boundary tree")


# --------------------------------------------------------------------------- randomized plan shapes
GROUPINGS = [[], [5], [6], [5, 6], [3]]


def _random_table(cg, rng, key):
    n = 6000
    chunk = int(rng.choice([1000, 1500]))
    rate = float(rng.choice([0.0, 0.03, 0.3]))
    cols = [rng.integers(INT64_MIN, INT64_MAX, n, endpoint=True) if rng.random() < 0.5 else rng.integers(-10**6, 10**6, n),
            rng.integers(-2**31, 2**31, n), rng.integers(-2**15, 2**15, n), rng.integers(-128, 128, n),
            rng.normal(size=n) * 1e3, rng.integers(-3, 4, n), rng.integers(0, 60, n)]
    if rng.random() < 0.5:
        cols[0] = np.sort(cols[0])
    cols[4][rng.random(n) < 0.01] = np.nan
    nulls = [(rng.random(n) < rate).astype(np.uint8) for _ in range(5)] + [None, None]
    if rate:
        nulls[int(rng.integers(0, 5))][chunk:2 * chunk] = 1          # an all-NULL chunk in one column
    return Table.write(cg, [8, 4, 2, 1, 8, 1, 4], cols, nulls, float_cols=(4,), stripe_rows=2 * chunk, chunk_rows=chunk,
                       key=key)


def _random_aggs(cg, rng):
    pool = [cg.count_star(), cg.count(0), cg.sum_(0), cg.sum_(1), cg.sum_(2), cg.min_(0), cg.max_(3), cg.min_(2),
            cg.sum_(4, True), cg.min_(4, True), cg.max_(4, True), cg.count(4)]
    idx = rng.choice(len(pool), int(rng.integers(1, 6)), replace=False)
    return [pool[i] for i in idx]


@pytest.mark.parametrize("family", FAMILIES)
def test_randomized_where_trees_and_plan_shapes(cg, kernel_family, family):
    """fixed-seed differential: random WHERE trees x group columns (none, one, two, narrow and negative) x aggregate
    kinds x column widths x NULL rates x chunk sizes; NULL-bearing chunk groups run the generated kernels' nullable
    form and its three-valued logic"""
    kernel_family(family)
    for seed in range(4):
        rng = np.random.default_rng(1000 + seed)
        tab = _random_table(cg, rng, f"random {seed}")
        pools = constant_pools(tab.minmax, [8, 4, 2, 1, 8, 1, 4], (4,))

        def atom():
            c = int(rng.integers(0, 7))
            return (c, OPS[int(rng.integers(0, 6))], pools[c][int(rng.integers(0, len(pools[c])))])
        for q in range(5):
            where = random_tree(rng, atom)
            group = GROUPINGS[int(rng.integers(0, len(GROUPINGS)))]
            aggs = _random_aggs(cg, rng)
            check(cg, tab, where, group, aggs, force_hash=bool(rng.random() < 0.3), what=f"seed {1000 + seed} query {q}")


# --------------------------------------------------------------------------- varlena columns
@pytest.mark.parametrize("family", FAMILIES)
def test_char1_high_bytes_compare_unsigned(cg, oracle, kernel_family, family):
    """char(1) bytes 0x80-0xFF under =, <>, <, > and as a group key (alone and with a second column): PostgreSQL's
    bpchar order is memcmp's, so 0xE9 sorts above 'A' and equals 233"""
    kernel_family(family)
    rng = np.random.default_rng(109)
    n = 6000
    flag = rng.integers(0, 256, n)
    flag[:6] = [0x41, 0x7F, 0x80, 0xE9, 0xFF, 0x00]
    hi = np.sort(rng.integers(0x80, 0x100, n))                       # sorted: chunks skipped on the high bytes
    cols = [flag, hi, rng.integers(-10**6, 10**6, n), rng.integers(0, 3, n)]
    tab = Table.oracle(cg, oracle, [-1, -1, 8, 4], [BPCHAR1, BPCHAR1, 0, 0], cols, stripe_rows=2000, chunk_rows=1000,
                       key="char1")
    aggs = [cg.count_star(), cg.sum_(2), cg.min_(0), cg.max_(0), cg.max_(1)]
    for col in (0, 1):
        for k in (0x41, 0x80, 0xE9, 0xFF):
            for op in ("=", "<>", "<", ">"):
                check(cg, tab, [(col, op, k)], [], aggs, path="dma" if k == 0xE9 else "shard", what="char(1)")
    for group in ([0], [1], [0, 3], [3, 1]):
        check(cg, tab, [(1, ">", 0xA0)], group, aggs, what="char(1) key")


@pytest.mark.parametrize("family", FAMILIES)
def test_numeric_quals_at_the_int64_edges(cg, oracle, kernel_family, family):
    """numeric(19, 0) and numeric(p, 2) columns holding +-(2^63 - 1) and -2^63 (as scaled integers) under quals whose
    scaled constants sit on those values"""
    kernel_family(family)
    rng = np.random.default_rng(113)
    n = 4000
    a = rng.integers(INT64_MIN, INT64_MAX, n, endpoint=True)
    a[:3] = [INT64_MAX, -INT64_MAX, INT64_MIN]
    b = rng.integers(-10**17, 10**17, n)
    b[:2] = [INT64_MAX, INT64_MIN]
    cols = [a, b, rng.integers(0, 4, n)]
    tab = Table.oracle(cg, oracle, [-1, -1, 8], [2, 2 | (2 << 8), 0], cols, stripe_rows=2000, chunk_rows=1000,
                       key="numeric")
    aggs = [cg.count_star(), cg.min_(0), cg.max_(0), cg.sum_(1), cg.sum_(0)]
    for col in (0, 1):
        for k in (INT64_MAX, INT64_MAX - 1, -INT64_MAX, INT64_MIN, 0):
            for op in OPS:
                check(cg, tab, [(col, op, k)], [2] if op in ("=", "<>") else [], aggs, what="numeric")


@pytest.mark.parametrize("family", FAMILIES)
def test_hand_assembled_numeric_datums(cg, oracle, kernel_family, family):
    """numeric datums written byte by byte from PostgreSQL's format: short and long headers, 1- and 4-byte varlena
    headers, negative weight, stripped trailing digit groups, zero, +-2^63 edges: decoded exactly; NaN, +-Infinity,
    2^63 and a value with more fractional digits than the column's scale: CG_EUNSUPPORTED"""
    from citus_b200 import capi
    kernel_family(family)
    aggs = [cg.count_star(), cg.sum_(1), cg.min_(1), cg.max_(1)]
    for datum, scale, want in HAND_DATUMS:
        pages, stripes, nodes = image_with_datums(oracle, [datum], scale)
        rel = cg.Relation.from_image(pages, stripes, nodes, [8, -1], [0, 2 | (scale << 8)])
        tab = Table(rel, [[0], [0]], None, 1000, 1000)
        for path in ("shard", "dma"):
            if want is None:
                with pytest.raises(capi.CitusGpuError) as e:
                    gpu_scan(cg, tab, [], [], aggs, path=path)
                assert e.value.code == capi.CG_EUNSUPPORTED, datum.hex()
                continue
            st, got = gpu_scan(cg, tab, [(1, "<=", want)], [], aggs, path=path)
            g = got[()]
            assert st.rows_passed == 1 and (g[1]["sum"], g[2]["minmax"], g[3]["minmax"]) == (want, want, want), datum.hex()
