"""IN / NOT IN lists and IS [NOT] NULL atoms in the fused scan against the exact reference (tests/reference.py), on
every kernel family: groups and aggregates, rows scanned, rows removed by the filter and chunk groups removed by the
filter, in WHERE, in FILTERs and in bool_and / bool_or arguments, over every column type the atoms take."""
import dataclasses

import numpy as np
import pytest

import reference as ref
from test_gpu_agg_filter import mixed_relation
from test_gpu_bool_bit_agg import assert_exact
from test_gpu_composite_key import ATTLENS, TYPES, table
from test_where_reference import constant_pools
from gpu_harness import cg, kernel_family, FAMILIES  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

OPS = ("<", "<=", "=", ">=", ">", "<>")
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


def keyed(groups, group_cols):
    out = {}
    for k, per in groups.items():
        out[() if not group_cols else (k,) if len(group_cols) == 1 else ref.unpack_two_column_key(k)] = per
    return out


def prepare(cg, rel, where, group, aggs, float_cols, expected_groups=0, force_hash=False, packing=True):
    """a partial with the skip lists' key range and term bounds, as a caller plans one"""
    aggs = [dataclasses.replace(a) for a in aggs]
    d = cg.make_desc(where, group, aggs, float_cols=float_cols, expected_groups=expected_groups)
    kmin, kmax, proven, rows = cg.relation_bounds(rel, d)
    for a, b in zip(aggs, proven):
        a.term_abs_bound = b
    d = cg.make_desc(where, group, aggs, float_cols=float_cols, expected_groups=expected_groups)
    if force_hash:
        kmin, kmax = 0, -1
    agg = cg.GpuColumnarAgg(d, rel.column_descs(), kmin, kmax, max(rows, 1))
    if not packing:
        agg.set_packing(False)
    return agg


def run(cg, rel, where, group, aggs, float_cols=(), stage="shard", **kw):
    agg = prepare(cg, rel, where, group, aggs, float_cols, **kw)
    try:
        if stage == "shard":
            shard = cg.Shard(rel)
            st = agg.scan_shard(shard)
            shard.free()
        elif stage == "pageable":
            st = agg.scan_relation(rel)
        else:
            rel.register()
            try:
                st = agg.scan_relation(rel)
            finally:
                rel.unregister()
        got = keyed(agg.groups(), group)
    finally:
        agg.free()
    return st, got


_WANT = {}


def check(cg, rel, cols, nulls, where, group, aggs, stripe_rows, chunk_rows, float_cols=(), key=None, **kw):
    """groups, aggregates and the three counters equal the reference's"""
    n = len(cols[0])
    ck = (key, repr(where), tuple(group), repr(aggs))
    if key is None or ck not in _WANT:
        want = ref.aggregate(cols, nulls, where, group, aggs, float_cols)
        mask = ref.selected_chunk_mask(cols, nulls, where, stripe_rows, chunk_rows, float_cols=float_cols)
        _WANT[ck] = (want, mask)
    want, mask = _WANT[ck]
    st, got = run(cg, rel, where, group, aggs, float_cols, **kw)
    assert st.chunk_groups_filtered == ref.chunks_filtered(mask), where
    assert st.rows_scanned == ref.rows_kept(mask, n, stripe_rows, chunk_rows), where
    assert_exact(st, got, want, aggs, n)
    return st, got


# --------------------------------------------------------------------------- random trees
def atom_maker(rng, pools, ncols):
    def list_atom(c):
        size = int(rng.choice([1, 2, 3, 8, 100, 101]))
        vals = [pools[c][int(rng.integers(0, len(pools[c])))] for _ in range(size)]
        if rng.random() < 0.25:
            vals[int(rng.integers(0, size))] = None
        return (c, "in" if rng.random() < 0.6 else "not in", tuple(vals))

    def atom():
        c = int(rng.integers(0, ncols))
        r = rng.random()
        if r < 0.35:
            return list_atom(c)
        if r < 0.55:
            return (c, "is null" if rng.random() < 0.5 else "is not null")
        return (c, OPS[int(rng.integers(0, 6))], pools[c][int(rng.integers(0, len(pools[c])))])
    return atom


def small_tree(rng, atom, max_atoms=3):
    atoms = [atom() for _ in range(int(rng.integers(1, max_atoms + 1)))]
    while len(atoms) > 1:
        i = int(rng.integers(0, len(atoms) - 1))
        atoms[i:i + 2] = [("and" if rng.random() < 0.5 else "or", atoms[i], atoms[i + 1])]
    return atoms[0]


SHAPES = [dict(group=[]), dict(group=[0]), dict(group=[0, 1]), dict(group=[2], expected_groups=4096, force_hash=True)]


@pytest.mark.parametrize("family", FAMILIES)
def test_random_trees_mixing_the_new_atoms(cg, kernel_family, family):
    """random WHERE trees, FILTERs and bool_and / bool_or arguments mixing IN / NOT IN (1 to 101 elements, NULL elements,
    duplicates) and IS [NOT] NULL with comparisons over int2 / int4 / int8 / float8 columns (NaN, +-inf, +-0.0, NULL-bearing
    and all-NULL chunk groups): plain aggregate, one- and two-column direct-indexed tables and the hash table"""
    kernel_family(family)
    rng = np.random.default_rng(20261017)
    rel, cols, nulls, stripe_rows, chunk_rows = mixed_relation(cg, rng)
    fc = (5,)
    minmax = ref.skip_minmax(cols, nulls, stripe_rows, chunk_rows, fc)
    pools = constant_pools(minmax, [2, 4, 2, 4, 8, 8], fc)
    for c in range(6):                                            # values the rows hold, so that lists find some
        pools[c] = pools[c] + [float(v) if c in fc else int(v) for v in cols[c][:40]]
    atom = atom_maker(rng, pools, 6)
    for i in range(12):
        shape = SHAPES[i % len(SHAPES)]
        where = small_tree(rng, atom)
        aggs = [cg.count_star(), cg.sum_(4, filter=small_tree(rng, atom, 2)), cg.bool_or(small_tree(rng, atom)),
                cg.bool_and(small_tree(rng, atom, 2)), cg.count(5, filter=small_tree(rng, atom, 1))]
        try:
            cg.make_desc(where, shape["group"], aggs, float_cols=fc)
        except Exception:                                         # more than 8 pool atoms / lists: drawn again next time
            continue
        check(cg, rel, cols, nulls, where, shape["group"], aggs, stripe_rows, chunk_rows, fc, key=("random", i),
              expected_groups=shape.get("expected_groups", 0), force_hash=shape.get("force_hash", False))


# --------------------------------------------------------------------------- every column type
def typed_relation(cg, oracle):
    """bool, int1, int2, int4, int8, char(1), numeric(12, 2), int8, float8 (NULLs in the second half of the rows, so both
    the NULL-free and the nullable forms run), and a column added afterwards"""
    rel, cols, nulls, n = table(cg, oracle)
    rel10 = cg.Relation.from_image(rel.pages(), rel.stripes_bytes(), rel.nodes_bytes(), ATTLENS + [8], TYPES + [0])
    cols10 = [np.asarray(c) for c in cols] + [np.zeros(n, np.int64)]
    nulls10 = [np.asarray(z).astype(np.uint8) for z in nulls] + [np.ones(n, np.uint8)]
    return rel10, cols10, nulls10, n


def typed_queries(cg, cols):
    """per column: IN of values it holds and a value it does not, NOT IN with a NULL element, the IS tests; FILTERs
    count(*) FILTER (WHERE x IS NULL) and sum(...) FILTER (WHERE k IN ...); bool_or over a list with a NULL element, whose
    rows outside the list are UNKNOWN rather than FALSE"""
    qs = []
    for c in range(10):
        if c == 8:
            held = [float(v) for v in np.asarray(cols[c])[:3]]
            out = [1e300]
        else:
            held = ([int(v) for v in np.unique(np.asarray(cols[c])[:200])] + [77, 78])[:3]
            out = [10**15 + 7]
        aggs = [cg.count_star(), cg.count_star(filter=(c, "is null")), cg.sum_(7, filter=(3, "in", (-8, 0, 5, 7))),
                cg.bool_or((c, "in", tuple(held[:1]) + (None,))), cg.bool_and((c, "not in", tuple(held[1:2])))]
        qs.append(([(c, "in", tuple(held + out))], [], aggs))
        qs.append(([(c, "not in", tuple(held[:2]) + (None,))], [3], aggs[:3]))
        qs.append(([(c, "is null")], [], aggs))
        qs.append(([(c, "is not null")], [0], aggs[:2]))
    return qs


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("stage", ["shard", "pageable", "dma"])
def test_every_column_type_and_staging_path(cg, oracle, kernel_family, family, stage):
    kernel_family(family)
    rel, cols, nulls, n = typed_relation(cg, oracle)
    for i, (where, group, aggs) in enumerate(typed_queries(cg, cols)):
        for packing in ((True, False) if group else (True,)):
            check(cg, rel, cols, nulls, where, group, aggs, 4000, 1000, (8,), key=("typed", i), stage=stage, packing=packing)


# --------------------------------------------------------------------------- citus issue 5803, in integers
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("stage", ["shard", "pageable", "dma"])
def test_in_list_over_four_chunk_groups_restates_citus_5803(cg, kernel_family, family, stage):
    """four chunk groups holding two values each and WHERE c IN (three values) falling in two of them: the scan removes two
    chunk groups, scans the 2000 rows of the other two (the writer's smallest chunk group is 1000 rows), removes the one
    row holding the fourth value and passes 1999"""
    kernel_family(family)
    c = np.concatenate([[10] + [11] * 999, [20] * 500 + [21] * 500, [30] * 500 + [31] * 500, [40] * 500 + [41] * 500]).astype(np.int64)
    rel = cg.Relation.write([8], [c], None, stripe_row_limit=4000, chunk_row_limit=1000)
    st, _ = check(cg, rel, [c], None, [(0, "in", (11, 20, 21))], [], [cg.count_star(), cg.sum_(0)], 4000, 1000, stage=stage)
    assert (st.chunk_groups_filtered, st.rows_scanned, st.rows_removed_by_filter, st.rows_passed) == (2, 2000, 1, 1999)


# --------------------------------------------------------------------------- list sizes and int64 extremes
@pytest.mark.parametrize("family", FAMILIES)
def test_list_sizes_at_int64_extremes(cg, kernel_family, family):
    """lists of 1, 2, 8, 100, 101 and 1024 elements holding INT64_MIN, INT64_MAX and their neighbours, over an int8 column
    that holds them too; sorted data, so that lists refute chunk groups"""
    kernel_family(family)
    rng = np.random.default_rng(5)
    n = 16_000
    v = np.sort(rng.integers(-10**6, 10**6, n))
    v[:3] = [INT64_MIN, INT64_MIN + 1, INT64_MIN + 2]
    v[-3:] = [INT64_MAX - 2, INT64_MAX - 1, INT64_MAX]
    g = rng.integers(0, 7, n)
    z = (rng.random(n) < 0.02).astype(np.uint8)
    z[:2] = 0
    cols, nulls = [g, v], [None, z]
    rel = cg.Relation.write([8, 8], cols, nulls, stripe_row_limit=4000, chunk_row_limit=1000)
    pool = [int(x) for x in v[::17]]
    for size in (1, 2, 8, 100, 101, 1024):
        vals = [INT64_MIN, INT64_MAX, INT64_MAX - 1, INT64_MIN + 1] + [pool[int(rng.integers(0, len(pool)))] for _ in range(size)]
        vals = vals[:size]
        for where in ([(1, "in", tuple(vals))], [(1, "not in", tuple(vals))], [(1, "in", tuple(vals[:-1]) + (None,))] if size > 1 else []):
            if not where:
                continue
            arg = (1, "not in", tuple(vals[:4]) + (None,)) if size < 1000 else (1, "is not null")     # 1024 values fill the table
            aggs = [cg.count_star(), cg.sum_(0), cg.min_(1), cg.max_(1), cg.bool_or(arg)]
            check(cg, rel, cols, nulls, where, [0], aggs, 4000, 1000, (), key=("sizes", size, repr(where)[:40]))


# --------------------------------------------------------------------------- IN as an OR tree
@pytest.mark.parametrize("family", FAMILIES)
def test_eight_value_in_equals_the_or_tree(cg, kernel_family, family):
    """x IN (8 values) gives exactly the groups, aggregates and counters of the OR of eight "=" atoms (a list of at
    most 100 elements refutes chunk groups as the OR does)"""
    kernel_family(family)
    rng = np.random.default_rng(8)
    n = 20_000
    q = np.sort(rng.integers(100, 5100, n))
    cols = [rng.integers(0, 4, n), q, rng.integers(0, 10**6, n)]
    rel = cg.Relation.write([8, 8, 8], cols, None, stripe_row_limit=4000, chunk_row_limit=1000)
    vals = (150, 900, 901, 2400, 2401, 3000, 4999, 5000)
    aggs = [cg.count_star(), cg.sum_(2), cg.max_(2)]
    for group in ([], [0]):
        st1, got1 = run(cg, rel, [(1, "in", vals)], group, aggs)
        st2, got2 = run(cg, rel, ("or",) + tuple((1, "=", v) for v in vals), group, aggs)
        assert got1 == got2
        assert (st1.rows_scanned, st1.rows_removed_by_filter, st1.chunk_groups_filtered) == \
            (st2.rows_scanned, st2.rows_removed_by_filter, st2.chunk_groups_filtered)
        assert st1.chunk_groups_filtered > 0
        check(cg, rel, cols, None, [(1, "in", vals)], group, aggs, 4000, 1000)


# --------------------------------------------------------------------------- asynchronous scans, kernel reuse
def test_back_to_back_asynchronous_scans_with_different_lists(cg, kernel_family):
    """scans without statistics are asynchronous: several of them with different lists into one partial, enqueued back
    to back, must equal the sum of separate scans (a later scan never overwrites the codes an earlier one still reads);
    the same holds for cg_scan_relation over several shards.  The generated kernel is compiled once for the shape."""
    from citus_b200 import capi
    kernel_family("jit_always")
    rng = np.random.default_rng(3)
    n = 40_000
    cols = [rng.integers(0, 16, n), rng.integers(0, 1000, n), rng.integers(-10**6, 10**6, n)]
    rels = [cg.Relation.write([8, 8, 8], [c[i * 10_000:(i + 1) * 10_000] for c in cols], None, stripe_row_limit=10_000,
                              chunk_row_limit=1000) for i in range(4)]
    lists = [tuple(int(x) for x in rng.integers(0, 1000, k)) for k in (1, 37, 300, 1000)]
    aggs = [cg.count_star(), cg.sum_(2)]
    wheres = [[(1, "in", l)] for l in lists]

    def partial_for(where):
        aggs2 = [dataclasses.replace(a, term_abs_bound=10**6) for a in aggs]
        d = cg.make_desc(where, [0], aggs2)
        return cg.GpuColumnarAgg(d, rels[0].column_descs(), 0, 15, n)

    # separate scans, one partial each
    want = {}
    for where in wheres:
        p = partial_for(where)
        for rel in rels:
            sh = cg.Shard(rel)
            p.scan_shard(sh)
            sh.free()
        for k, per in p.groups().items():
            w = want.setdefault(k, [0, 0])
            w[0] += per[0]["count"]
            w[1] += per[1]["sum"]
        p.free()
    shards = [cg.Shard(rel) for rel in rels]
    before = capi.lib().cg_jit_compiles()
    p = partial_for(wheres[0])
    descs = [cg.make_desc(where, [0], [dataclasses.replace(a, term_abs_bound=10**6) for a in aggs]) for where in wheres]
    for sh in shards:                                            # the same partial, a new list every scan (16 changes, so the
        for d in descs:                                          # pinned staging ring wraps), no statistics: asynchronous
            p.desc = d
            p.scan_shard(sh, want_stats=False)
    got = {k: [per[0]["count"], per[1]["sum"]] for k, per in p.groups().items()}
    assert got == want
    assert capi.lib().cg_jit_compiles() - before <= 1
    p.reset()
    for where in wheres:                                         # cg_scan_relation across the shards
        p.desc = cg.make_desc(where, [0], [dataclasses.replace(a, term_abs_bound=10**6) for a in aggs])
        for rel in rels:
            p.scan_relation(rel, want_stats=False)
    got = {k: [per[0]["count"], per[1]["sum"]] for k, per in p.groups().items()}
    assert got == want
    p.free()
    for sh in shards:
        sh.free()
    # each list alone against the reference
    for where in wheres:
        want1 = ref.aggregate(cols, None, where, [0], aggs)
        p = partial_for(where)
        for rel in rels:
            p.scan_relation(rel)
        got1 = {(k,): per for k, per in p.groups().items()}
        assert {k: (v[0]["count"], v[1]["sum"]) for k, v in got1.items()} == \
            {k: (v[0].count, v[1].sum) for k, v in want1.groups.items()}
        p.free()
