"""The group table the fused scan writes into, against tests/group_table_reference.py, on every kernel family.

  A. packed words (count(*) and one bounded sum in one 64-bit word) at every shift C = 12..24, terms at +-bound, the
     packed image word for word, and a group of exactly 2^C - 1 rows (exact) or 2^C rows (CG_ERETRY_UNPACKED) in one launch;
  B. drains across launches on both sides of the capacity * 2^C / 32 limit, through scan_shard and scan_relation;
  C. life-cycle programs of scans, reads, resets, packing changes, merges and dense-word exports;
  D. hash addressing: keys that share one home slot, clusters that wrap, runs just under the probe limit, over-full
     tables, the NULL key next to the key equal to the empty-slot value, and the lane-paired update;
  E. direct-indexed addressing at the 2^26 range limit and at the int64 / int32 ends, and the dense words' layout;
  F. the per-lane narrow cells of the shared-memory kernels at the term bound, at every chunk-group size that changes
     how many chunk groups a CTA may take, and a scan long enough that the generated kernel must cut its launches.
Which kernel ran is asserted through cg_jit_launches and the partial's packed state (GpuColumnarAgg.packed_state)."""

import numpy as np
import pytest

import group_table_reference as gt
from gpu_harness import kernel_family, FAMILIES  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

DENSE, HASH = "dense", "hash"
I64_MIN, I64_MAX = gt.I64_MIN, gt.I64_MAX
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
TB = 13421772                    # the largest term bound whose sums may live in 32-bit halves (tbound * 160 < 2^31)


@pytest.fixture(scope="module")
def cg():
    import torch
    assert torch.cuda.is_available(), "these tests need an H100"
    from citus_b200 import build
    build.build()
    from citus_b200 import columnar
    columnar.init(0)
    yield columnar
    # the module's relations and staged shards go while the library is still loaded, not at interpreter exit
    for r in _RELS:
        if r._shard is not None:
            r._shard.free()
    for _, shard, _ in _CAP.values():
        shard.free()
    for cache in (_RELS, _SHIFT_RELS, _BOUNDARY_RELS, _EXPECT, _LIFE, _CAP, _LIMIT_RELS):
        cache.clear()


def capi():
    from citus_b200 import capi as c
    return c


def jit_launches():
    return capi().lib().cg_jit_launches()


def packs(family, nullable):
    """whether a scan of NULL-free (or NULL-bearing) chunk groups into a packing partial writes packed words: the fast
    kernel and the generated table kernel do, in both its forms; the interpretive kernels never do"""
    return family in ("jit", "jit_always") or (family == "aot" and not nullable)


# --------------------------------------------------------------------------- data, partials, answers
_RELS = []


class Rel:
    """a relation of int columns (key columns first, then the sum arguments), its arrays and NULL flags"""

    def __init__(self, cg, cols, nulls=None, attlens=None, stripe=150_000, chunk=10_000):
        self.cols = [np.ascontiguousarray(c, np.int64) for c in cols]
        self.nulls = nulls or [None] * len(cols)
        self.rel = cg.Relation.write(attlens or [8] * len(cols), self.cols, nulls=[None if x is None else x.astype(np.uint8)
                                                                                      for x in self.nulls],
                                     stripe_row_limit=stripe, chunk_row_limit=chunk)
        self._shard = None
        _RELS.append(self)

    def shard(self, cg):
        if self._shard is None:
            self._shard = cg.Shard(self.rel)
        return self._shard

    @property
    def n(self):
        return len(self.cols[0])


def exact_sums(inv, ng, v):
    """per group sums of int64 values v, exact: 16-bit pieces summed in float64 (exact below 2^53 per piece sum)"""
    out = [0] * ng
    for sh in (0, 16, 32, 48):
        piece = (v >> sh) if sh == 48 else ((v >> sh) & 0xFFFF)
        s = np.bincount(inv, weights=piece.astype(np.float64), minlength=ng)
        for g in range(ng):
            out[g] += int(s[g]) << sh
    return out


_EXPECT = {}


def expect(rels, ngroup=1):
    k = (tuple(id(r) for r in rels), ngroup)
    if k not in _EXPECT:
        _EXPECT[k] = (rels, _expect(rels, ngroup))           # the relations are kept alive with their answer
    return _EXPECT[k][1]


def _expect(rels, ngroup):
    """{key or None: (rows, (count, sum) per sum argument)} of count(*), sum(col) ... GROUP BY the key column(s); two key
    columns give the packed key (low 32 bits: the first)"""
    cols = [np.concatenate([r.cols[c] for r in rels]) for c in range(len(rels[0].cols))]
    nulls = [None if all(r.nulls[c] is None for r in rels) else
             np.concatenate([np.zeros(r.n, bool) if r.nulls[c] is None else r.nulls[c].astype(bool) for r in rels])
             for c in range(len(cols))]
    if ngroup == 2:
        key = (cols[0] & 0xFFFFFFFF) | (cols[1] << 32)
    else:
        key = cols[0]
    knull = nulls[0] if nulls[0] is not None else np.zeros(len(key), bool)
    out = {}
    for isnull in (False, True):
        m = knull == isnull
        if not m.any():
            continue
        uk, inv = np.unique(np.where(isnull, 0, key[m]), return_inverse=True)
        rows = np.bincount(inv, minlength=len(uk))
        per = []
        for c in range(ngroup, len(cols)):
            ok = np.ones(m.sum(), bool) if nulls[c] is None else ~nulls[c][m]
            cnt = np.bincount(inv[ok], minlength=len(uk))
            per.append((cnt, exact_sums(inv[ok], len(uk), cols[c][m][ok])))
        for g, k in enumerate(uk):
            out[None if isnull else int(k)] = (int(rows[g]),) + tuple((int(cnt[g]), s[g]) for cnt, s in per)
    return out


def add(a, b):
    out = dict(a)
    for k, v in b.items():
        if k in out:
            w = out[k]
            out[k] = (w[0] + v[0],) + tuple((x[0] + y[0], x[1] + y[1]) for x, y in zip(w[1:], v[1:]))
        else:
            out[k] = v
    return out


def answer(agg):
    return {k: (per[0]["count"],) + tuple((p["count"], p["sum"] if p["count"] else 0) for p in per[1:])
            for k, per in agg.groups().items()}


def partial(cg, rels, mode, nsums=None, expected_groups=1, packing=True, ngroup=1, max_rows=None):
    """count(*), sum(col) for every non-key column, GROUP BY the key column(s), with the bounds the relations prove"""
    nsums = len(rels[0].cols) - ngroup if nsums is None else nsums
    group = list(range(ngroup))
    aggs = [cg.count_star()] + [cg.sum_(ngroup + i) for i in range(nsums)]
    d = cg.make_desc([], group, aggs)
    kmin = kmax = None
    bounds, rows = [0] * len(aggs), 0
    for r in rels:
        a, b, bs, n = cg.relation_bounds(r.rel, d)
        if a <= b:
            kmin = a if kmin is None else min(kmin, a)
            kmax = b if kmax is None else max(kmax, b)
        bounds = [max(x, y) for x, y in zip(bounds, bs)]
        rows += n
    for a, b in zip(aggs, bounds):
        a.term_abs_bound = b
    d = cg.make_desc([], group, aggs, expected_groups=expected_groups if mode == HASH else 0)
    lo, hi = (kmin, kmax) if mode == DENSE else (0, -1)
    agg = cg.GpuColumnarAgg(d, rels[0].rel.column_descs(), lo, hi, max_rows or max(rows, 1))
    if not packing:
        agg.set_packing(False)
    nw, _, dense, cap = agg.layout()
    assert nw == 1 + 2 * nsums, (nw, nsums)            # one-word sums: [rows, sum 1, NULL inputs 1, sum 2, ...]
    agg.kmin, agg.capacity = (kmin if dense else None), cap
    return agg


def device_words(ptr, n):
    import torch

    class View:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "strides": None, "version": 3}
    return torch.as_tensor(View(), device="cuda").cpu().numpy().view(np.uint64)


def check_packed_image(agg, groups, c):
    """the packed words after one pass over NULL-free rows, no drain: (sum << C) + n at each group's entry (a hash key's
    slot depends on the order keys arrive in: those words as a multiset, the NULL and empty-value entries in place)"""
    shift, _, state, words = agg.packed_state()
    dense = agg.kmin is not None
    assert shift == c and words.size == agg.capacity + (1 if dense else 2)
    special = {None: agg.capacity} if dense else {None: agg.capacity, gt.HASH_EMPTY: agg.capacity + 1}
    at, rest = {}, []
    for k, (n, (_, s)) in groups.items():
        w = gt.pack(s, n, c)
        if k in special:
            at[special[k]] = w
        elif dense:
            at[k - agg.kmin] = w
        else:
            rest.append(w)
    got = {int(e): int(words[e]) for e in np.flatnonzero(words)}
    for e, w in at.items():
        assert got.pop(e, 0) == w, e
    assert sorted(got.values()) == sorted(rest)
    return state


# --------------------------------------------------------------------------- A. packed words at every shift
SHIFTS = list(range(12, 25))


def shift_rel(cg, c, mode, hot_rows, sign, seed, nullable=False):
    """key, x: a hot key with hot_rows rows of term sign * bound(C), 300 more rows over the key domain (dense: 6000
    keys, more than the shared-memory kernels take; hash: keys anywhere in int64) with terms in [-bound, bound].  The
    NULL-bearing relation's hot key is another one, and no other row falls on either, so that a hot group holds exactly
    hot_rows rows of one relation"""
    rng = np.random.default_rng(seed)
    b = gt.bound_for_shift(c)
    n = hot_rows + 300
    lo = -3000
    hot = lo + (18 if nullable else 17) if mode == DENSE else int(rng.integers(-(1 << 62), 1 << 62))
    others = rng.integers(lo + 19, lo + 6000, 300) if mode == DENSE else rng.integers(-(1 << 62), 1 << 62, 300)
    key = np.concatenate([np.full(hot_rows, hot), others])
    x = np.concatenate([np.full(hot_rows, sign * b), rng.integers(-b, b + 1, 300)])
    x[-1], x[-2] = -b, b
    key[-1], key[-2] = lo, lo + 5999
    p = rng.permutation(n)
    key, x = key[p], x[p]
    nulls = None
    if nullable:                     # NULL keys and NULL sum inputs, in every chunk group
        kn, xn = rng.random(n) < 0.05, rng.random(n) < 0.05
        kn[:1], xn[1:2] = True, True
        nulls = [kn, xn]
    return Rel(cg, [key, x], nulls, chunk=1000 if hot_rows < 20_000 else 10_000)


_SHIFT_RELS = {}


def shift_rels(cg, c, mode):
    k = (c, mode)
    if k not in _SHIFT_RELS:
        hot = (1 << c) - 1 if c <= 14 else 5000
        sign = 1 if c % 2 else -1
        _SHIFT_RELS[k] = (shift_rel(cg, c, mode, hot, sign, c), shift_rel(cg, c, mode, 500, -sign, 100 + c, nullable=True))
    return _SHIFT_RELS[k]


@pytest.mark.parametrize("family", FAMILIES)
def test_packed_words_at_every_shift(cg, kernel_family, family):
    """count(*) and sum(x) at every shift: the packed image after a NULL-free shard equals (sum << C) + n per entry, and
    the answer after a NULL-bearing shard on top (NULL keys, NULL inputs: the nullable generated kernel, or the
    interpretive one) is exact.  From C = 16 up the terms fit 32 bits, so a direct-indexed table's key and argument both
    have narrow images, and the fast kernel reads those (bytes_scanned: the bit-packed streams, not 8 bytes a value)"""
    P = capi()
    kernel_family(family)
    for mode in (DENSE, HASH):
        for c in SHIFTS:
            plain, nully = shift_rels(cg, c, mode)
            agg = partial(cg, [plain, nully], mode)
            try:
                assert agg.packed_state()[0] == c == gt.pack_shift(gt.bound_for_shift(c))
                st = agg.scan_shard(plain.shard(cg))
                narrow = family in ("jit", "aot") and mode == DENSE and c >= 16
                assert (st.bytes_scanned < 12 * plain.n) == narrow and (narrow or st.bytes_scanned >= 16 * plain.n), \
                    (mode, c, st.bytes_scanned)
                want = expect([plain])
                if packs(family, False):
                    state = check_packed_image(agg, want, c)
                    assert state & P.CG_PSTATE_PACKED_DIRTY and not state & P.CG_PSTATE_WIDE_DIRTY
                else:
                    assert not agg.packed_state()[3].any()
                agg.scan_shard(nully.shard(cg))
                assert answer(agg) == add(want, expect([nully])), (mode, c)
            finally:
                agg.free()


@pytest.mark.parametrize("family", FAMILIES)
def test_packed_path_with_more_sums(cg, kernel_family, family):
    """count(*), sum(x) packed plus one or two wide sums (the fast kernel's PACK instances with NS = 2, 3; the
    generated table kernel's packed form), terms at +-bound, dense and hash"""
    kernel_family(family)
    rng = np.random.default_rng(9)
    n = 30_000
    for mode in (DENSE, HASH):
        key = rng.integers(0, 7000, n) if mode == DENSE else rng.integers(-(1 << 62), 1 << 62, 2000)[rng.integers(0, 2000, n)]
        b = gt.bound_for_shift(13)
        cols = [key, np.where(rng.random(n) < 0.5, b, -b), rng.integers(-(1 << 40), 1 << 40, n), np.full(n, -(1 << 20))]
        r = Rel(cg, cols, chunk=4096)
        for nsums in (2, 3):
            agg = partial(cg, [r], mode, nsums=nsums, expected_groups=2000)
            try:
                agg.scan_shard(r.shard(cg))
                state = agg.packed_state()[2]
                assert bool(state & capi().CG_PSTATE_PACKED_DIRTY) == packs(family, False)
                assert answer(agg) == {k: v[:1 + nsums] for k, v in expect([r]).items()}
            finally:
                agg.free()


BOUNDARY = [(12, DENSE), (12, HASH), (13, DENSE), (13, HASH), (20, DENSE), (24, DENSE)]
_BOUNDARY_RELS = {}


def boundary_rels(cg, c, mode, sign):
    k = (c, mode, sign)
    if k not in _BOUNDARY_RELS:
        _BOUNDARY_RELS[k] = (shift_rel(cg, c, mode, (1 << c) - 1, sign, 7 * c), shift_rel(cg, c, mode, 1 << c, sign, 7 * c))
    return _BOUNDARY_RELS[k]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("c,mode", BOUNDARY)
def test_one_launch_of_two_to_the_c_rows(cg, kernel_family, family, c, mode):
    """one group receiving 2^C - 1 rows in one launch is exact; 2^C rows wrap its row count, which the read reports as
    CG_ERETRY_UNPACKED (where the kernel packs); with packing off, reset and rescanned, the answer is exact"""
    P = capi()
    kernel_family(family)
    for sign in ((1, -1) if c < 20 else (-1,)):
        under, over = boundary_rels(cg, c, mode, sign)
        for r, rows in ((under, (1 << c) - 1), (over, 1 << c)):
            agg = partial(cg, [r], mode)
            try:
                agg.scan_shard(r.shard(cg))
                want = expect([r])
                assert max(v[0] for v in want.values()) == rows
                t = gt.PackedTable(agg.capacity, c)
                t.launch(r.n, {k: (v[0], v[1][1]) for k, v in want.items()})
                if packs(family, False) and t.read() is None:
                    with pytest.raises(P.CitusGpuError) as e:
                        agg.groups()
                    assert e.value.code == P.CG_ERETRY_UNPACKED
                    agg.reset()
                    agg.set_packing(False)
                    agg.scan_shard(r.shard(cg))
                    assert not agg.packed_state()[2] & P.CG_PSTATE_PACKED_DIRTY
                assert answer(agg) == want
            finally:
                agg.free()


# --------------------------------------------------------------------------- B. drains across launches
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("path", ["shard", "relation"])
def test_drains_across_launches(cg, kernel_family, family, path):
    """a hash table of 1024 slots at C = 12 drains once the rows since the last drain pass 1024 * 4096 / 32 = 131072.  A
    hot group takes 3000 rows per scan: three scans of 140 000 rows are exact (a drain after each), two scans of 120 000
    rows are not (no drain in between: 6000 >= 4096 rows in one packed word)"""
    P = capi()
    kernel_family(family)
    rng = np.random.default_rng(31)
    b = gt.bound_for_shift(12)
    keys = rng.integers(-(1 << 62), 1 << 62, 200)
    for n, scans in ((140_000, 3), (120_000, 2)):
        key = keys[rng.integers(1, 200, n)]
        key[np.linspace(0, n - 1, 3000).astype(np.int64)] = keys[0]      # the hot group, spread over the whole scan
        x = np.where(rng.random(n) < 0.5, -b, b)
        r = Rel(cg, [key, x], chunk=10_000)
        agg = partial(cg, [r], HASH, expected_groups=1, max_rows=scans * n)
        assert agg.capacity == 1024 and agg.packed_state()[0] == 12
        want, t = expect([r]), gt.PackedTable(1024, 12)
        if path == "relation":
            r.rel.register()
        try:
            for _ in range(scans):
                if path == "shard":
                    agg.scan_shard(r.shard(cg))
                else:
                    agg.scan_relation(r.rel)
                t.launch(n, {k: (v[0], v[1][1]) for k, v in want.items()})
            total = {k: (v[0] * scans, (v[1][0] * scans, v[1][1] * scans)) for k, v in want.items()}
            predicted = t.read()
            assert (predicted is None) == (n == 120_000)
            # staging may cut a relation into several launches, and a drain can then fall between two of them: there the
            # overflow the schedule predicts is allowed, not required
            required = predicted is None and packs(family, False) and path == "shard"
            if required:
                with pytest.raises(P.CitusGpuError) as e:
                    agg.groups()
                assert e.value.code == P.CG_ERETRY_UNPACKED
            else:
                try:
                    got = answer(agg)
                except P.CitusGpuError as e:
                    assert predicted is None and packs(family, False) and e.code == P.CG_ERETRY_UNPACKED
                else:
                    assert got == total
        finally:
            if path == "relation":
                r.rel.unregister()
            agg.free()


# --------------------------------------------------------------------------- C. life-cycle programs
def life_rels(cg):
    """three small shards over one dense key domain of 5000 keys (more than the shared-memory kernels take): two
    NULL-free, one with NULL keys and NULL sum inputs"""
    out = []
    for i in range(3):
        rng = np.random.default_rng(50 + i)
        n = 9000 + 1111 * i
        key = rng.integers(-2500, 2500, n)
        key[:2] = -2500, 2499
        b = gt.bound_for_shift(14)
        cols = [key, np.where(rng.random(n) < 0.5, b, -b), rng.integers(-10**9, 10**9, n)]
        nulls = None
        if i == 2:
            nulls = [rng.random(n) < 0.03, rng.random(n) < 0.03, None]
        out.append(Rel(cg, cols, nulls, chunk=3000))
    return out


def export(agg, cap):
    import torch
    nw = agg.layout()[0]
    keys = torch.empty(cap, dtype=torch.int64, device="cuda")
    kn = torch.empty(cap, dtype=torch.uint8, device="cuda")
    words = torch.empty(cap * nw, dtype=torch.int64, device="cuda")
    n = agg.export_device(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), cap)
    return keys, kn, words, n


def merge_rows_from(cg, agg, r, nsums):
    """a hash partial of the same aggregates over shard r, exported on the device and merged row-wise into agg"""
    other = partial(cg, [r], HASH, nsums=nsums, expected_groups=6000, max_rows=agg.max_rows)
    try:
        other.scan_shard(r.shard(cg))
        keys, kn, words, n = export(other, 6000)
        agg.merge_rows(keys.data_ptr(), kn.data_ptr(), words.data_ptr(), n)
    finally:
        other.free()
    return {k: v[:1 + nsums] for k, v in expect([r]).items()}


def merge_values_into(agg, rng, nsums):
    n = 40
    keys = rng.integers(-2500, 2500, n)
    keys = np.unique(keys)
    n = len(keys)
    na = 1 + nsums
    count = np.zeros((n, na), np.int64)
    hi, lo = np.zeros((n, na), np.int64), np.zeros((n, na), np.uint64)
    rows = rng.integers(1, 50, n)
    count[:, 0] = rows
    want = {}
    for i in range(n):
        per = [int(rows[i])]
        for a in range(1, na):
            c = int(rng.integers(0, rows[i] + 1))
            s = int(rng.integers(-(1 << 50), 1 << 50)) if c else 0
            count[i, a], hi[i, a], lo[i, a] = c, s >> 64, s & gt.MASK64
            per.append((c, s))
        want[int(keys[i])] = tuple(per)
    agg.merge_values(keys, None, hi, lo, count, np.zeros((n, na), np.int64), np.zeros((n, na)))
    return want


def check_dense_words(agg, want, enqueue):
    if enqueue:
        p, total, stride = agg.dense_words_enqueue()
        agg.check()
    else:
        p, total, stride = agg.dense_words()
    nw = agg.layout()[0]
    shape = gt.Shape(DENSE, agg.capacity, agg.capacity + 1, gt.pow2_at_least(nw))
    assert (total, stride) == (shape.entries * shape.stride, shape.stride)
    words = {k: [v[0]] + [x for cnt, s in v[1:] for x in (s, v[0] - cnt)] for k, v in want.items()}
    ref_words = np.array(gt.dense_words(words, shape, agg.kmin, nw), np.uint64)
    got = device_words(p, total)
    assert np.array_equal(got, ref_words), np.flatnonzero(got != ref_words)[:5]
    assert not agg.packed_state()[3].any()          # drained


def run_program(cg, P, family, rels, steps, nsums, rng, log):
    """steps: list of ops; the reference is the sum of everything scanned or merged since the last reset, and the
    partial's flags follow gt.PartialFlags, step by step"""
    agg = partial(cg, rels, DENSE, nsums=nsums, max_rows=1 << 20)
    agg.max_rows = 1 << 20
    want, flags = {}, gt.PartialFlags()
    sub = lambda g: {k: v[:1 + nsums] for k, v in g.items()}
    try:
        for op in steps:
            log.append(op)
            kind = op[0]
            if kind == "scan":
                r = rels[op[1]]
                agg.scan_shard(r.shard(cg))
                want = add(want, sub(expect([r])))
                nullable = r.nulls[0] is not None
                # NULL-free chunk groups: count(*) and one sum write the packed word only; NULL inputs need their counter
                flags.scan(packs(family, nullable), nsums == 1 and not nullable)
            elif kind == "read":
                flags.read(direct_form=True)
                how = op[1]
                if how == "groups":
                    assert answer(agg) == want, log
                elif how == "ngroups":
                    assert agg.ngroups() == len(want), log
                else:
                    keys, kn, words, n = export(agg, 6000)
                    assert n == len(want), log
                    nw = agg.layout()[0]
                    k, z, w = keys[:n].cpu().numpy(), kn[:n].cpu().numpy(), words[:n * nw].cpu().numpy().reshape(n, nw)
                    got = {None if z[i] else int(k[i]): (int(w[i, 0]),) + tuple(
                        (int(w[i, 0]) - int(w[i, 2 + 2 * a]), int(w[i, 1 + 2 * a])) for a in range(nsums)) for i in range(n)}
                    exp = {kk: (v[0],) + tuple((c, s) for c, s in v[1:]) for kk, v in want.items()}
                    assert got == exp, log
            elif kind == "reset":
                agg.reset()
                want = {}
                flags.reset()
                assert not agg.packed_state()[3].any(), log
            elif kind == "packing":
                if flags.set_packing(op[1]):
                    agg.set_packing(op[1])
                else:
                    with pytest.raises(P.CitusGpuError) as e:
                        agg.set_packing(op[1])
                    assert e.value.code == P.CG_EINVAL, log
            elif kind == "merge_rows":
                want = add(want, merge_rows_from(cg, agg, rels[op[1]], nsums))
                flags.merge()
            elif kind == "merge_values":
                want = add(want, merge_values_into(agg, rng, nsums))
                flags.merge()
            elif kind == "dense_words":
                check_dense_words(agg, want, op[1])
                flags.drain()
            state = agg.packed_state()[2]
            assert state == (P.CG_PSTATE_TABLE_INITIALISED | (P.CG_PSTATE_PACKED_DIRTY if flags.packed else 0) |
                             (P.CG_PSTATE_WIDE_DIRTY if flags.wide else 0) |
                             (P.CG_PSTATE_READ_PACKED_DIRECT if flags.direct else 0)), (log, state, flags)
    finally:
        agg.free()


FIXED_PROGRAMS = [
    # packed-only scan, direct read, scan (drains first), reset, packed-only scan, read
    [("scan", 0), ("read", "groups"), ("read", "groups"), ("scan", 1), ("read", "ngroups"), ("reset",), ("scan", 0),
     ("read", "groups")],
    # a packed launch with NULL inputs (wide words written too), then reset: the wide table must start over
    [("scan", 2), ("reset",), ("scan", 2), ("read", "groups"), ("reset",), ("scan", 0), ("read", "groups"), ("scan", 2),
     ("read", "export")],
    # wide words from an unpacked scan, reset, packing back on
    [("reset",), ("packing", False), ("scan", 0), ("read", "groups"), ("reset",), ("packing", True), ("scan", 1),
     ("read", "groups"), ("reset",), ("scan", 0), ("read", "export")],
    # merges and dense words between scans and resets
    [("scan", 0), ("merge_rows", 1), ("read", "groups"), ("reset",), ("scan", 1), ("dense_words", False), ("scan", 0),
     ("merge_values",), ("dense_words", True), ("read", "groups"), ("reset",), ("scan", 0), ("packing", False),
     ("read", "groups")],
]


def random_program(rng, length):
    steps, dirty = [], False
    for _ in range(length):
        x = rng.random()
        if x < 0.3:
            steps.append(("scan", int(rng.integers(0, 3))))
        elif x < 0.55:
            steps.append(("read", ["groups", "ngroups", "export"][int(rng.integers(0, 3))]))
        elif x < 0.65:
            steps.append(("reset",))
        elif x < 0.75:
            steps.append(("packing", bool(rng.integers(0, 2))))
        elif x < 0.82:
            steps.append(("merge_rows", int(rng.integers(0, 3))))
        elif x < 0.88:
            steps.append(("merge_values",))
        else:
            steps.append(("dense_words", bool(rng.integers(0, 2))))
    return steps + [("read", "groups")]


_LIFE = {}


@pytest.mark.parametrize("family", FAMILIES)
def test_life_cycle_programs(cg, kernel_family, family):
    P = capi()
    kernel_family(family)
    if "rels" not in _LIFE:
        _LIFE["rels"] = life_rels(cg)
    rels = _LIFE["rels"]
    rng = np.random.default_rng(77)
    for nsums in (1, 2):
        for prog in FIXED_PROGRAMS:
            run_program(cg, P, family, rels, prog, nsums, rng, [("fixed", nsums)])
        for seed in range(6):
            prog = random_program(np.random.default_rng(1000 * nsums + seed), 14)
            run_program(cg, P, family, rels, prog, nsums, rng, [("seed", nsums, seed)])


@pytest.mark.parametrize("family", FAMILIES)
def test_read_state_bits(cg, kernel_family, family):
    """the packed-only plan on NULL-free chunk groups is read straight from its packed words (and marks the partial so),
    the next scan drains first; a plan with a second sum writes wide words as well and is read after a drain"""
    P = capi()
    kernel_family(family)
    if "rels" not in _LIFE:
        _LIFE["rels"] = life_rels(cg)
    rels = _LIFE["rels"]
    for nsums in (1, 2):
        agg = partial(cg, rels, DENSE, nsums=nsums, max_rows=1 << 20)
        try:
            assert agg.packed_state()[2] == P.CG_PSTATE_TABLE_INITIALISED
            agg.scan_shard(rels[0].shard(cg))
            state = agg.packed_state()[2]
            packed = packs(family, False)
            assert bool(state & P.CG_PSTATE_PACKED_DIRTY) == packed
            assert bool(state & P.CG_PSTATE_WIDE_DIRTY) == (nsums == 2 or not packed)
            agg.groups()
            direct = packed and nsums == 1
            assert bool(agg.packed_state()[2] & P.CG_PSTATE_READ_PACKED_DIRECT) == direct
            agg.scan_shard(rels[1].shard(cg))
            assert not agg.packed_state()[2] & P.CG_PSTATE_READ_PACKED_DIRECT
            assert answer(agg) == {k: v[:1 + nsums] for k, v in expect(rels[:2]).items()}
        finally:
            agg.free()


# --------------------------------------------------------------------------- D. hash addressing
def hash_case(cg, keys, rows_per_key, seed, nsums=1, extra=(), chunk=1003, null_keys=0):
    rng = np.random.default_rng(seed)
    key = np.repeat(np.array(list(keys) + list(extra), np.int64), rows_per_key)
    key = key[rng.permutation(len(key))]
    n = len(key)
    cols = [key] + [rng.integers(-(1 << 30), 1 << 30, n) for _ in range(nsums)]
    nulls = None
    if null_keys:
        kn = np.zeros(n, bool)
        kn[rng.choice(n, null_keys, replace=False)] = True
        nulls = [kn] + [None] * nsums
    return Rel(cg, cols, nulls, stripe=chunk * 13, chunk=chunk)


@pytest.mark.parametrize("family", FAMILIES)
def test_keys_sharing_one_home_slot(cg, kernel_family, family):
    """3000 keys whose home slot is the table's last (a cluster that wraps to slot 0), with the NULL key and the key
    equal to the empty-slot value; 8191 keys on one home slot (a run just under the probe limit): exact"""
    kernel_family(family)
    cases = [(4096, 1024, [gt.key_with_home(4095, j, 4096) for j in range(3000)], [I64_MIN, I64_MAX, 0], 40),
             (16384, 4096, [gt.key_with_home(77, j, 16384) for j in range(8191)], [], 0)]
    for cap, eg, keys, extra, nk in cases:
        assert gt.hash_verdict(keys + extra, cap) == "exact"
        for packing in (True, False):
            r = hash_case(cg, keys, 3, cap, extra=extra, null_keys=nk)
            agg = partial(cg, [r], HASH, expected_groups=eg, packing=packing)
            try:
                assert agg.capacity == cap
                agg.scan_shard(r.shard(cg))
                assert answer(agg) == expect([r])
            finally:
                agg.free()


@pytest.mark.parametrize("family", FAMILIES)
def test_over_full_hash_table(cg, kernel_family, family):
    """1025 distinct keys in 1024 slots: CG_ETABLEFULL, never an answer"""
    P = capi()
    kernel_family(family)
    rng = np.random.default_rng(3)
    keys = [int(k) for k in rng.integers(-(1 << 62), 1 << 62, 1025)]
    assert gt.hash_verdict(keys, 1024) == "full"
    r = hash_case(cg, keys, 2, 4)
    for packing in (True, False):
        agg = partial(cg, [r], HASH, expected_groups=1, packing=packing)
        try:
            assert agg.capacity == 1024
            with pytest.raises(P.CitusGpuError) as e:
                agg.scan_shard(r.shard(cg))
                agg.groups()
            assert e.value.code == P.CG_ETABLEFULL
        finally:
            agg.free()


@pytest.mark.parametrize("family", FAMILIES)
def test_paired_update_at_odd_chunk_ends(cg, kernel_family, family):
    """packing off, hash tables with one and two single-word sums (the fast kernel's lane-paired update), odd row
    counts and chunk groups of 1003 and 1077 rows that end in the middle of a warp"""
    kernel_family(family)
    rng = np.random.default_rng(8)
    keys = [int(k) for k in rng.integers(-(1 << 62), 1 << 62, 700)]
    for nsums in (1, 2):
        for chunk, per in ((1003, 5), (1077, 3)):
            r = hash_case(cg, keys, per, chunk, nsums=nsums, chunk=chunk)
            agg = partial(cg, [r], HASH, expected_groups=700, packing=False)
            try:
                agg.scan_shard(r.shard(cg))
                assert answer(agg) == expect([r])
            finally:
                agg.free()


# --------------------------------------------------------------------------- E. dense addressing
@pytest.mark.parametrize("family", FAMILIES)
def test_dense_key_range_limit_and_int64_ends(cg, kernel_family, family):
    """a key range of 2^26 - 1 is a direct-indexed table, 2^26 a hash table; key ranges at both ends of int64"""
    kernel_family(family)
    rng = np.random.default_rng(12)
    for lo, hi, mode in ((0, (1 << 26) - 1, DENSE), (5, 5 + (1 << 26), HASH), (I64_MIN, I64_MIN + 99, DENSE),
                         (I64_MAX - 99, I64_MAX, DENSE), (-(1 << 25), (1 << 25) - 1, DENSE)):
        assert gt.table_shape(1, lo, hi, 0, 3).mode == mode
        n = 20_000
        key = lo + rng.integers(0, hi - lo + 1, n, dtype=np.int64)
        key[:2] = lo, hi
        r = Rel(cg, [key, rng.integers(-(1 << 33), 1 << 33, n)], chunk=5000)
        agg = partial(cg, [r], DENSE, expected_groups=n)
        try:
            assert agg.layout()[2] == (mode == DENSE)
            if mode == DENSE:
                assert agg.capacity == hi - lo + 1
            agg.scan_shard(r.shard(cg))
            assert answer(agg) == expect([r])
        finally:
            agg.free()


@pytest.mark.parametrize("family", FAMILIES)
def test_two_column_keys_at_the_int32_ends(cg, kernel_family, family):
    kernel_family(family)
    rng = np.random.default_rng(13)
    n = 12_000
    a = rng.choice([I32_MIN, I32_MIN + 1, I32_MIN + 2], n)
    b = rng.choice([I32_MAX - 2, I32_MAX - 1, I32_MAX], n)
    r = Rel(cg, [a, b, rng.integers(-10**6, 10**6, n)], attlens=[4, 4, 8], chunk=4000)
    agg = partial(cg, [r], DENSE, ngroup=2)
    try:
        assert agg.capacity == 9
        agg.scan_shard(r.shard(cg))
        got = answer(agg)
        assert {gt.s64(k): v for k, v in got.items()} == {gt.s64(k): v for k, v in expect([r], ngroup=2).items()}
    finally:
        agg.free()


@pytest.mark.parametrize("family", FAMILIES)
def test_dense_words_layout(cg, kernel_family, family):
    """dense_words after packed scans: the drained table, [entry][stride], NULL entry at capacity, padding 0; on a hash
    partial it is CG_EINVAL"""
    P = capi()
    kernel_family(family)
    if "rels" not in _LIFE:
        _LIFE["rels"] = life_rels(cg)
    rels = _LIFE["rels"]
    for nsums in (1, 2):
        for enqueue in (False, True):
            agg = partial(cg, rels, DENSE, nsums=nsums, max_rows=1 << 20)
            try:
                for r in rels:
                    agg.scan_shard(r.shard(cg))
                check_dense_words(agg, {k: v[:1 + nsums] for k, v in expect(rels).items()}, enqueue)
            finally:
                agg.free()
    agg = partial(cg, rels[:1], HASH, nsums=1, expected_groups=5000)
    try:
        for f in (agg.dense_words, agg.dense_words_enqueue):
            with pytest.raises(P.CitusGpuError) as e:
                f()
            assert e.value.code == P.CG_EINVAL
    finally:
        agg.free()


# --------------------------------------------------------------------------- F. per-lane cells
SUM_SIGNS = (-1, 1, 1, -1, -1)
# chunk groups per relation: at least cgs_per_cta (and at least two: no slicing) per CTA of the largest grid, 132 SMs x 8
# CTAs of 256 threads, so that every CTA of the first launch takes cgs_per_cta whole chunk groups and every lane of it sees
# cgs_per_cta * rows_per_cg_lane = 160 rows (10 000-row chunk groups: 4 x 40, 10 241: 3 x 42 = 126, 20 480: 2 x 80, 40 960:
# 1 x 160)
LANE_CAP_CGS = {10_000: 4288, 10_241: 3200, 20_480: 2150, 40_960: 2150}
_CAP = {}


def lane_cap_rel(cg, cg_rows):
    """(relation, shard, rows): an int2 key, 3 on every row, and five int4 sums at the narrow bound: -tb (the row count's
    partner: a lane's high half reaches -2^31 + 128 at 160 rows), +tb, +tb (a biased pair: the low half reaches
    2 tb * 160 = 2^32 - 256, the high half 2^31 - 128), -tb, -tb (the low half stays 0, the high half -2^31 + 128)"""
    if cg_rows not in _CAP:
        ncg = LANE_CAP_CGS[cg_rows]
        rel = cg.Relation.generate([(2, 0, 3, 3, 0)] + [(4, 0, s * TB, s * TB, 0) for s in SUM_SIGNS], ncg * cg_rows,
                                   seed=cg_rows, stripe_row_limit=cg_rows * 15, chunk_row_limit=cg_rows)
        _CAP[cg_rows] = (rel, cg.Shard(rel), ncg * cg_rows)
    return _CAP[cg_rows]


def sums_partial(cg, rel, nsums, rows):
    aggs = [cg.count_star()] + [cg.sum_(1 + i) for i in range(nsums)]
    d = cg.make_desc([], [0], aggs)
    kmin, kmax, bounds, n = cg.relation_bounds(rel, d)
    assert (kmin, kmax, n) == (3, 3, rows) and bounds[1:] == [TB] * nsums
    for a in aggs[1:]:
        a.term_abs_bound = TB
    return cg.GpuColumnarAgg(cg.make_desc([], [0], aggs), rel.column_descs(), kmin, kmax, n)


def possible_launches(ncg, cg_rows):
    """launches of the generated shared-memory kernel for ncg chunk groups, for every occupancy of 1..8 CTAs per SM"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert ncg >= max(gt.cgs_per_cta(cg_rows), 2) * sms * 8
    return {gt.jit_small_launches(ncg, cg_rows, sms * occ) for occ in range(1, 9)}


def cell_rel(cg, cg_rows, ncg, seed):
    """int2 key (three keys, one hot), five int4 sums at the narrow bound, signs as SUM_SIGNS"""
    rng = np.random.default_rng(seed)
    n = cg_rows * ncg
    key = np.where(rng.random(n) < 0.01, rng.integers(0, 3, n), 1)
    cols = [key] + [np.full(n, s * TB) for s in SUM_SIGNS]
    return Rel(cg, cols, attlens=[2, 4, 4, 4, 4, 4], stripe=cg_rows * 4, chunk=cg_rows)


@pytest.mark.parametrize("family", FAMILIES)
def test_narrow_cells_at_every_chunk_group_size(cg, kernel_family, family):
    """chunk groups of 10 000, 10 241, 20 480 and 40 960 rows, enough of them that every CTA of a launch takes 4, 3, 2
    and 1 whole chunk groups and every lane sees its full 160 (126 for 10 241) rows, with every term at +-tbound in the
    row count's partner and in two biased pairs: the sums are exact, and the generated kernel cuts the scan into as many
    launches as its per-CTA cap asks for.  Chunk groups of 40 961 rows exceed 160 rows per lane: the generated kernel
    declines them and the ahead-of-time shared-memory kernel takes them"""
    kernel_family(family)
    shape = gt.narrow_shape(1, [(TB, 1)] * 5)
    assert (shape.kind, shape.rows_partner, shape.pairs, shape.min_blocks) == ("small", 0, [(1, 2), (3, 4)], 4)
    for cg_rows, ncg in LANE_CAP_CGS.items():
        rel, shard, n = lane_cap_rel(cg, cg_rows)
        agg = sums_partial(cg, rel, 5, n)
        try:
            j0 = jit_launches()
            agg.scan_shard(shard)
            launches = jit_launches() - j0
            if family in ("jit", "jit_always"):
                assert launches in possible_launches(ncg, cg_rows) and launches >= 2, (cg_rows, launches)
            else:
                assert launches == 0
            got = agg.groups()
            assert list(got) == [3] and got[3][0]["count"] == n
            for i, sign in enumerate(SUM_SIGNS):
                assert (got[3][1 + i]["count"], got[3][1 + i]["sum"]) == (n, sign * TB * n), (cg_rows, i)
        finally:
            agg.free()
    r = cell_rel(cg, 40_961, 9, 40_961)
    agg = partial(cg, [r], DENSE)
    try:
        j0 = jit_launches()
        agg.scan_shard(r.shard(cg))
        assert jit_launches() == j0 and gt.cgs_per_cta(40_961) == 0
        assert answer(agg) == expect([r])
    finally:
        agg.free()


@pytest.mark.parametrize("family", FAMILIES)
def test_long_scan_cuts_the_generated_kernels_launches(cg, kernel_family, family):
    """4288 chunk groups of 10 000 rows in one group, count(*) and sum(x) with x = -tbound: the sum rides in the high half
    of the row count's cell.  More chunk groups than 4 per CTA of the largest grid, so the generated kernel must cut the
    scan into two launches or more, and no lane may see more than 160 rows of a launch (200 terms at -tbound leave the
    32-bit half)"""
    kernel_family(family)
    rel, shard, n = lane_cap_rel(cg, 10_000)
    agg = sums_partial(cg, rel, 1, n)
    try:
        j0 = jit_launches()
        agg.scan_shard(shard)
        if family in ("jit", "jit_always"):
            assert jit_launches() - j0 in possible_launches(LANE_CAP_CGS[10_000], 10_000)
            assert jit_launches() - j0 >= 2
        got = agg.groups()
        assert got[3][0]["count"] == n and got[3][1]["count"] == n and got[3][1]["sum"] == -n * TB
    finally:
        agg.free()


_LIMIT_RELS = {}


@pytest.mark.parametrize("family", FAMILIES)
def test_shared_memory_limits(cg, kernel_family, family):
    """count(*) and sum(x), x = +-tbound, over 25, 26, 50, 51, 100 and 101 keys on 8-byte columns.  The generated kernel
    keeps its shared-memory kind while capacity x cells x 2 KB fits 200 KB (one cell: 100 entries; four CTAs per SM up to
    25), the ahead-of-time one while its two hot words fit (50 entries); past them the table kernels (the fast kernel
    first) take the scan.  Which one ran shows in cg_jit_launches and in the packed words, which only the table kernels
    write.  Every answer is exact"""
    P = capi()
    kernel_family(family)
    for cap in (25, 26, 50, 51, 100, 101):
        if cap not in _LIMIT_RELS:
            rng = np.random.default_rng(cap)
            n = 90_000
            key = rng.integers(0, cap, n)
            key[:2] = 0, cap - 1
            _LIMIT_RELS[cap] = Rel(cg, [key, np.where(rng.random(n) < 0.5, -TB, TB)])
        r = _LIMIT_RELS[cap]
        jit_small = gt.narrow_shape(cap, [(TB, 1)])
        aot_small = gt.interp_small_eligible(cap, 2)
        assert (jit_small.kind == "small", jit_small.min_blocks == 4, aot_small) == (cap <= 100, cap <= 25, cap <= 50)
        ran_jit = {"jit": aot_small, "jit_always": True, "aot": False, "general": False}[family]
        packed = {"jit": not aot_small, "jit_always": jit_small.kind == "table", "aot": not aot_small, "general": False}[family]
        agg = partial(cg, [r], DENSE)
        try:
            assert agg.capacity == cap
            j0 = jit_launches()
            agg.scan_shard(r.shard(cg))
            assert (jit_launches() > j0, bool(agg.packed_state()[2] & P.CG_PSTATE_PACKED_DIRTY)) == (ran_jit, packed), cap
            assert answer(agg) == expect([r])
        finally:
            agg.free()
