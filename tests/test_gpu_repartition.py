"""The map side of the hash repartition on the GPU against the plain reference (tests/partition_reference.py), exactly,
row order included: routing (cg_partition_index and the exchange's route_row, whose uniform shortcut divides or
shifts and clamps into the widened last interval, and searches caller bounds), the stable scatter (the multi-chunk
offset scan past 2048 blocks, skewed partitions, caller-chosen partition order), the one-GPU repartition exchange
and the join over its partitions, and the COPY text / binary partition files at the edges of decimal lengths, of the
column and partition limits and of the output capacity."""
import ctypes as C

import numpy as np
import pytest

import partition_reference as pr
from gpu_harness import cg  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

PS = [1, 2, 3, 7, 32, 255, 256, 257, 1000, 1024]
CHUNK_ROWS = 2048 * 4096          # the offset scan's chunk of 2048 blocks of 4096 rows
W = 64                             # hash values searched on either side of every interval boundary


def _dev(a, dtype=np.int64):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def _host(ptr, n, typestr="<i8"):
    """a copy of n values at a device address the library owns"""
    import torch

    class View:
        def __init__(self):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}
    if n == 0:
        return np.zeros(0, np.int64)
    return torch.as_tensor(View(), device="cuda").cpu().numpy()


def _lib():
    from citus_b200 import capi
    return capi.lib()


def _err():
    return _lib().cg_last_error().decode()


# --------------------------------------------------------------------------- keys whose hashes hit chosen values
def _hash_uint32_torch(k):
    """hash_uint32 over an int64 tensor of values in [0, 2^32): only used to find keys, which the reference re-checks"""
    M = 0xFFFFFFFF

    def rot(x, s):
        return ((x << s) & M) | (x >> (32 - s))
    init = pr._INIT
    a = (k + init) & M
    c = ((init ^ init) - pr._rot(init, 14)) & M              # b = c = init: the first line is a constant
    a = ((a ^ c) - rot(c, 11)) & M
    b = ((a ^ init) - rot(a, 25)) & M
    c = ((b ^ c) - rot(b, 16)) & M
    a = ((a ^ c) - rot(c, 4)) & M
    b = ((b ^ a) - rot(a, 14)) & M
    c = ((c ^ b) - rot(b, 24)) & M
    return c


def _boundary_windows(P):
    """hash values within W of every boundary of the synthetic intervals of P, the ends, and the widened top"""
    mins, _ = pr.synthetic_intervals(P)
    w = [np.arange(b - W, b + W, dtype=np.int64) for b in mins[1:]]
    w += [np.arange(pr.INT32_MIN, pr.INT32_MIN + W, dtype=np.int64), np.arange(pr.INT32_MAX - W + 1, pr.INT32_MAX + 1, dtype=np.int64)]
    top = pr.INT32_MIN + P * (pr.HASH_TOKEN_COUNT // P)
    w.append(np.arange(top - W, pr.INT32_MAX + 1, dtype=np.int64))
    return np.unique(np.concatenate(w))


@pytest.fixture(scope="module")
def preimages(cg):
    """(hashes, uint32 keys) of EVERY 32-bit key whose hash lies in the boundary windows of every P in PS: an
    exhaustive search over 2^32 keys on the GPU, so the nearest reachable hash on either side of a boundary is known"""
    import torch
    targets = np.unique(np.concatenate([_boundary_windows(P) for P in PS]))
    T = torch.from_numpy(np.sort(targets & 0xFFFFFFFF)).cuda()
    hs, ks = [], []
    B = 1 << 23
    for start in range(0, 1 << 32, B):
        k = torch.arange(start, start + B, dtype=torch.int64, device="cuda")
        h = _hash_uint32_torch(k)
        i = torch.searchsorted(T, h).clamp_(max=T.numel() - 1)
        hit = T[i] == h
        hs.append(h[hit].cpu())
        ks.append(k[hit].cpu())
        del k, h, i, hit
    h = torch.cat(hs).numpy().astype(np.uint32).view(np.int32).astype(np.int64)
    k = torch.cat(ks).numpy().astype(np.uint32)
    torch.cuda.empty_cache()
    assert np.array_equal(pr.hash_uint32_np(k).view(np.int32), h)          # the reference confirms every find
    o = np.argsort(h, kind="stable")
    return h[o], k[o]


def _keys_for_hashes(u32, key_len, rng):
    """keys of key_len 4 or 8 whose hashint4 / hashint8 equals hash_uint32 of u32: the int4 value, and for int8 the
    same low word with a zero and an all-ones high word (both signs) and with random high words folded in"""
    u32 = np.asarray(u32, np.uint32)
    if key_len == 4:
        return u32.view(np.int32).astype(np.int64)
    hi = rng.integers(0, 1 << 32, len(u32), dtype=np.uint64).astype(np.uint32)
    lo = u32 ^ np.where(hi < (1 << 31), hi, ~hi)
    folded = ((hi.astype(np.uint64) << np.uint64(32)) | lo.astype(np.uint64)).view(np.int64)
    return np.concatenate([u32.astype(np.int64), u32.astype(np.int64) - (1 << 32), folded])


def _synthetic_case(preimages, P, key_len, rng, extra=20_000):
    """keys that hit both sides of every synthetic boundary as tightly as any key can, the widened top, random keys
    and NULLs; asserts that every target was reached"""
    H, K = preimages
    mins, _ = pr.synthetic_intervals(P)
    for b in mins[1:]:
        below = H[(H < b) & (H >= b - W)]
        above = H[(H >= b) & (H < b + W)]
        assert below.size and above.size, (P, b)
    top = pr.INT32_MIN + P * (pr.HASH_TOKEN_COUNT // P)
    if top <= pr.INT32_MAX:
        assert (H >= top).any(), P                                  # a key in the clamped top of the last interval
    assert H[0] == pr.INT32_MIN and H[-1] == pr.INT32_MAX
    sel = np.isin(H, _boundary_windows(P))
    keys = _keys_for_hashes(K[sel], key_len, rng)
    lo, hi = (pr.INT32_MIN, pr.INT32_MAX) if key_len == 4 else (pr.INT64_MIN, pr.INT64_MAX)
    nulls = np.concatenate([np.zeros(len(keys), np.uint8), (rng.random(extra) < 0.05).astype(np.uint8)])
    keys = np.concatenate([keys, rng.integers(lo, hi, extra, dtype=np.int64, endpoint=True)])
    perm = rng.permutation(len(keys))
    return keys[perm], nulls[perm], mins, pr.synthetic_intervals(P)[1]


def _caller_bounds(preimages, P, rng):
    """P contiguous-where-it-matters intervals whose every min and max is the hash of a key (from the preimage pool):
    cuts between two consecutive reachable hashes h, h + 1, plus width-1 intervals [INT32_MIN, INT32_MIN] and
    [INT32_MAX, INT32_MAX] next to gaps that no key can reach"""
    H, _ = preimages
    h = np.unique(H)
    m = len(h)
    assert h[1] < pr.INT32_MIN + W and h[-2] > pr.INT32_MAX - W      # the gaps below are empty of reachable hashes
    if P == 1:
        return [pr.INT32_MIN], [pr.INT32_MAX]
    adj = np.flatnonzero(np.diff(h) == 1)
    adj = adj[(adj > 0) & (adj < m - 2)]
    pairs = adj[np.isin(adj + 1, adj)]
    cuts = {0} if P == 2 else {0, m - 2}
    for c in rng.permutation(pairs)[:max(0, (P - 3) // 4)]:
        if len(cuts) + 2 <= P - 1:
            cuts.update((int(c), int(c) + 1))                        # a width-1 interval [h[c + 1], h[c + 1]]
    for c in rng.permutation(adj):
        if len(cuts) >= P - 1:
            break
        cuts.add(int(c))
    cuts = sorted(cuts)
    assert len(cuts) == P - 1
    mins = [pr.INT32_MIN] + [int(h[c + 1]) for c in cuts]
    maxs = [int(h[c]) for c in cuts] + [pr.INT32_MAX]
    return mins, maxs


def _partition_index(keys, nulls, key_len, by_hash, mins, maxs):
    import torch
    n = len(keys)
    dk = _dev(keys)
    dn = _dev(nulls, np.uint8) if nulls is not None else None
    idx = torch.empty(max(n, 1), dtype=torch.int32, device="cuda")
    cnt = torch.empty(max(len(mins), 1) + 1, dtype=torch.int64, device="cuda")
    mins = np.ascontiguousarray(mins, np.int32)
    maxs = np.ascontiguousarray(maxs, np.int32)
    torch.cuda.synchronize()
    rc = _lib().cg_partition_index(dk.data_ptr(), dn.data_ptr() if dn is not None else None, n, key_len, by_hash,
                                   mins.ctypes.data, maxs.ctypes.data, len(mins), idx.data_ptr(), cnt.data_ptr())
    if rc:
        return rc, None, None
    return 0, idx[:n].cpu().numpy().astype(np.int64), cnt[:len(mins)].cpu().numpy()


# --------------------------------------------------------------------------- routing
@pytest.mark.parametrize("key_len", [4, 8])
@pytest.mark.parametrize("P", PS)
def test_hash_routing_synthetic_bounds(cg, preimages, P, key_len):
    rng = np.random.default_rng(P * 10 + key_len)
    keys, nulls, mins, maxs = _synthetic_case(preimages, P, key_len, rng)
    want_idx, want_cnt, bad = pr.route(keys, nulls, key_len, "hash", mins, maxs)
    assert bad == 0
    assert np.array_equal(want_idx[nulls == 0], pr.uniform_index(
        (pr.hashint4_np(keys) if key_len == 4 else pr.hashint8_np(keys))[nulls == 0].astype(np.int64), P))
    rc, idx, cnt = _partition_index(keys, nulls, key_len, 1, mins, maxs)
    assert rc == 0, _err()
    assert np.array_equal(idx, want_idx)
    assert np.array_equal(cnt, want_cnt)


@pytest.mark.parametrize("key_len", [4, 8])
@pytest.mark.parametrize("P", PS)
def test_hash_routing_caller_bounds(cg, preimages, P, key_len):
    rng = np.random.default_rng(1000 + P * 10 + key_len)
    mins, maxs = _caller_bounds(preimages, P, rng)
    H, K = preimages
    keys = _keys_for_hashes(K, key_len, rng)
    lo, hi = (pr.INT32_MIN, pr.INT32_MAX) if key_len == 4 else (pr.INT64_MIN, pr.INT64_MAX)
    nulls = np.concatenate([np.zeros(len(keys), np.uint8), (rng.random(20_000) < 0.05).astype(np.uint8)])
    keys = np.concatenate([keys, rng.integers(lo, hi, 20_000, dtype=np.int64, endpoint=True)])
    perm = rng.permutation(len(keys))
    keys, nulls = keys[perm], nulls[perm]
    hashes = pr.hashint4_np(keys) if key_len == 4 else pr.hashint8_np(keys)
    hs = set(hashes[nulls == 0].tolist())
    assert all(m in hs and x in hs for m, x in zip(mins, maxs))          # rows on every min and every max
    if P >= 8:
        assert sum(m == x for m, x in zip(mins, maxs)) >= 3               # width-1 intervals, at both ends too
        assert mins[0] == maxs[0] == pr.INT32_MIN and mins[-1] == maxs[-1] == pr.INT32_MAX
    want_idx, want_cnt, bad = pr.route(keys, nulls, key_len, "hash", mins, maxs)
    assert bad == 0
    rc, idx, cnt = _partition_index(keys, nulls, key_len, 1, mins, maxs)
    assert rc == 0, _err()
    assert np.array_equal(idx, want_idx)
    assert np.array_equal(cnt, want_cnt)


def test_key_len_8_routes_int4_values_like_key_len_4(cg):
    rng = np.random.default_rng(48)
    keys = np.concatenate([rng.integers(pr.INT32_MIN, pr.INT32_MAX, 200_000, endpoint=True),
                           [0, -1, 1, pr.INT32_MIN, pr.INT32_MAX]])
    for P in (7, 1000):
        mins, maxs = pr.synthetic_intervals(P)
        rc4, idx4, _ = _partition_index(keys, None, 4, 1, mins, maxs)
        rc8, idx8, _ = _partition_index(keys, None, 8, 1, mins, maxs)
        assert rc4 == rc8 == 0
        assert np.array_equal(idx4, idx8)
        assert np.array_equal(idx8, pr.route(keys, None, 8, "hash", mins, maxs)[0])


@pytest.mark.parametrize("key_len", [4, 8])
@pytest.mark.parametrize("P", [1, 2, 3, 257, 1024])
def test_range_routing(cg, P, key_len):
    rng = np.random.default_rng(2000 + P + key_len)
    # contiguous intervals over the int4 range: width-1 intervals at INT32_MAX, at INT32_MIN and in between
    starts = {pr.INT32_MIN}
    if P >= 2:
        starts.add(pr.INT32_MAX)
    if P >= 3:
        starts.add(pr.INT32_MIN + 1)
    while len(starts) < P:
        x = int(rng.integers(pr.INT32_MIN + 2, pr.INT32_MAX - 1))
        starts.add(x)
        if len(starts) < P and rng.random() < 0.3:
            starts.add(x + 1)
    starts = sorted(starts)
    mins, maxs = starts, [s - 1 for s in starts[1:]] + [pr.INT32_MAX]
    if P >= 32:
        assert sum(m == x for m, x in zip(mins, maxs)) >= 3
    b = np.array(mins + maxs, np.int64)
    keys = np.unique(np.clip(np.concatenate([b - 1, b, b + 1]), pr.INT32_MIN, pr.INT32_MAX))
    keys = np.concatenate([keys, rng.integers(pr.INT32_MIN, pr.INT32_MAX, 10_000, endpoint=True)])
    nulls = (rng.random(len(keys)) < 0.02).astype(np.uint8)
    want_idx, want_cnt, bad = pr.route(keys, nulls, key_len, "range", mins, maxs)
    assert bad == 0
    rc, idx, cnt = _partition_index(keys, nulls, key_len, 0, mins, maxs)
    assert rc == 0, _err()
    assert np.array_equal(idx, want_idx) and np.array_equal(cnt, want_cnt)


def test_routing_refusals(cg):
    from citus_b200 import capi
    # a hash in a gap between caller bounds: "could not find shard"
    keys = np.arange(1000)
    mins, maxs = [pr.INT32_MIN, 0], [-1 << 30, pr.INT32_MAX]        # (-2^30, 0) is a gap
    assert pr.route(keys, None, 8, "hash", mins, maxs)[2] > 0
    rc, _, _ = _partition_index(keys, None, 8, 1, mins, maxs)
    assert rc == capi.CG_EINVAL and "could not find shard" in _err()
    # an int8 range key outside the int4 bounds lies in no interval: it is not truncated into one
    for k in (1 << 31, -(1 << 31) - 1, 1 << 32, pr.INT64_MIN):
        assert pr.route([k], None, 8, "range", [pr.INT32_MIN], [pr.INT32_MAX])[2] == 1
        rc, _, _ = _partition_index(np.array([5, k]), None, 8, 0, [pr.INT32_MIN], [pr.INT32_MAX])
        assert rc == capi.CG_EINVAL and "could not find shard" in _err(), k
    # P = 0 and P past the limit
    rc, _, _ = _partition_index(keys, None, 8, 1, [], [])
    assert rc == capi.CG_EINVAL
    mins, maxs = pr.synthetic_intervals(1025)
    rc, _, _ = _partition_index(keys, None, 8, 1, mins, maxs)
    assert rc == capi.CG_EUNSUPPORTED
    rc, _, _ = _partition_index(keys, None, 8, 1, *pr.synthetic_intervals(1024))
    assert rc == 0


# --------------------------------------------------------------------------- stable scatter
def _scatter(index, cols, P, order=None):
    """(rc, columns, offsets) of cg_partition_scatter / cg_partition_scatter_ordered"""
    import torch
    n = len(index)
    di = _dev(index, np.int32)
    dc = [_dev(c) for c in cols]
    do = [torch.full((max(n, 1),), -7, dtype=torch.int64, device="cuda") for _ in cols]
    cp = (C.c_void_p * max(len(cols), 1))(*[c.data_ptr() for c in dc])
    op = (C.c_void_p * max(len(cols), 1))(*[c.data_ptr() for c in do])
    offs = np.zeros(P + 1, np.int64)
    torch.cuda.synchronize()
    if order is None:
        rc = _lib().cg_partition_scatter(di.data_ptr(), n, P, cp, len(cols), op, offs.ctypes.data)
    else:
        o = np.ascontiguousarray(order, np.int32)
        rc = _lib().cg_partition_scatter_ordered(di.data_ptr(), n, P, o.ctypes.data, cp, len(cols), op, offs.ctypes.data)
    if rc:
        return rc, None, None
    torch.cuda.synchronize()
    return 0, [c[:n].cpu().numpy() for c in do], offs


def _check_scatter(index, cols, P, order=None):
    rc, got, offs = _scatter(index, cols, P, order)
    assert rc == 0, _err()
    want, want_offs = pr.stable_scatter(index, cols, P, order)
    assert np.array_equal(offs, want_offs)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 4095, 4096, 4097, 8 * 4096 + 1])
@pytest.mark.parametrize("P", [1, 3, 1024])
def test_scatter_sizes(cg, n, P):
    rng = np.random.default_rng(n * 7 + P)
    index = rng.integers(0, P, n)
    cols = [rng.integers(pr.INT64_MIN, pr.INT64_MAX, n, dtype=np.int64, endpoint=True), np.arange(n, dtype=np.int64)]
    _check_scatter(index, cols, P)


@pytest.mark.parametrize("n,P", [(CHUNK_ROWS + 1, 3), (CHUNK_ROWS + 1, 1024), (2 * CHUNK_ROWS + 4097, 257)])
def test_scatter_past_the_scan_chunk(cg, n, P):
    """more than 2048 blocks: the offset scan carries partition totals from one chunk of blocks to the next"""
    rng = np.random.default_rng(n + P)
    index = rng.integers(0, P, n)
    index[:4096] = P - 1                                           # an uneven first block
    _check_scatter(index, [np.arange(n, dtype=np.int64)], P)


def _skewed(kind, n, P):
    r = np.arange(n)
    if kind == "one partition":
        return np.full(n, P - 1)
    if kind == "lanes of a step":
        return (r // 32) % P                                       # all 32 lanes of a warp step in one partition
    if kind == "partition per block":
        return (r // 4096 * 37) % P
    if kind == "alternating":
        return r % 2 * (P - 1)
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["one partition", "lanes of a step", "partition per block", "alternating"])
@pytest.mark.parametrize("P", [2, 1024])
def test_scatter_skew(cg, kind, P):
    n = 9 * 4096 + 123
    index = _skewed(kind, n, P)
    rng = np.random.default_rng(9)
    _check_scatter(index, [rng.integers(pr.INT64_MIN, pr.INT64_MAX, n, dtype=np.int64, endpoint=True)], P)


def test_scatter_eight_columns_and_nine_refused(cg):
    from citus_b200 import capi
    rng = np.random.default_rng(88)
    n, P = 3 * 4096 + 5, 257
    index = rng.integers(0, P, n)
    cols = [rng.integers(pr.INT64_MIN, pr.INT64_MAX, n, dtype=np.int64, endpoint=True) for _ in range(8)]
    _check_scatter(index, cols, P)
    rc, _, _ = _scatter(index, cols + [cols[0]], P)
    assert rc == capi.CG_EUNSUPPORTED


@pytest.mark.parametrize("P", [1, 7, 1024])
def test_scatter_ordered(cg, P):
    """cg_partition_scatter_ordered: h_offsets[i]..h_offsets[i + 1] delimit the partition at position i"""
    from citus_b200 import capi
    rng = np.random.default_rng(P + 5)
    n = 5 * 4096 + 77
    index = rng.integers(0, P, n)
    index[rng.random(n) < 0.3] = P - 1
    cols = [rng.integers(pr.INT64_MIN, pr.INT64_MAX, n, dtype=np.int64, endpoint=True), np.arange(n, dtype=np.int64)]
    for order in (np.arange(P), np.arange(P)[::-1].copy(), rng.permutation(P)):
        _check_scatter(index, cols, P, order)
        rc, got, offs = _scatter(index, cols, P, order)
        inv = np.argsort(order)                                      # partition at position i
        for i in range(P):
            assert np.array_equal(got[1][offs[i]:offs[i + 1]], np.flatnonzero(index == inv[i]))
    bad = [np.zeros(P, np.int32), np.arange(P) + 1, np.arange(P) - 1]
    for order in bad[0 if P > 1 else 1:]:
        rc, _, _ = _scatter(index, cols, P, order)
        assert rc == capi.CG_EINVAL and "permutation" in _err()


def test_scatter_refusals(cg):
    from citus_b200 import capi
    index = np.zeros(10)
    for P in (0, 1025):
        rc, _, _ = _scatter(index, [np.arange(10)], P)
        assert rc == capi.CG_EINVAL


# --------------------------------------------------------------------------- the one-GPU repartition exchange
@pytest.fixture(scope="module")
def comm(cg):
    from citus_b200 import distributed
    distributed.init(0, 1)
    yield distributed
    distributed.destroy()


def _exchange(slot, cols, nulls, key_len, mins, maxs):
    """(rc, received columns, part_counts[P]) of cg_comm_repartition_exchange over device copies of cols"""
    import torch
    n = len(cols[0])
    dc = [_dev(c) for c in cols]
    dn = _dev(nulls, np.uint8) if nulls is not None else None
    mins = np.ascontiguousarray(mins, np.int32)
    maxs = np.ascontiguousarray(maxs, np.int32)
    P = len(mins)
    cp = (C.c_void_p * len(cols))(*[c.data_ptr() for c in dc])
    got = C.c_int64(-1)
    torch.cuda.synchronize()
    rc = _lib().cg_comm_repartition_exchange(slot, cp, dn.data_ptr() if dn is not None else None, n, len(cols), key_len, P,
                                             mins.ctypes.data, maxs.ctypes.data, C.byref(got))
    if rc:
        return rc, None, None
    assert got.value == n                                          # one rank receives every row
    assert _lib().cg_comm_exchange_wait(slot) == 0 and _lib().cg_synchronize() == 0
    return 0, *_exchange_result(slot, len(cols), P)


def _exchange_result(slot, ncols, P):
    ptrs = (C.c_void_p * 8)()
    nrows, nlocal = C.c_int64(), C.c_int32()
    counts = np.full(P, -1, np.int64)
    assert _lib().cg_comm_exchange_result(slot, ptrs, C.byref(nrows), counts.ctypes.data, C.byref(nlocal), None, None) == 0
    assert nlocal.value == P
    return [_host(ptrs[c] or 0, nrows.value) for c in range(ncols)], counts


def _check_exchange(slot, cols, nulls, key_len, mins, maxs):
    rc, got, counts = _exchange(slot, cols, nulls, key_len, mins, maxs)
    assert rc == 0, _err()
    P = len(mins)
    idx, want_counts, bad = pr.route(cols[0], nulls, key_len, "hash", mins, maxs)
    assert bad == 0
    want, offs = pr.stable_scatter(idx, cols, P)
    assert np.array_equal(counts, want_counts)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    return got, counts


@pytest.mark.parametrize("ncols", [1, 8])
@pytest.mark.parametrize("key_len", [4, 8])
@pytest.mark.parametrize("P", [1, 3, 7, 8, 1000])
def test_exchange_synthetic_bounds(cg, comm, preimages, P, key_len, ncols):
    """P = 8: the shift; 3, 7, 1000: the division and the clamp into the widened last interval; 1: the search"""
    rng = np.random.default_rng(3000 + P * 100 + key_len * 10 + ncols)
    keys, nulls, mins, maxs = _synthetic_case(preimages, P, key_len, rng)
    cols = [keys] + [rng.integers(pr.INT64_MIN, pr.INT64_MAX, len(keys), dtype=np.int64, endpoint=True) for _ in range(ncols - 1)]
    _check_exchange(0, cols, nulls, key_len, mins, maxs)


@pytest.mark.parametrize("key_len", [4, 8])
@pytest.mark.parametrize("P", [2, 257, 1024])
def test_exchange_caller_bounds(cg, comm, preimages, P, key_len):
    """bounds that are not the synthetic ones take route_row's interval search"""
    rng = np.random.default_rng(4000 + P + key_len)
    mins, maxs = _caller_bounds(preimages, P, rng)
    keys = _keys_for_hashes(preimages[1], key_len, rng)
    keys = keys[rng.permutation(len(keys))]
    nulls = (rng.random(len(keys)) < 0.01).astype(np.uint8)
    _check_exchange(1, [keys, np.arange(len(keys), dtype=np.int64)], nulls, key_len, mins, maxs)


def test_exchange_sizes_and_slots(cg, comm):
    """n = 0, n past the offset scan's chunk of blocks, two slots alive at once, a slot reused larger then smaller"""
    rng = np.random.default_rng(77)
    mins, maxs = pr.synthetic_intervals(1000)
    empty = np.zeros(0, np.int64)
    got, counts = _check_exchange(2, [empty, empty], None, 8, mins, maxs)
    assert counts.sum() == 0 and len(got[0]) == 0
    big = CHUNK_ROWS + 4097
    kb = rng.integers(pr.INT64_MIN, pr.INT64_MAX, big, dtype=np.int64, endpoint=True)
    nb = (rng.random(big) < 0.001).astype(np.uint8)
    big_got, _ = _check_exchange(2, [kb, np.arange(big, dtype=np.int64)], nb, 8, mins, maxs)
    ks = rng.integers(-1000, 1000, 5000)
    small_got, _ = _check_exchange(3, [ks, -ks], None, 4, *pr.synthetic_intervals(7))
    # slot 2 still holds the large result while slot 3 holds the small one
    again, counts = _exchange_result(2, 2, 1000)
    assert np.array_equal(again[0], big_got[0]) and np.array_equal(again[1], big_got[1])
    again, _ = _exchange_result(3, 2, 7)
    assert np.array_equal(again[0], small_got[0])
    _check_exchange(2, [ks[:100], ks[:100]], None, 8, mins, maxs)         # the large slot reused with fewer rows


def test_exchange_unroutable_key_is_refused(cg, comm):
    from citus_b200 import capi
    keys = np.arange(1000)
    mins, maxs = [pr.INT32_MIN, 0], [-1 << 30, pr.INT32_MAX]        # (-2^30, 0) is a gap
    assert pr.route(keys, None, 8, "hash", mins, maxs)[2] > 0
    rc, _, _ = _exchange(3, [keys], None, 8, mins, maxs)
    assert rc == capi.CG_EINVAL and "could not find shard" in _err()
    rc, _, _ = _exchange(3, [keys], None, 8, *pr.synthetic_intervals(1025))
    assert rc == capi.CG_EINVAL


# --------------------------------------------------------------------------- exchange -> join
def _join_reference(bk, bp, pk, pp):
    """(rows, exact sum(b.payload + p.payload), the joined rows sorted) of an equi-join on NULL-free keys"""
    ub, ib, cb = np.unique(bk, return_inverse=True, return_counts=True)
    up, ip, cp = np.unique(pk, return_inverse=True, return_counts=True)
    common, xb, xp = np.intersect1d(ub, up, assume_unique=True, return_indices=True)
    nb = np.zeros(len(ub), np.int64); nb[xb] = cp[xp]                 # matches of every build row's key
    npb = np.zeros(len(up), np.int64); npb[xp] = cb[xb]
    rows = int((cb[xb] * cp[xp]).sum())
    total = sum(int(v) * int(m) for v, m in zip(bp, nb[ib]) if m) + sum(int(v) * int(m) for v, m in zip(pp, npb[ip]) if m)
    ob, op = np.argsort(bk, kind="stable"), np.argsort(pk, kind="stable")
    bs = np.searchsorted(bk[ob], common); ps = np.searchsorted(pk[op], common)
    sizes = cb[xb] * cp[xp]
    g = np.repeat(np.arange(len(common)), sizes)
    within = np.arange(rows) - np.repeat(np.cumsum(sizes) - sizes, sizes)
    i = ob[bs[g] + within // cp[xp][g]]
    j = op[ps[g] + within % cp[xp][g]]
    out = np.stack([bk[i], bp[i], pp[j]])
    return rows, total, out[:, np.lexsort(out[::-1])]


def test_exchange_then_join(cg, comm):
    import torch
    rng = np.random.default_rng(90)
    P = 8
    mins, maxs = pr.synthetic_intervals(P)
    big = (1 << 63) - 1
    nb, npr = 400_000, 300_000
    bk = rng.integers(-50_000, 50_000, nb)
    pk = rng.integers(-50_000, 50_000, npr)
    bk[:3000] = 123456789                                               # one key with 3000 x 3000 matches
    pk[:3000] = 123456789
    bk[3000:3010] = pr.INT64_MIN                                        # the join table's EMPTY key
    pk[3000:3004] = pr.INT64_MIN
    bp = rng.integers(-(1 << 62), 1 << 62, nb)
    pp = rng.integers(-(1 << 62), 1 << 62, npr)
    bp[:1500], pp[:1500] = big, big
    bp[1500:3000], pp[1500:2000] = pr.INT64_MIN, -big
    bp[3000:3005] = big
    pb, pq = rng.permutation(nb), rng.permutation(npr)
    bk, bp, pk, pp = bk[pb], bp[pb], pk[pq], pp[pq]
    b, _ = _check_exchange(0, [bk, bp], None, 8, mins, maxs)
    p, _ = _check_exchange(1, [pk, pp], None, 8, mins, maxs)
    # the two received tables stay in their slots: join partition by partition on the device
    ptr_b = (C.c_void_p * 8)(); ptr_p = (C.c_void_p * 8)()
    cnt_b, cnt_p = np.zeros(P, np.int64), np.zeros(P, np.int64)
    assert _lib().cg_comm_exchange_result(0, ptr_b, None, cnt_b.ctypes.data, None, None, None) == 0
    assert _lib().cg_comm_exchange_result(1, ptr_p, None, cnt_p.ctypes.data, None, None, None) == 0
    ob, op = np.concatenate([[0], np.cumsum(cnt_b)]), np.concatenate([[0], np.cumsum(cnt_p)])
    for q in range(P):
        sb, sp = slice(ob[q], ob[q + 1]), slice(op[q], op[q + 1])
        want_rows, want_sum, want = _join_reference(b[0][sb], b[1][sb], p[0][sp], p[1][sp])
        a = [ptr_b[0] + 8 * int(ob[q]), ptr_b[1] + 8 * int(ob[q]), ptr_p[0] + 8 * int(op[q]), ptr_p[1] + 8 * int(op[q])]
        rows, s = cg.join_count_sum(a[0], a[1], int(cnt_b[q]), a[2], a[3], int(cnt_p[q]))
        assert (rows, s) == (want_rows, want_sum), q
        n = cg.join_rows(a[0], a[1], int(cnt_b[q]), a[2], a[3], int(cnt_p[q]))
        assert n == want_rows
        out = [torch.empty(max(n, 1), dtype=torch.int64, device="cuda") for _ in range(3)]
        n2 = cg.join_rows(a[0], a[1], int(cnt_b[q]), a[2], a[3], int(cnt_p[q]), capacity=n, d_out=[o.data_ptr() for o in out])
        assert n2 == n
        got = np.stack([o[:n].cpu().numpy() for o in out])
        assert np.array_equal(got[:, np.lexsort(got[::-1])], want), q
    assert any(123456789 in b[0][ob[q]:ob[q + 1]] for q in range(P))


# --------------------------------------------------------------------------- COPY partition files
def _files(index, cols, lens, P, binary, nulls=None, gen_empty=False, capacity_delta=0):
    """(rc, files, rows, bytes) of cg_partition_copy_bytes + cg_partition_copy_serialize"""
    import torch
    from citus_b200 import capi
    n = len(index)
    di = _dev(index, np.int32)
    dc = [_dev(c) for c in cols]
    dn = None if nulls is None else [None if x is None else _dev(x, np.uint8) for x in nulls]
    nptr = None if dn is None else [None if x is None else x.data_ptr() for x in dn]
    torch.cuda.synchronize()
    rows, nbytes = cg_mod().partition_copy_bytes(di.data_ptr(), n, P, [c.data_ptr() for c in dc], lens, binary, d_null_ptrs=nptr,
                                                 generate_empty_results=gen_empty)
    total = int(nbytes.sum())
    out = torch.full((total + 4096,), 0xA5, dtype=torch.uint8, device="cuda")
    try:
        offs = cg_mod().partition_copy_serialize(di.data_ptr(), n, P, [c.data_ptr() for c in dc], lens, binary, out.data_ptr(),
                                                 total + capacity_delta, d_null_ptrs=nptr, generate_empty_results=gen_empty)
    except capi.CitusGpuError as e:
        host = out.cpu().numpy()
        assert (host == 0xA5).all(), "a refused call wrote into the output"
        return e.code, None, rows, nbytes
    assert np.array_equal(np.diff(offs), nbytes) and offs[0] == 0
    host = out.cpu().numpy().tobytes()
    assert host[total:] == b"\xa5" * 4096                             # nothing written past the files
    return 0, [host[offs[p]:offs[p + 1]] for p in range(P)], rows, nbytes


def cg_mod():
    from citus_b200 import columnar
    return columnar


def _check_files(index, cols, lens, P, binary, nulls=None, gen_empty=False):
    rc, files, rows, nbytes = _files(index, cols, lens, P, binary, nulls, gen_empty)
    assert rc == 0, _err()
    want = pr.copy_files(index, cols, lens, P, binary, nulls=nulls, generate_empty_results=gen_empty)
    assert np.array_equal(rows, np.bincount(np.asarray(index, np.int64), minlength=P))
    assert [len(w) for w in want] == nbytes.tolist()
    for p in range(P):
        assert files[p] == want[p], (p, files[p][:80], want[p][:80])


def _decimal_edges():
    v = [0, pr.INT64_MIN, pr.INT64_MAX, pr.INT64_MIN + 1, pr.INT64_MAX - 1]
    for k in range(19):
        for x in (10 ** k - 1, 10 ** k, 10 ** k + 1):
            v += [x, -x]
    return np.array(v, np.int64)


@pytest.mark.parametrize("binary", [False, True])
def test_copy_decimal_and_binary_edges(cg, binary):
    rng = np.random.default_rng(11)
    e = _decimal_edges()
    n = len(e) * 40
    c8 = np.tile(e, 40)
    c4 = rng.integers(pr.INT32_MIN, pr.INT32_MAX, n, endpoint=True)
    c2 = rng.integers(-32768, 32767, n, endpoint=True)
    c4[:4], c2[:4] = [pr.INT32_MIN, -1, pr.INT32_MAX, -2], [-32768, -1, 32767, -2]
    c4[4:4 + len(e[::2])] = np.clip(e[::2], pr.INT32_MIN, pr.INT32_MAX)
    cols, lens = [c8, c4, c2, c8[::-1].copy()], [8, 4, 2, 8]
    nulls = [(rng.random(n) < 0.15).astype(np.uint8) for _ in cols]
    for x in nulls:
        x[-10:] = 1                                                     # all-NULL rows
    P = 5
    index = rng.integers(0, P, n)
    _check_files(index, cols, lens, P, binary)
    _check_files(index, cols, lens, P, binary, nulls=nulls)
    _check_files(index, [c8], [8], P, binary)
    _check_files(index, [c8], [8], P, binary, nulls=[nulls[0]])


@pytest.mark.parametrize("binary", [False, True])
def test_copy_sixteen_columns_and_seventeen_refused(cg, binary):
    from citus_b200 import capi
    rng = np.random.default_rng(16)
    n, P = 3 * 4096 + 9, 33
    e = _decimal_edges()
    cols = [rng.choice(e, n) if c % 2 else rng.integers(pr.INT32_MIN, pr.INT32_MAX, n, endpoint=True) for c in range(16)]
    lens = [8 if c % 2 else 4 for c in range(16)]
    nulls = [(rng.random(n) < 0.05 * (c % 3)).astype(np.uint8) for c in range(16)]
    index = rng.integers(0, P, n)
    _check_files(index, cols, lens, P, binary, nulls=nulls)
    with pytest.raises(capi.CitusGpuError) as ex:
        cg.partition_copy_bytes(_dev(index, np.int32).data_ptr(), n, P, [_dev(cols[0]).data_ptr()] * 17, [8] * 17, binary)
    assert ex.value.code == capi.CG_EUNSUPPORTED
    d = _dev(cols[0])
    with pytest.raises(capi.CitusGpuError) as ex:
        cg.partition_copy_serialize(_dev(index, np.int32).data_ptr(), n, P, [d.data_ptr()] * 17, [8] * 17, binary, d.data_ptr(), 0)
    assert ex.value.code == capi.CG_EUNSUPPORTED


@pytest.mark.parametrize("gen_empty", [False, True])
@pytest.mark.parametrize("binary", [False, True])
@pytest.mark.parametrize("P", [1, 33, 257, 1024])
def test_copy_many_partitions(cg, P, binary, gen_empty):
    """P > 32: the per-partition layout (present[] after the 4P offsets) must fit its device buffer"""
    rng = np.random.default_rng(P * 4 + binary * 2 + gen_empty)
    n = 20_000
    index = rng.integers(0, P, n)
    if P > 1:
        index[index % 3 == 1] = 0                                      # every third partition receives nothing
    k = rng.integers(pr.INT64_MIN, pr.INT64_MAX, n, dtype=np.int64, endpoint=True)
    a = rng.integers(-32768, 32767, n, endpoint=True)
    na = (rng.random(n) < 0.1).astype(np.uint8)
    _check_files(index, [k, a], [8, 2], P, binary, nulls=[None, na], gen_empty=gen_empty)


def test_copy_five_million_rows(cg):
    """5M rows = 1221 blocks of 4096 rows: the block offset scan in one chunk of 2048 blocks; 9M rows = 2198 blocks: the
    offsets of the second chunk carry the first chunk's bytes"""
    rng = np.random.default_rng(5)
    P = 3
    for n in (5_000_000, 9_000_000):
        index = rng.integers(0, P, n)
        k = rng.integers(pr.INT64_MIN, pr.INT64_MAX, n, dtype=np.int64, endpoint=True)
        a = rng.integers(-1000, 1000, n)
        for binary in (False, True):
            _check_files(index, [k, a], [8, 4], P, binary)


@pytest.mark.parametrize("binary", [False, True])
def test_copy_output_capacity(cg, binary):
    from citus_b200 import capi
    rng = np.random.default_rng(12)
    n, P = 10_000, 40
    index = rng.integers(0, P, n)
    cols = [rng.integers(-10 ** 12, 10 ** 12, n)]
    rc, files, _, _ = _files(index, cols, [8], P, binary, capacity_delta=0)
    assert rc == 0 and files == pr.copy_files(index, cols, [8], P, binary)
    rc, files, _, _ = _files(index, cols, [8], P, binary, capacity_delta=-1)
    assert rc == capi.CG_EINVAL and files is None
