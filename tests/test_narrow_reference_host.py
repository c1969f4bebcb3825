"""tests/narrow_reference.py against first principles and against the library's layout function: pack() against a
bit-by-bit loop, and narrow_layout() against cg_narrow_plan over random relations with short chunk groups, NULLs,
non-candidate columns and columns one of whose chunks spans 2^32.  CPU only."""
import ctypes as C
import random

import numpy as np
import pytest

import narrow_reference as nr
import reference as ref

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


@pytest.fixture(scope="module")
def lib():
    from citus_b200 import build
    build.build()
    from citus_b200 import capi
    return capi.lib()


def bitwise_pack(values, width):
    """field r, bit b -> bit r * width + b of the stream, one bit at a time"""
    base = min(values)
    words = [0] * ((len(values) + 63) // 64 * width)
    for r, v in enumerate(values):
        for b in range(width):
            if ((v - base) >> b) & 1:
                pos = r * width + b
                words[pos // 64] |= 1 << (pos % 64)
    return words


def test_pack_small_example():
    base, width, words = nr.pack([5, 6, 7, 8])
    assert (base, width) == (5, 2) and words.tolist() == [0b11100100, 0]     # a 64-row block takes `width` words
    base, width, words = nr.pack([9] * 65)
    assert (base, width, words.size) == (9, 0, 0)
    # one row at each end of int64: the span is 2^64 - 1, a Python integer, not a wrapped difference
    assert nr.pack([I64_MIN, I64_MAX])[1] == 64


@pytest.mark.parametrize("seed", range(6))
def test_pack_matches_bitwise_loop(seed):
    rng = random.Random(seed)
    for _ in range(40):
        rows = rng.choice([1, 2, 31, 63, 64, 65, 127, 128, 129, rng.randint(1, 300)])
        width = rng.randint(0, 32)
        base = rng.choice([I64_MIN, I64_MAX - (1 << width) + 1, rng.randint(-(1 << 62), 1 << 62)])
        vals = [base + rng.randint(0, (1 << width) - 1) for _ in range(rows)]
        if rows > 1:
            vals[rng.randrange(rows)] = base
            vals[rng.randrange(rows)] = base + (1 << width) - 1
        b, w, words = nr.pack(vals)
        assert b == min(vals) and w == (max(vals) - min(vals)).bit_length()
        assert words.tolist() == bitwise_pack(vals, w)
        # rows past `rows` are not part of the stream
        assert nr.pack(vals + [base], rows)[2].tolist() == words.tolist()


def lib_plan(lib, groups, staged, cols, nulls, candidate):
    ncg, ns = len(groups), len(staged)
    rows = np.array([n for _, n in groups], np.uint32)
    cand = np.array([candidate[a] for a in staged], np.uint8)
    nullfree = np.zeros((ncg, ns), np.uint8)
    mins = np.zeros((ncg, ns), np.int64)
    maxs = np.zeros((ncg, ns), np.int64)
    for g, (first, n) in enumerate(groups):
        for j, a in enumerate(staged):
            v = cols[a][first:first + n]
            nm = None if nulls[a] is None else nulls[a][first:first + n]
            vv = v if nm is None else v[nm == 0]
            nullfree[g, j] = vv.size == n
            if vv.size:
                mins[g, j], maxs[g, j] = vv.min(), vv.max()
    col = np.zeros(ns, np.uint8)
    widths = np.zeros((ncg, ns), np.uint8)
    bases = np.zeros((ncg, ns), np.int64)
    offs = np.zeros((ncg, ns), np.uint64)
    total = C.c_uint64(0)
    rc = lib.cg_narrow_plan(ncg, ns, cand.ctypes.data, rows.ctypes.data, nullfree.ctypes.data, mins.ctypes.data,
                            maxs.ctypes.data, col.ctypes.data, widths.ctypes.data, bases.ctypes.data, offs.ctypes.data,
                            C.byref(total))
    assert rc == 0
    return col, widths, bases, offs, total.value


@pytest.mark.parametrize("seed", range(8))
def test_layout_matches_cg_narrow_plan(lib, seed):
    rng = np.random.default_rng(seed)
    nrows = int(rng.integers(1, 700))
    natts = int(rng.integers(1, 7))
    cols, nulls = [], []
    for a in range(natts):
        w = int(rng.integers(0, 34))
        base = int(rng.integers(-(1 << 62), 1 << 62)) if a % 3 else (I64_MIN if a % 2 else I64_MAX - (1 << 33))
        cols.append(base + rng.integers(0, 1 << w, nrows, dtype=np.uint64).astype(np.int64))
        nulls.append((rng.random(nrows) < 0.01).astype(np.uint8) if rng.random() < 0.3 else None)
    candidate = [bool(rng.random() < 0.85) for _ in range(natts)]
    layout = ref.chunk_layout(nrows, int(rng.integers(1, 400)), int(rng.choice([1, 63, 64, 65, 100, 128])))
    groups = [g for s in layout for g in s]
    staged = list(rng.permutation(natts)[: int(rng.integers(1, natts + 1))])
    want = nr.narrow_layout(cols, nulls, layout, staged, candidate)
    col, widths, bases, offs, total = lib_plan(lib, groups, staged, cols, nulls, candidate)
    for g in range(len(groups)):
        for j, a in enumerate(staged):
            im = want.image[(g, a)]
            if im is None:
                # no image: either the column has none, or there are none at all in the shard (nothing was a candidate
                # NULL-free chunk column), in which case the plan's widths are NONE as well
                assert widths[g, j] == nr.NONE or not want.any_images
                continue
            assert (int(bases[g, j]), int(widths[g, j]), int(offs[g, j])) == (im[0], im[1], want.offs[(g, a)])
    if want.any_images:
        assert total == want.total
        assert [bool(c) for c in col] == [want.col_narrow[a] for a in staged]
        assert want.narrow_bytes == total + len(groups) * len(staged) * nr.DEVPACKCOL_BYTES
    else:
        assert want.narrow_bytes == 0


def test_layout_edge_cases(lib):
    # a 2^32 span in one chunk group leaves the whole column without images; a column whose only NULL-free chunk
    # groups are narrow keeps them; constants have width 0 and take no stream bytes
    n = 200
    wide = np.arange(n, dtype=np.int64)
    wide[70] = wide[64] + (1 << 32)
    withnull = np.arange(n, dtype=np.int64) * 3
    nulls = [None, np.zeros(n, np.uint8), None]
    nulls[1][5] = 1
    const = np.full(n, -7, np.int64)
    layout = ref.chunk_layout(n, n, 64)
    lay = nr.narrow_layout([wide, withnull, const], nulls, layout, [0, 1, 2])
    assert lay.col_narrow == {0: False, 1: True, 2: True}
    assert [lay.image[(g, 1)] for g in range(4)] == [None, (192, 8), (384, 8), (576, 5)]
    assert all(lay.image[(g, 2)] == (-7, 0) for g in range(4))
    assert lay.total == 64 + 64 + 48                # two 8-word blocks, and 5 words padded to 16 bytes
    col, widths, bases, offs, total = lib_plan(lib, [g for s in layout for g in s], [0, 1, 2], [wide, withnull, const], nulls,
                                               [True] * 3)
    assert col.tolist() == [0, 1, 1] and total == lay.total
    assert lay.scan_bytes([1, 2], [True] * 4, narrow=True) == (lay.plain_bytes(0, 1) + lay.plain_bytes(0, 2)) + 2 * 64 + 5 * 8
