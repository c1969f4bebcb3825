"""The layout of the narrow (bit-packed, frame-of-reference) images cg_shard_stage keeps next to the plain arena
(cg_narrow_plan): which columns get images, and each chunk column's width, base and stream offset.  CPU only."""
import ctypes as C

import numpy as np
import pytest

NONE = 255
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


@pytest.fixture(scope="module")
def lib():
    from citus_b200 import build
    build.build()
    from citus_b200 import capi
    return capi.lib()


def plan(lib, rows, mins, maxs, nullfree=None, candidate=None):
    """rows [ncg]; mins / maxs [ncg][ncols] -> (col_narrow, widths, bases, offs, total)"""
    mins = np.ascontiguousarray(mins, np.int64)
    maxs = np.ascontiguousarray(maxs, np.int64)
    ncg, ncols = mins.shape
    rows = np.ascontiguousarray(rows, np.uint32)
    nullfree = np.ones((ncg, ncols), np.uint8) if nullfree is None else np.ascontiguousarray(nullfree, np.uint8)
    candidate = np.ones(ncols, np.uint8) if candidate is None else np.ascontiguousarray(candidate, np.uint8)
    col = np.zeros(ncols, np.uint8)
    widths = np.zeros((ncg, ncols), np.uint8)
    bases = np.zeros((ncg, ncols), np.int64)
    offs = np.zeros((ncg, ncols), np.uint64)
    total = C.c_uint64(0)
    rc = lib.cg_narrow_plan(ncg, ncols, candidate.ctypes.data, rows.ctypes.data, nullfree.ctypes.data, mins.ctypes.data,
                            maxs.ctypes.data, col.ctypes.data, widths.ctypes.data, bases.ctypes.data, offs.ctypes.data,
                            C.byref(total))
    assert rc == 0
    return col, widths, bases, offs, total.value


def stream_bytes(rows, w):
    return ((rows + 63) // 64 * w * 8 + 15) // 16 * 16


def test_constant_chunk_has_width_zero(lib):
    col, widths, bases, offs, total = plan(lib, [10000], [[7]], [[7]])
    assert col.tolist() == [1] and widths[0, 0] == 0 and bases[0, 0] == 7 and total == 0


@pytest.mark.parametrize("span,width", [(1, 1), (99, 7), (10**6 - 1, 20), (2 * 10**9, 31), ((1 << 32) - 1, 32)])
def test_width_is_bits_of_the_span(lib, span, width):
    col, widths, bases, offs, total = plan(lib, [10000], [[-5]], [[-5 + span]])
    assert col[0] == 1 and widths[0, 0] == width and bases[0, 0] == -5
    assert total == stream_bytes(10000, width)


def test_33_bit_chunk_leaves_the_column_unpacked(lib):
    # chunk group 1 of column 0 spans 2^32: column 0 gets no image in any chunk group; column 1 is unaffected
    mins = [[0, 0], [-(1 << 31), 0], [0, 0]]
    maxs = [[100, 3], [1 << 31, 3], [100, 3]]
    col, widths, bases, offs, total = plan(lib, [10000, 10000, 10000], mins, maxs)
    assert col.tolist() == [0, 1]
    assert (widths[:, 0] == NONE).all() and (widths[:, 1] == 2).all()
    assert total == 3 * stream_bytes(10000, 2)


def test_int64_extremes(lib):
    # spans near 2^32 at both ends of int64, and a full-range column (wrapping difference) that must stay unpacked
    mins = [[I64_MIN, I64_MAX - (1 << 32) + 1, I64_MIN]]
    maxs = [[I64_MIN + (1 << 32) - 1, I64_MAX, I64_MAX]]
    col, widths, bases, offs, total = plan(lib, [5], mins, maxs)
    assert col.tolist() == [1, 1, 0]
    assert widths[0].tolist() == [32, 32, NONE]
    assert bases[0, 0] == I64_MIN and bases[0, 1] == I64_MAX - (1 << 32) + 1


def test_negative_bases(lib):
    col, widths, bases, offs, total = plan(lib, [64, 64], [[-10**9], [-1]], [[10**9], [0]])
    assert widths[:, 0].tolist() == [31, 1] and bases[:, 0].tolist() == [-10**9, -1]


def test_one_row_chunk_and_short_last_chunk_group(lib):
    rows = [10000, 10000, 3337, 1]
    mins = [[0, -7]] * 4
    maxs = [[999_999, 92]] * 4
    col, widths, bases, offs, total = plan(lib, rows, mins, maxs)
    assert (widths[:, 0] == 20).all() and (widths[:, 1] == 7).all()
    # streams back to back in (chunk group, column) order, each 16-byte aligned and covering whole 64-row blocks
    expect, off = [], 0
    for r in rows:
        for w in (20, 7):
            expect.append(off)
            off += stream_bytes(r, w)
    assert offs.reshape(-1).tolist() == expect and total == off
    assert all(o % 16 == 0 for o in expect)
    assert stream_bytes(1, 20) == 160 and stream_bytes(3337, 7) == 2976      # 53 blocks of 7 words, padded to 16 B


def test_nulls_and_non_candidates(lib):
    # chunk columns with NULLs get no image (and their min / max are not read); a non-candidate column never does
    mins = [[0, 0, 0], [0, 0, 0]]
    maxs = [[15, 15, 15], [15, 1 << 40, 15]]
    nullfree = [[1, 1, 1], [1, 0, 1]]
    col, widths, bases, offs, total = plan(lib, [100, 100], mins, maxs, nullfree=nullfree, candidate=[1, 1, 0])
    assert col.tolist() == [1, 1, 0]
    assert widths.tolist() == [[4, 4, NONE], [4, NONE, NONE]]
    assert total == 3 * stream_bytes(100, 4)
