"""The repartition reference (tests/partition_reference.py) pinned to Citus's own outputs in tests/golden/expected.json
(hash values, synthetic intervals, partition members, COPY file sizes), then to the oracle's routing on random keys,
and its uniform shortcut to its interval search at every boundary.  CPU only."""
import datetime

import numpy as np
import pytest

import partition_reference as pr


def test_hash_functions_match_postgres_outputs(expected):
    for k, v in expected["hashint4"].items():
        assert pr.hashint4(int(k)) == v
    assert pr.hashint4(123) == expected["worker_hash_123"]
    date = (datetime.date(1997, 8, 8) - datetime.date(2000, 1, 1)).days
    assert date == expected["date_1997_08_08"]
    assert pr.hashint4(date) == expected["worker_hash_date_1997_08_08"]       # date hashes like int4
    assert sorted(pr.hashint8(v) for v in expected["hashint8_inputs"]) == expected["hashint8_sorted"]
    assert pr.hashint8(2608474032) == pr.INT32_MAX
    assert pr.hashint8(963809240) == pr.INT32_MIN


def test_vectorised_hashes_equal_the_scalar_forms():
    rng = np.random.default_rng(1)
    edges = [0, 1, -1, 2, -2, pr.INT32_MIN, pr.INT32_MAX, pr.INT32_MIN + 1, pr.INT32_MAX - 1, 1 << 32, (1 << 32) - 1,
             -(1 << 32), pr.INT64_MIN, pr.INT64_MAX, pr.INT64_MIN + 1, pr.INT64_MAX - 1, 2608474032, 963809240]
    v8 = np.concatenate([np.array(edges, np.int64), rng.integers(pr.INT64_MIN, pr.INT64_MAX, 3000, dtype=np.int64, endpoint=True)])
    assert pr.hashint8_np(v8).tolist() == [pr.hashint8(int(x)) for x in v8]
    v4 = np.concatenate([np.array([e for e in edges if pr.INT32_MIN <= e <= pr.INT32_MAX], np.int64),
                         rng.integers(pr.INT32_MIN, pr.INT32_MAX, 3000, endpoint=True)])
    assert pr.hashint4_np(v4).tolist() == [pr.hashint4(int(x)) for x in v4]
    # an int8 holding an int4 value hashes like that int4, for both signs
    assert np.array_equal(pr.hashint8_np(v4), pr.hashint4_np(v4))


def test_intervals_members_and_file_sizes_match_citus(expected):
    mins, maxs = pr.synthetic_intervals(4)
    assert (mins, maxs) == (expected["squares_hash_mins"], expected["squares_hash_maxs"])
    i = np.arange(1, 11)
    idx, counts, bad = pr.route(i, None, 4, "hash", mins, maxs)
    assert bad == 0
    assert [i[idx == p].tolist() for p in range(4)] == expected["squares_hash_members"]
    # worker_partition_query_result's return rows (partitioned_intermediate_results.out): rows and COPY bytes
    files = pr.copy_files(idx, [i, i * i], [4, 4], 4, False)
    assert [[p, int(counts[p]), len(files[p])] for p in range(4)] == expected["squares_hash_text"]
    ridx, rcounts, _ = pr.route(i * i, None, 4, "range", [0, 21, 41, 61], [20, 40, 60, 100])
    files = pr.copy_files(ridx, [i, i * i], [4, 4], 4, True)
    assert [[p, int(rcounts[p]), len(files[p])] for p in range(4)] == expected["squares_range_binary"]
    i = np.arange(1, 1_000_001)
    idx, counts, _ = pr.route(i, None, 4, "hash", mins, maxs)
    files = pr.copy_files(idx, [i, 2 * i], [4, 4], 4, False)
    assert [[p, int(counts[p]), len(files[p])] for p in range(4)] == expected["doubles_hash_text"]
    ridx, rcounts, _ = pr.route(i, None, 4, "range", [0, 250001, 500001, 750001], [250000, 500000, 750000, 1000000])
    files = pr.copy_files(ridx, [i, 2 * i], [4, 4], 4, True)
    assert [[p, int(rcounts[p]), len(files[p])] for p in range(4)] == expected["doubles_range_binary"]


@pytest.mark.parametrize("P", [1, 3, 4, 7, 32, 1000])
def test_routing_equals_the_oracle(oracle, P):
    rng = np.random.default_rng(P)
    n = 20_000
    keys = rng.integers(pr.INT64_MIN, pr.INT64_MAX, n, dtype=np.int64, endpoint=True)
    keys[:100] = rng.integers(pr.INT32_MIN, pr.INT32_MAX, 100, endpoint=True)
    nulls = (rng.random(n) < 0.02).astype(np.uint8)
    mins, maxs = pr.synthetic_intervals(P)
    omins, omaxs = oracle.synthetic_intervals(P)
    assert omins.tolist() == mins and omaxs.tolist() == maxs
    for key_len in (4, 8):
        k = keys.astype(np.int32).astype(np.int64) if key_len == 4 else keys
        idx, counts, bad = pr.route(k, nulls, key_len, "hash", mins, maxs)
        want_idx, want_rows = oracle.partition_rows(k, nulls, key_len, "h", omins, omaxs)
        assert bad == 0
        assert np.array_equal(idx, want_idx) and np.array_equal(counts, want_rows)


@pytest.mark.parametrize("P", [1, 2, 3, 7, 32, 255, 256, 257, 1000, 1024])
def test_uniform_shortcut_equals_the_interval_search(P):
    mins, maxs = pr.synthetic_intervals(P)
    assert mins[0] == pr.INT32_MIN and maxs[-1] == pr.INT32_MAX
    assert all(maxs[i] + 1 == mins[i + 1] for i in range(P - 1))
    near = np.array(mins + maxs, np.int64)[:, None] + np.arange(-2, 3)[None, :]
    h = np.unique(np.clip(near.ravel(), pr.INT32_MIN, pr.INT32_MAX))
    top = np.arange(pr.INT32_MIN + P * (pr.HASH_TOKEN_COUNT // P) - 2, pr.INT32_MAX + 1, dtype=np.int64)   # the widened end
    h = np.union1d(h, top)
    got = pr.uniform_index(h, P)
    assert np.array_equal(got, pr.find_interval(h, mins, maxs))
    assert [pr.uniform_index(int(x), P) for x in h[:50]] == got[:50].tolist()
    assert pr.uniform_index(pr.INT32_MAX, P) == P - 1


def test_find_interval_reports_gaps():
    mins, maxs = [-10, 0, 5], [-5, 0, 9]
    assert pr.find_interval(np.array([-11, -10, -5, -4, -1, 0, 1, 4, 5, 9, 10]), mins, maxs).tolist() == \
        [-1, 0, 0, -1, -1, 1, -1, -1, 2, 2, -1]
    idx, counts, bad = pr.route(np.array([-7, 3, 0, 8]), np.array([0, 1, 0, 0]), 8, "range", mins, maxs)
    assert idx.tolist() == [0, 0, 1, 2] and counts.tolist() == [2, 1, 1] and bad == 0
    idx, counts, bad = pr.route(np.array([-7, 3, 1 << 40]), None, 8, "range", mins, maxs)
    assert idx.tolist() == [0, -1, -1] and bad == 2


def test_stable_scatter_keeps_input_order():
    index = np.array([2, 0, 2, 1, 0, 2])
    cols, offs = pr.stable_scatter(index, [np.arange(6)], 4)
    assert cols[0].tolist() == [1, 4, 3, 0, 2, 5] and offs.tolist() == [0, 2, 3, 6, 6]
    cols, offs = pr.stable_scatter(index, [np.arange(6)], 4, order=[3, 2, 0, 1])
    assert cols[0].tolist() == [0, 2, 5, 3, 1, 4] and offs.tolist() == [0, 3, 3, 4, 6]


def _decimal_edges():
    v = [0, pr.INT64_MIN, pr.INT64_MAX, pr.INT64_MIN + 1]
    for k in range(19):
        for x in (10 ** k - 1, 10 ** k, 10 ** k + 1):
            v += [x, -x]
    return np.array(v, np.int64)


@pytest.mark.parametrize("binary", [False, True])
def test_vectorised_copy_files_equal_the_row_at_a_time_files(binary):
    rng = np.random.default_rng(3)
    e = _decimal_edges()
    n = len(e)
    i2 = rng.integers(-32768, 32768, n)
    i4 = rng.integers(pr.INT32_MIN, pr.INT32_MAX, n, endpoint=True)
    i2[:2], i4[:2] = [-32768, 32767], [pr.INT32_MIN, pr.INT32_MAX]
    cols, lens = [e, i2, i4, e[::-1].copy()], [8, 2, 4, 8]
    nulls = [(rng.random(n) < 0.2).astype(np.uint8) for _ in cols]
    nulls[1][5] = nulls[2][5] = nulls[0][5] = nulls[3][5] = 1            # an all-NULL row
    P = 7
    index = rng.integers(0, P - 2, n)                                    # the last two partitions receive nothing
    for gen_empty in (False, True):
        for nl in (None, nulls):
            got = pr.copy_files(index, cols, lens, P, binary, nulls=nl, generate_empty_results=gen_empty)
            want = pr.copy_files_rowwise(index, cols, lens, P, binary, nulls=nl, generate_empty_results=gen_empty)
            assert got == want
    assert pr.copy_files([], [np.zeros(0, np.int64)], [8], 2, True, generate_empty_results=True) == \
        [pr.COPY_HEADER + pr.COPY_TRAILER] * 2
    assert pr.copy_files([], [np.zeros(0, np.int64)], [8], 2, True) == [b"", b""]
