"""The numpy equi-join of tests/join_agg_reference.py against a nested-loop join, on small random inputs with duplicate
keys on both sides, NULL keys, INT64_MIN keys, an empty side and no matches (no GPU)."""
import numpy as np
import pytest

import join_agg_reference as jref

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


def _side(rng, n, key_pool, ncols, null_rate):
    keys = rng.choice(key_pool, n) if n else np.zeros(0, np.int64)
    cols = [np.asarray(keys, np.int64)] + [rng.integers(INT64_MIN, INT64_MAX, n, dtype=np.int64, endpoint=True)
                                          for _ in range(ncols - 1)]
    nulls = [(rng.random(n) < null_rate).astype(np.uint8) for _ in range(ncols)]
    return cols, nulls


def _check(bc, bn, bkey, pc, pn, pkey):
    got = jref.join(bc, bn, bkey, pc, pn, pkey)
    want = jref.nested_loop_join(bc, bn, bkey, pc, pn, pkey)
    assert jref.rows_of(*got) == jref.rows_of(*want)
    return got


@pytest.mark.parametrize("seed", range(12))
def test_join_matches_nested_loop(seed):
    rng = np.random.default_rng(seed)
    pool = np.array([INT64_MIN, INT64_MAX, -1, 0, 1, 7, 7, 1 << 40], np.int64)
    nb, npr = int(rng.integers(0, 60)), int(rng.integers(0, 60))
    bc, bn = _side(rng, nb, pool, 3, 0.15)
    pc, pn = _side(rng, npr, pool[rng.permutation(len(pool))[:5]], 2, 0.15)
    bkey, pkey = 0, 0
    (cols, nulls) = _check(bc, bn, bkey, pc, pn, pkey)
    assert len(cols) == 5 and len(nulls) == 5
    # the joined keys agree and are never NULL
    if len(cols[0]):
        assert np.array_equal(cols[0], cols[3]) and not nulls[0].any() and not nulls[3].any()


def test_duplicates_on_both_sides_multiply():
    bc = [np.array([5, 5, 5, 9], np.int64), np.arange(4, dtype=np.int64)]
    pc = [np.array([5, 5, 9, 9, 9], np.int64)]
    cols, _ = _check(bc, None, 0, pc, None, 0)
    assert len(cols[0]) == 3 * 2 + 1 * 3


def test_null_keys_join_nothing_even_with_the_same_value():
    bc = [np.array([0, 0, 3], np.int64)]
    pc = [np.array([0, 3, 3], np.int64)]
    bn = [np.array([1, 0, 0], np.uint8)]
    pn = [np.array([0, 1, 0], np.uint8)]
    cols, nulls = _check(bc, bn, 0, pc, pn, 0)
    assert jref.rows_of(cols, nulls) == [(0, 0), (3, 3)]


def test_int64_min_is_an_ordinary_key():
    bc = [np.array([INT64_MIN, INT64_MIN, 1], np.int64)]
    pc = [np.array([INT64_MIN, 2], np.int64)]
    cols, _ = _check(bc, None, 0, pc, None, 0)
    assert list(cols[0]) == [INT64_MIN, INT64_MIN]


@pytest.mark.parametrize("nb,npr", [(0, 5), (5, 0), (0, 0)])
def test_an_empty_side_joins_nothing(nb, npr):
    bc = [np.arange(nb, dtype=np.int64), np.arange(nb, dtype=np.int64)]
    pc = [np.arange(npr, dtype=np.int64)]
    cols, nulls = _check(bc, None, 0, pc, None, 0)
    assert all(len(c) == 0 for c in cols) and len(cols) == 3


def test_no_matches():
    bc = [np.arange(0, 20, 2, dtype=np.int64)]
    pc = [np.arange(1, 21, 2, dtype=np.int64), np.arange(10, dtype=np.int64)]
    cols, _ = _check(bc, None, 0, pc, None, 0)
    assert len(cols[0]) == 0


def test_key_need_not_be_the_first_column():
    rng = np.random.default_rng(5)
    bc, bn = _side(rng, 40, np.arange(6), 3, 0.1)
    pc, pn = _side(rng, 30, np.arange(4, 9), 3, 0.1)
    bc[0], bc[2] = bc[2], bc[0]
    bn[0], bn[2] = bn[2], bn[0]
    bc[2] = rng.choice(np.arange(6), 40)
    pc[1] = rng.choice(np.arange(4, 9), 30)
    _check(bc, bn, 2, pc, pn, 1)


def test_exact_sum():
    a = np.array([INT64_MAX, INT64_MAX, INT64_MIN, -1, 12345], np.int64)
    assert jref.exact_sum(a) == sum(int(x) for x in a)
