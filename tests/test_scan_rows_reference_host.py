"""tests/scan_rows_reference.py's vectorised WHERE mask against tests/reference.py's tree_value, row by row, on random
trees over every atom kind -- range operators, IN / NOT IN with NULL elements, IS [NOT] NULL, column atoms across
numeric scales and in float order -- with NULLs, NaN, +-0.0, +-inf and the int64 edges in the data and the constants."""
import math

import numpy as np
import pytest

import reference as ref
import scan_rows_reference as srr

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
OPS = ("<", "<=", "=", ">=", ">", "<>")


class Col:
    def __init__(self, index):
        self.index = index

    def __repr__(self):
        return f"Col({self.index})"


# attribute -> (class, numeric scale): int, int, numeric(s=2), numeric(s=4), float, float
CLASSES = [("int", 0), ("int", 0), ("int", 2), ("int", 4), ("float", 0), ("float", 0)]
FLOAT_COLS = (4, 5)
SCALES = {2: 2, 3: 4}


def columns(rng, n):
    ints = np.array([INT64_MIN, INT64_MIN + 1, -1, 0, 1, INT64_MAX - 1, INT64_MAX], np.int64)
    vals = [rng.integers(-5, 6, n).astype(np.int64), rng.integers(-5, 6, n).astype(np.int64),
            rng.integers(-500, 501, n).astype(np.int64), rng.integers(-50000, 50001, n).astype(np.int64),
            rng.choice([-2.0, -1.5, -0.0, 0.0, 1.5, 2.0], n), rng.choice([-2.0, -0.0, 0.0, 2.0], n)]
    edge = rng.random(n) < 0.1
    vals[1][edge] = ints[rng.integers(0, len(ints), int(edge.sum()))]
    for c in (4, 5):
        sp = rng.random(n) < 0.15
        vals[c][sp] = np.array([math.nan, math.inf, -math.inf])[rng.integers(0, 3, int(sp.sum()))]
    nulls = [(rng.random(n) < rate).astype(np.uint8) for rate in (0.0, 0.1, 0.1, 0.05, 0.1, 0.2)]
    nulls[0] = None
    return vals, nulls


def pool(c):
    if c in FLOAT_COLS:
        return [-2.0, -1.5, -0.0, 0.0, 1.5, 2.0, math.nan, math.inf, -math.inf]
    if c == 1:
        return [INT64_MIN, INT64_MIN + 1, -1, 0, 1, INT64_MAX - 1, INT64_MAX]
    return [-500, -5, -1, 0, 1, 5, 500, 50000]


def random_atom(rng):
    c = int(rng.integers(0, len(CLASSES)))
    r = rng.random()
    p = pool(c)
    if r < 0.3:
        vals = tuple(p[int(rng.integers(0, len(p)))] for _ in range(int(rng.integers(1, 5))))
        if rng.random() < 0.3:
            vals = vals + (None,)
        return (c, "in" if rng.random() < 0.5 else "not in", vals)
    if r < 0.45:
        return (c, "is null" if rng.random() < 0.5 else "is not null")
    if r < 0.65:
        same = [o for o in range(len(CLASSES)) if CLASSES[o][0] == CLASSES[c][0]]
        return (c, OPS[int(rng.integers(0, 6))], Col(int(rng.choice(same))))
    return (c, OPS[int(rng.integers(0, 6))], p[int(rng.integers(0, len(p)))])


def random_tree(rng, max_atoms=5):
    nodes = [random_atom(rng) for _ in range(int(rng.integers(1, max_atoms + 1)))]
    while len(nodes) > 1:
        i = int(rng.integers(0, len(nodes) - 1))
        nodes[i:i + 2] = [("and" if rng.random() < 0.5 else "or", nodes[i], nodes[i + 1])]
    return nodes[0]


def row_values(vals, nulls, r):
    v = [float(col[r]) if c in FLOAT_COLS else int(col[r]) for c, col in enumerate(vals)]
    isnull = [bool(nn[r]) if nn is not None else False for nn in nulls]
    return v, isnull


@pytest.mark.parametrize("seed", range(6))
def test_mask_equals_tree_value_row_by_row(seed):
    rng = np.random.default_rng(20261019 + seed)
    n = 400
    vals, nulls = columns(rng, n)
    rows = [row_values(vals, nulls, r) for r in range(n)]
    for _ in range(40):
        tree = random_tree(rng)
        t, f = srr.tree_masks(tree, vals, nulls, FLOAT_COLS, SCALES)
        assert not np.any(t & f), tree
        for r, (v, isnull) in enumerate(rows):
            want = ref.tree_value(tree, v, isnull, FLOAT_COLS, SCALES)
            got = True if t[r] else (False if f[r] else None)
            assert got is want, (tree, r, v, isnull)


def test_atom_lists_and_empty_where():
    """an AND-list and a single atom are trees too; no WHERE keeps every row"""
    rng = np.random.default_rng(7)
    vals, nulls = columns(rng, 200)
    assert srr.where_mask(None, vals, nulls, FLOAT_COLS, SCALES).all()
    atoms = [(0, ">", -3), (1, "is not null"), (4, "<", 2.0)]
    got = srr.where_mask(atoms, vals, nulls, FLOAT_COLS, SCALES)
    for r in range(200):
        v, isnull = row_values(vals, nulls, r)
        assert got[r] == (ref.tree_value(atoms, v, isnull, FLOAT_COLS, SCALES) is True)
    one = srr.where_mask((2, "=", 5), vals, nulls, FLOAT_COLS, SCALES)
    assert np.array_equal(one, (vals[2] == 5) & (nulls[2] == 0))


def test_expected_rows_form():
    """projected rows in row order, floats as float8 bits, 0 in a NULL's value slot, repeated attributes allowed"""
    vals = [np.array([3, -1, 7, 2], np.int64), np.array([-0.0, math.nan, 1.5, 2.5])]
    nulls = [np.array([0, 1, 0, 0], np.uint8), np.array([0, 0, 1, 0], np.uint8)]
    v, nn = srr.expected_rows(vals, nulls, ("or", (0, ">", 2), (1, "<", 0.0)), [1, 0, 1], float_cols=(1,))
    assert list(v[1]) == [3, 7] and list(nn[1]) == [0, 0]
    assert list(nn[0]) == [0, 1]
    assert v[0][0] == np.array([-0.0]).view(np.int64)[0] and v[0][1] == 0
    assert np.array_equal(v[0], v[2]) and np.array_equal(nn[0], nn[2])
