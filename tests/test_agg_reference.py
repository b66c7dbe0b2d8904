"""Pins tests/agg_reference.py (the aggregates over a full-text query's matches) on hand-computed cases: COUNT(*) and
COUNT(value) with NULL values and NULL keys, exact integer sums at INT64_MIN / INT64_MAX, IEEE float64 sums with NaN and
infinities, MIN / MAX under the sorted scan's order (-0.0 == +0.0, NaN above +inf), all-NULL groups, keys outside the
range, and the ungrouped cell equal to the merge of the grouped ones."""
import math

import numpy as np
import pytest

import agg_reference as ar

I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1


def test_counts_and_nulls():
    # docs 1..6; doc 6 lies past both columns' rows (NULL key, NULL value)
    lists = [np.array([1, 2, 3, 5, 6], np.uint32)]
    keys = (np.array([10, 11, 10, 11, 12], np.int64), np.array([1, 1, 1, 0, 1], bool))   # row 3 (doc 4): NULL key
    vals = (np.array([5, -7, 100, 1, 9], np.int32), np.array([1, 1, 0, 1, 1], bool))     # row 2 (doc 3): NULL value
    cells, null = ar.aggregate([lists], "OR", [0], [keys], [vals], 10, 3)
    assert cells[0] == dict(count=2, count_value=1, sum=5, min=5, max=5)                # docs 1 and 3
    assert cells[1] == dict(count=1, count_value=1, sum=-7, min=-7, max=-7)             # doc 2
    assert cells[2] == dict(count=1, count_value=1, sum=9, min=9, max=9)                # doc 5
    assert null == dict(count=1, count_value=0, sum=0, min=0, max=0)                    # doc 6
    with pytest.raises(ValueError):
        ar.aggregate([lists], "OR", [0], [keys], [vals], 11, 2)


def test_int64_extremes_exact():
    n = 1000
    v = np.array([I64_MAX] * n + [I64_MIN] * (n + 3), np.int64)
    docs = [np.arange(1, len(v) + 1, dtype=np.uint32)]
    (c,), null = ar.aggregate([docs], "OR", [0], None, [(v, None)])
    assert c["sum"] == n * I64_MAX + (n + 3) * I64_MIN == -n - 3 * 2 ** 63
    assert (c["min"], c["max"], c["count"], c["count_value"]) == (I64_MIN, I64_MAX, 2 * n + 3, 2 * n + 3)
    assert null["count"] == 0
    (c,), _ = ar.aggregate([docs], "OR", [0], None, [(np.full(n, I64_MAX, np.int64), None)])
    assert c["sum"] == n * I64_MAX and c["count_value"] == n and c["count"] == 2 * n + 3   # docs past the rows: NULL


def test_float_rules():
    c = ar.cell_of([1.0, -0.0, 0.0, 2.5], True)
    assert c["sum"] == 3.5 and math.copysign(1.0, c["min"]) == 1.0 and c["min"] == 0.0 and c["max"] == 2.5
    c = ar.cell_of([-0.0], True)
    assert c["min"] == 0.0 and math.copysign(1.0, c["min"]) == 1.0
    c = ar.cell_of([1.0, math.nan, -math.inf], True)
    assert math.isnan(c["sum"]) and c["min"] == -math.inf and math.isnan(c["max"])
    c = ar.cell_of([math.inf, 3.0, -math.inf], True)
    assert math.isnan(c["sum"]) and c["min"] == -math.inf and c["max"] == math.inf
    assert ar.cell_of([math.inf, 3.0], True)["sum"] == math.inf
    assert ar.cell_of([-math.inf, 3.0], True)["sum"] == -math.inf
    c = ar.cell_of([math.nan, -math.nan], True)
    assert math.isnan(c["min"]) and math.isnan(c["max"]) and math.isnan(c["sum"])
    assert ar.cell_of([1e100, 1.0, -1e100], True)["sum"] == 1.0   # exact in the finite part
    assert ar.cell_of([], True, 4) == dict(count=4, count_value=0, sum=0.0, min=0.0, max=0.0, abs=0.0)
    assert ar.cell_of([-2.0, math.inf, 3.0], True)["abs"] == 5.0


def test_all_null_group_and_ungrouped_is_merge():
    rng = np.random.default_rng(3)
    n = 5000
    lists = [np.sort(rng.choice(np.arange(1, n + 1), 2000, replace=False)).astype(np.uint32),
             np.sort(rng.choice(np.arange(1, n + 1), 1500, replace=False)).astype(np.uint32)]
    keys = (rng.integers(0, 4, n).astype(np.int64), rng.random(n) < 0.9)
    keys[0][keys[0] == 3] = 2                                            # key 3 never occurs: an empty group
    kvalid = keys[1].copy()
    kvalid[keys[0] == 1] = True
    vvalid = rng.random(n) < 0.8
    vvalid[keys[0] == 2] = False                                         # key 2: every value NULL
    for vals in (rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64), rng.normal(size=n) * 1e6):
        col = [(vals, vvalid)]
        cells, null = ar.aggregate([lists], "OR", [0, 1], [(keys[0], kvalid)], col, 0, 4)
        (whole,), unull = ar.aggregate([lists], "OR", [0, 1], None, col)
        assert cells[2]["count"] > 0 and cells[2]["count_value"] == 0 and cells[2]["sum"] == 0
        assert cells[3] == ar.empty_cell(vals.dtype == np.float64)
        assert unull["count"] == 0
        is_f = vals.dtype == np.float64
        m = null
        for c in cells:
            m = ar.merge(m, c, is_f)
        assert m["count"] == whole["count"] and m["count_value"] == whole["count_value"]
        assert (m["min"], m["max"]) == (whole["min"], whole["max"])
        if is_f:
            assert math.isclose(m["sum"], whole["sum"], rel_tol=1e-12)
        else:
            assert m["sum"] == whole["sum"]


def test_groups_query():
    lists = [np.array([1, 2, 3, 4], np.uint32), np.array([2, 4], np.uint32), np.array([3, 4], np.uint32)]
    vals = (np.array([10, 20, 30, 40], np.int64), None)
    (c,), _ = ar.aggregate_groups([lists], [[0], [1, 2]], None, [vals])
    assert c == dict(count=3, count_value=3, sum=90, min=20, max=40)     # docs 2, 3, 4
    (c,), _ = ar.aggregate_groups([lists], [[0, 1, 2]], None, [vals], mins=[2])
    assert c == dict(count=3, count_value=3, sum=90, min=20, max=40)     # docs holding 2 of the 3 terms
