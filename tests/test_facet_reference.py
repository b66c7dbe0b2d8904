"""The NumPy statement of the facet counts (tests/facet_reference.py) against hand-written answers: NULL keys (NULL rows
and docs past the column), deleted docs, exclusions, a filter on the key column, two segments, the out-of-range error,
and the reference's faceted-search cookbook answers (`products_facets`)."""
import json
import os

import numpy as np
import pytest

import count_reference as cr
import facet_reference as fr

HERE = os.path.dirname(os.path.abspath(__file__))

# one segment of 10 docs; term 0: docs 1..6, term 1: docs 4..9, term 2: docs 2, 5, 8
LISTS = [np.arange(1, 7, dtype=np.uint32), np.arange(4, 10, dtype=np.uint32), np.array([2, 5, 8], np.uint32)]
# keys by row (doc - 1); rows 2 and 6 NULL; the column has 8 rows, so docs 9 and 10 have a NULL key
VALS = np.array([-1, 3, 7, 3, 3, -1, 0, 7], np.int64)
VALID = np.array([1, 1, 0, 1, 1, 1, 0, 1], bool)


def test_or_and_with_nulls():
    c, n = fr.facet_counts([LISTS], "OR", [0, 1], [(VALS, VALID)], -1, 9)
    # docs 1..9: keys -1, 3, NULL, 3, 3, -1, NULL, 7, NULL (past the column)
    assert c.tolist() == [2, 0, 0, 0, 3, 0, 0, 0, 1] and n == 3
    c, n = fr.facet_counts([LISTS], "AND", [0, 1], [(VALS, VALID)], -1, 9)
    # docs 4, 5, 6
    assert c.tolist() == [1, 0, 0, 0, 2, 0, 0, 0, 0] and n == 0
    assert fr.facet_dict([LISTS], "OR", [0, 1], [(VALS, VALID)]) == {-1: 2, 3: 3, 7: 1, None: 3}


def test_deleted_exclusions_and_filter_on_key():
    c, n = fr.facet_counts([LISTS], "OR", [0, 1], [(VALS, VALID)], -1, 9, excl=[2], deleted=[np.array([1, 9], np.uint32)])
    # docs 3, 4, 6, 7 (1 and 9 deleted, 2, 5 and 8 excluded): NULL, 3, -1, NULL
    assert c.tolist() == [1, 0, 0, 0, 1, 0, 0, 0, 0] and n == 2
    m = np.zeros(10, bool)
    m[:8] = cr.pred_mask(VALS, VALID, "GE", 3)      # the filter's column is the key column; rows past it never pass
    c, n = fr.facet_counts([LISTS], "OR", [0, 1], [(VALS, VALID)], 3, 5, masks=[m])
    assert c.tolist() == [3, 0, 0, 0, 1] and n == 0
    m[:8] = cr.pred_mask(VALS, VALID, "IS_NULL")
    c, n = fr.facet_counts([LISTS], "OR", [0, 1], [(VALS, VALID)], 0, 1, masks=[m])
    assert c.tolist() == [0] and n == 2


def test_two_segments_and_sum_invariant():
    lists2 = [np.array([1, 2], np.uint32), np.array([2], np.uint32)]
    cols = [(VALS, VALID), (np.array([5, 3], np.int32), None)]
    c, n = fr.facet_counts([LISTS, lists2], "OR", [0, 1], cols, -1, 9)
    assert c.tolist() == [2, 0, 0, 0, 4, 0, 1, 0, 1] and n == 3
    assert int(c.sum()) + n == cr.count([LISTS, lists2], "OR", [0, 1])


def test_extreme_range_and_out_of_range():
    top = np.iinfo(np.int64).max
    vals = np.array([top, top - 1, top], np.int64)
    c, n = fr.facet_counts([[np.array([1, 2, 3], np.uint32)]], "OR", [0], [(vals, None)], top - 1, 2)
    assert c.tolist() == [1, 2] and n == 0
    with pytest.raises(ValueError):
        fr.facet_counts([LISTS], "OR", [0, 1], [(VALS, VALID)], 0, 8)       # key -1 below the range
    with pytest.raises(ValueError):
        fr.facet_counts([LISTS], "OR", [0, 1], [(VALS, VALID)], -1, 8)      # key 7 above it


def products_segment(g):
    """The cookbook's 8 products as one segment: term 0 is held by every doc, so its matches are all rows."""
    return [np.arange(1, 9, dtype=np.uint32)], {f: np.asarray(g["rows"][f], np.int64) for f in ("category", "brand", "band")}


def test_products_facets():
    with open(os.path.join(HERE, "golden", "groupby_goldens.json")) as f:
        g = json.load(f)["products_facets"]
    lists, cols = products_segment(g)
    for f in ("category", "brand", "band"):
        got = fr.facet_dict([lists], "OR", [0], [(cols[f], None)])
        names = g[f + "_names"]
        assert {names[k]: v for k, v in got.items()} == g["expect_" + f]
