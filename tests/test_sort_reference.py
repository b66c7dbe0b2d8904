"""Pins tests/sort_reference.py, the NumPy statement of the sorted scan, to hand-written answers: ties across three
segments, NULLs first and last in both directions, NaN of both signs, +-0.0 and +-inf, INT64_MIN / INT64_MAX and
negative int32 values, docs past the column's rows, deleted docs and a filter mask. The full sorted list has as many
entries as count_reference.count."""
import numpy as np

import count_reference as cr
import sort_reference as sr

I64 = np.iinfo(np.int64)


def run(seg_lists, pos, columns, desc, nf, kind="OR", **kw):
    h = sr.sorted_hits(seg_lists, kind, pos, columns, desc, nf, **kw)
    return list(zip(h["segs"].tolist(), h["docs"].tolist())), h


def test_ties_across_three_segments():
    seg_lists = [[np.array([1, 2, 3], np.uint32)], [np.array([1, 2], np.uint32)], [np.array([2, 4], np.uint32)]]
    cols = [(np.array([5, 7, 5], np.int64), None), (np.array([7, 5], np.int64), None), (np.array([0, 5, 0, 7], np.int64), None)]
    order, h = run(seg_lists, [0], cols, False, False)
    assert order == [(0, 1), (0, 3), (1, 2), (2, 2), (0, 2), (1, 1), (2, 4)]
    assert h["values"].tolist() == [5, 5, 5, 5, 7, 7, 7]
    order, _ = run(seg_lists, [0], cols, True, False)
    assert order == [(0, 2), (1, 1), (2, 4), (0, 1), (0, 3), (1, 2), (2, 2)]
    order, _ = run(seg_lists, [0], cols, True, False, k=2)
    assert order == [(0, 2), (1, 1)]


def test_nulls_first_and_last_both_directions():
    lists = [np.arange(1, 7, dtype=np.uint32)]
    vals = np.array([3, 0, 1, 0, 2, 9], np.int64)
    valid = np.array([1, 0, 1, 0, 1, 1], bool)
    cols = [(vals, valid)]
    want = {(False, False): [3, 5, 1, 6, 2, 4], (False, True): [2, 4, 3, 5, 1, 6],
            (True, False): [6, 1, 5, 3, 2, 4], (True, True): [2, 4, 6, 1, 5, 3]}
    for (desc, nf), docs in want.items():
        order, h = run([lists], [0], cols, desc, nf)
        assert [d for _, d in order] == docs, (desc, nf)
        assert h["nulls"].tolist() == [d in (2, 4) for d in docs]
        assert all(v == 0 for v, n in zip(h["values"].tolist(), h["nulls"].tolist()) if n)


def test_float_specials():
    nan_pos = np.array([0x7FF8000000000001], np.uint64).view(np.float64)[0]
    nan_neg = np.array([0xFFF8000000000000], np.uint64).view(np.float64)[0]
    vals = np.array([nan_neg, 1.0, -0.0, np.inf, 0.0, -np.inf, nan_pos, -2.5], np.float64)
    lists = [np.arange(1, 9, dtype=np.uint32)]
    order, h = run([lists], [0], [(vals, None)], False, False)
    assert [d for _, d in order] == [6, 8, 3, 5, 2, 4, 1, 7]     # -inf, -2.5, -0.0 = +0.0 (by doc), 1, +inf, NaN = NaN
    assert h["values"].view(np.uint64).tolist() == vals[np.array([6, 8, 3, 5, 2, 4, 1, 7]) - 1].view(np.uint64).tolist()
    order, _ = run([lists], [0], [(vals, None)], True, False)
    assert [d for _, d in order] == [1, 7, 4, 2, 3, 5, 8, 6]     # NaNs first under DESC, ties still by doc


def test_integer_extremes():
    vals = np.array([I64.max, -1, I64.min, 0, I64.min], np.int64)
    lists = [np.arange(1, 6, dtype=np.uint32)]
    order, h = run([lists], [0], [(vals, None)], False, False)
    assert [d for _, d in order] == [3, 5, 2, 4, 1]
    assert h["values"].tolist() == [I64.min, I64.min, -1, 0, I64.max]
    v32 = np.array([-7, 3, -2147483648, 2147483647], np.int32)
    order, h = run([[np.arange(1, 5, dtype=np.uint32)]], [0], [(v32, None)], True, False)
    assert [d for _, d in order] == [4, 2, 1, 3]
    assert h["values"].dtype == np.int32 and h["values"].tolist() == [2147483647, 3, -7, -2147483648]


def test_docs_past_the_rows_are_null():
    lists = [np.array([1, 2, 5, 9], np.uint32)]
    cols = [(np.array([4, 2, 8], np.int64), None)]                 # rows 0..2: docs 5 and 9 lie past the column
    order, h = run([lists], [0], cols, False, False)
    assert [d for _, d in order] == [2, 1, 5, 9] and h["nulls"].tolist() == [False, False, True, True]
    order, _ = run([lists], [0], cols, False, True)
    assert [d for _, d in order] == [5, 9, 2, 1]


def test_deleted_docs_and_filter_mask():
    lists = [np.array([1, 2, 3, 4, 5, 6], np.uint32), np.array([2, 4, 6], np.uint32)]
    vals = np.array([6, 5, 4, 3, 2, 1], np.int64)
    mask = np.array([1, 1, 1, 1, 0, 1], bool)                      # doc 5 fails the filter
    order, _ = run([lists], [0, 1], [(vals, None)], False, False, kind="AND", deleted=[np.array([4], np.uint32)],
                   masks=[mask])
    assert [d for _, d in order] == [6, 2]
    order, _ = run([lists], [0], [(vals, None)], False, False, excl=[1], deleted=[np.array([3], np.uint32)], masks=[mask])
    assert [d for _, d in order] == [1]


def test_full_list_has_count_entries():
    rng = np.random.default_rng(4)
    seg_lists, cols = [], []
    for n in (500, 800, 300):
        seg_lists.append([np.unique(rng.integers(1, n + 1, m)).astype(np.uint32) for m in (200, 120, 60)])
        cols.append((rng.integers(-5, 5, n - 30).astype(np.int64), rng.random(n - 30) < 0.8))
    for kind in ("OR", "AND"):
        for desc in (False, True):
            h = sr.sorted_hits(seg_lists, kind, [0, 1], cols, desc, True, excl=[2])
            assert len(h["docs"]) == cr.count(seg_lists, kind, [0, 1], [2])
