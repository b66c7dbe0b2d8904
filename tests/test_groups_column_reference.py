"""The sort and facet reference of OR-group and min-match queries (tests/groups_column_reference.py) on the CPU:
hand-written answers for an OR-group query and a `2 of 3` query, the degenerate forms equal to the flat OR / AND
references (sort_reference, facet_reference), and the count invariants against min_match_reference.count."""
import numpy as np

import count_reference as cr
import facet_reference as fr
import groups_column_reference as gr
import min_match_reference as mr
import sort_reference as sr

# docs 1..10; row = doc - 1
LISTS = [np.array([1, 2, 3, 5, 8], np.uint32), np.array([2, 3, 4, 8, 9], np.uint32), np.array([3, 4, 5, 9, 10], np.uint32),
         np.array([1, 4, 8, 10], np.uint32)]
VALS = np.array([50, 20, 70, 10, 40, 90, 30, 60, 80, 0], np.int64)
VALID = np.ones(10, bool)
VALID[8] = False                                                      # doc 9 is NULL
COLS = [(VALS, VALID)]
NESTED = [[0], [1, 2]]                                                # t0 & (t1 | t2): docs 2, 3, 5, 8
TWO_OF_THREE = [[1, 2, 3]]                                            # 2 of (t1 | t2 | t3): docs 3, 4, 8, 9, 10


def test_hand_written_sort():
    h = gr.sorted_hits([LISTS], NESTED, COLS)
    assert h["docs"].tolist() == [2, 5, 8, 3] and h["values"].tolist() == [20, 40, 60, 70]
    h = gr.sorted_hits([LISTS], TWO_OF_THREE, COLS, mins=[2])
    assert h["docs"].tolist() == [10, 4, 8, 3, 9] and h["nulls"].tolist() == [False] * 4 + [True]
    h = gr.sorted_hits([LISTS], TWO_OF_THREE, COLS, descending=True, nulls_first=True, k=3, mins=[2])
    assert h["docs"].tolist() == [9, 3, 8] and h["values"].tolist() == [0, 70, 60]
    h = gr.sorted_hits([LISTS], TWO_OF_THREE, COLS, deleted=[[10]], masks=[VALS != 60], mins=[2])
    assert h["docs"].tolist() == [4, 3, 9]                             # doc 10 deleted, doc 8 filtered out


def test_hand_written_facets():
    keys = [(VALS // 20, VALID)]
    assert gr.facet_dict([LISTS], NESTED, keys) == {1: 1, 2: 1, 3: 2}
    assert gr.facet_dict([LISTS], TWO_OF_THREE, keys, mins=[2]) == {0: 2, 3: 2, None: 1}
    counts, nulls = gr.facet_counts([LISTS], TWO_OF_THREE, keys, 0, 4, excl=[3], mins=[2])
    assert counts.tolist() == [0, 0, 0, 1] and nulls == 1                # !t3 removes docs 4, 8 and 10: 3 and 9 (NULL) stay


def _random_segments(seed, n_segs=3, n=3000, n_terms=8):
    rng = np.random.default_rng(seed)
    seg_lists, cols = [], []
    for _ in range(n_segs):
        seg_lists.append([np.unique(rng.integers(1, n + 1, int(rng.integers(0, n)))).astype(np.uint32) for _ in range(n_terms)])
        cols.append((rng.integers(-50, 50, n).astype(np.int64), rng.random(n) < 0.8))
    return seg_lists, cols


def test_degenerate_forms_equal_flat_references():
    seg_lists, cols = _random_segments(1)
    masks = [cr.pred_mask(v, m, "GT", -40) for v, m in cols]
    deleted = [np.arange(1, 3000, 11, dtype=np.uint32), None, None]
    for terms, excl in (([0, 3, 5], []), ([1, 2], [4]), ([6], [0, 7])):
        for desc, nf in ((False, False), (True, True)):
            kw = dict(descending=desc, nulls_first=nf, k=500, excl=excl, deleted=deleted, masks=masks)
            flat_or = sr.sorted_hits(seg_lists, "OR", terms, cols, **kw)
            one_group = gr.sorted_hits(seg_lists, [terms], cols, **kw)
            flat_and = sr.sorted_hits(seg_lists, "AND", terms, cols, **kw)
            singles = gr.sorted_hits(seg_lists, [[t] for t in terms], cols, **kw)
            all_of = gr.sorted_hits(seg_lists, [terms], cols, mins=[len(terms)], **kw)
            for key in ("docs", "segs", "values", "nulls"):
                assert np.array_equal(flat_or[key], one_group[key])
                assert np.array_equal(flat_and[key], singles[key]) and np.array_equal(flat_and[key], all_of[key])
        kw = dict(excl=excl, deleted=deleted, masks=masks)
        assert fr.facet_dict(seg_lists, "OR", terms, cols, **kw) == gr.facet_dict(seg_lists, [terms], cols, **kw)
        assert fr.facet_dict(seg_lists, "AND", terms, cols, **kw) == gr.facet_dict(seg_lists, [[t] for t in terms], cols, **kw)


def test_count_invariants():
    seg_lists, cols = _random_segments(2)
    masks = [cr.pred_mask(v, m, "GT", -30) for v, m in cols]
    deleted = [np.arange(1, 3000, 7, dtype=np.uint32), None, np.arange(5, 50, dtype=np.uint32)]
    for groups, mins, excl in (([[0, 1, 2]], [2], []), ([[3], [4, 5, 6]], [1, 2], [7]), ([[0, 1], [2, 3, 4]], [1, 3], [])):
        count = mr.count(seg_lists, groups, excl, deleted, masks, mins=mins)
        assert count > 0
        for k in (1, count, count + 10):
            h = gr.sorted_hits(seg_lists, groups, cols, k=k, excl=excl, deleted=deleted, masks=masks, mins=mins)
            assert len(h["docs"]) == min(k, count)
        counts, nulls = gr.facet_counts(seg_lists, groups, cols, -50, 100, excl=excl, deleted=deleted, masks=masks,
                                        mins=mins)
        assert int(counts.sum()) + nulls == count
