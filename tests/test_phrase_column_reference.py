"""The sorted scan, facet, aggregate and match-scan reference of phrase queries (tests/phrase_column_reference.py) on the
CPU: hand-written answers on a six-doc segment, a one-slot phrase equal to the flat single-term references, and the
count invariants against phrase_reference.count. No GPU needed."""
import numpy as np

import agg_reference as ar
import facet_reference as fr
import phrase_column_reference as pc
import phrase_reference as pr
import sort_reference as sr

A, B, C = 0, 1, 2
# docs 1..6; "a b" matches docs 1, 2, 3 (twice) and 6; "a _ b" (rel 0, 2) matches doc 5 only
DOCS = [[A, B, C], [B, A, B], [A, B, A, B], [C, C], [A, C, B], [A, B]]
VALS = np.array([30, 10, 20, 99, 5, 40], np.int64)   # row = doc - 1
VALID = np.array([True, False, True, True, True, True])
COLS = [(VALS, VALID)]


def _m(phrase=(A, B), rel=None, **kw):
    return pc.matches([DOCS], list(phrase), rel, **kw)


def test_hand_written_matches():
    (ds, fs), = _m()
    assert ds.tolist() == [1, 2, 3, 6] and fs.tolist() == [1, 1, 2, 1]
    (ds, fs), = _m(rel=[0, 2])
    assert ds.tolist() == [5] and fs.tolist() == [1]


def test_hand_written_sort():
    h = pc.sorted_hits(_m(), COLS)
    assert h["docs"].tolist() == [3, 1, 6, 2] and h["values"].tolist() == [20, 30, 40, 0]
    assert h["nulls"].tolist() == [False, False, False, True]
    h = pc.sorted_hits(_m(), COLS, descending=True, nulls_first=True, k=2)
    assert h["docs"].tolist() == [2, 6]
    h = pc.sorted_hits(_m(deleted=[[3]], masks=[VALS != 40]), COLS)
    assert h["docs"].tolist() == [1, 2]                                   # doc 3 deleted, doc 6 filtered out
    h = pc.sorted_hits(_m(excl=[C]), COLS)
    assert h["docs"].tolist() == [3, 6, 2]                                # doc 1 holds the excluded c


def test_hand_written_facets():
    counts, nulls = pc.facet_counts(_m(), [(VALS // 10, VALID)], 0, 5)
    assert counts.tolist() == [0, 0, 1, 1, 1] and nulls == 1


def test_hand_written_aggregates():
    cells, null_cell = pc.aggregate(_m(), None, COLS)
    assert cells[0]["count"] == 4 and cells[0]["count_value"] == 3
    assert cells[0]["sum"] == 90 and cells[0]["min"] == 20 and cells[0]["max"] == 40
    assert null_cell["count"] == 0
    cells, null_cell = pc.aggregate(_m(), [(VALS // 10, VALID)], COLS, 2, 3)
    assert [c["count"] for c in cells] == [1, 1, 1] and [c["sum"] for c in cells] == [20, 30, 40]
    assert null_cell["count"] == 1 and null_cell["count_value"] == 0


def test_hand_written_scan():
    two = [DOCS, [[C, A, B], [B, B]]]                                     # a second segment: doc 1 matches
    m = pc.matches(two, [A, B])
    (segs, docs, scores), total = pc.scan(m)
    assert total == 5 and segs.tolist() == [0, 0, 0, 0, 1] and docs.tolist() == [1, 2, 3, 6, 1]
    assert not scores.any()
    (segs, docs, _), total = pc.scan(m, offset=3, limit=10)
    assert total == 5 and segs.tolist() == [0, 1] and docs.tolist() == [6, 1]
    (segs, docs, _), total = pc.scan(m, offset=5, limit=10)
    assert total == 5 and len(docs) == 0
    c = (np.float32(2.2), np.float32(0.3), np.float32(0.45))              # c0, norm_const, norm_length * (1/avgdl)
    norms = [np.array([len(d) for d in s], np.uint32) for s in two]
    (segs, docs, scores), _ = pc.scan(m, norms, c, limit=4)
    want = [pr.score(f, n, *c) for f, n in ((1, 3), (1, 3), (2, 4), (1, 2))]
    assert scores.view(np.uint32).tolist() == np.array(want, np.float32).view(np.uint32).tolist()
    assert scores[2] > scores[1]                                          # phrase frequency 2 beats 1 at a similar length


def _random_corpus(seed, n_segs=3, n=400, vocab=5):
    rng = np.random.default_rng(seed)
    segs, cols = [], []
    for _ in range(n_segs):
        segs.append([rng.integers(0, vocab, int(rng.integers(1, 12))).tolist() for _ in range(n)])
        cols.append((rng.integers(-20, 20, n).astype(np.int64), rng.random(n) < 0.8))
    return segs, cols


def test_one_slot_equals_flat_references():
    segs, cols = _random_corpus(3)
    post = [pr.postings(s, 5) for s in segs]
    for t in range(5):
        m = pc.matches(segs, [t])
        lists = [[p[t][0]] for p in post]
        for desc, nf in ((False, False), (True, True)):
            got = pc.sorted_hits(m, cols, desc, nf, k=100)
            want = sr.sorted_hits(lists, "AND", [0], cols, desc, nf, k=100)
            for f in ("docs", "segs", "values", "nulls"):
                assert np.array_equal(got[f], want[f]), (t, f)
        assert [x.tolist() for x in pc.facet_counts(m, cols, -20, 40)[:1]] == \
               [x.tolist() for x in fr.facet_counts(lists, "AND", [0], cols, -20, 40)[:1]]
        assert pc.aggregate(m, cols, cols, -20, 40) == ar.aggregate(lists, "AND", [0], cols, cols, -20, 40)


def test_count_invariants():
    segs, cols = _random_corpus(4)
    deleted = [np.arange(1, 400, 7, dtype=np.uint32), None, None]
    for phrase, rel, excl in (([0, 1], None, ()), ([2, 2], None, (4,)), ([1, 3], [0, 2], ()), ([0], None, (1,))):
        m = pc.matches(segs, phrase, rel, excl, deleted)
        n = pr.count(segs, phrase, rel, excl, deleted)
        assert sum(len(ds) for ds, _ in m) == n
        counts, nulls = pc.facet_counts(m, cols, -20, 40)
        assert int(counts.sum()) + nulls == n
        cells, null_cell = pc.aggregate(m, None, cols)
        assert cells[0]["count"] == n
        assert len(pc.sorted_hits(m, cols)["docs"]) == n
        assert pc.scan(m)[1] == n
