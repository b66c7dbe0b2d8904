"""The reference for OR groups with a minimum match count (`2 of (a | b | c) & d`, tests/min_match_reference.py):
hand-written answers on tiny lists, agreement of m = 1 with the plain groups statement (tests/groups_reference.py) and
of m = s with the AND, and the reference's top-k against the NumPy statement (docs of the flat OR that every group holds at least m_g times, scored as
the flat OR scores them). No GPU needed."""
import numpy as np
import pytest

import count_reference as cr
import groups_reference as gr
import min_match_reference as mr
import orc

u = lambda *v: np.array(v, np.uint32)
TINY = [u(1, 2, 3, 4), u(2, 3, 5), u(3, 4, 5, 6), u(1, 6, 7), u(9)]


@pytest.mark.parametrize("groups,mins,excl,want", [
    ([[0, 1, 2]], [2], [], [2, 3, 4, 5]),          # docs in at least two of {1,2,3,4}, {2,3,5}, {3,4,5,6}
    ([[0, 1, 2]], [3], [], [3]),                   # all three: the AND
    ([[0, 1, 2]], [1], [], [1, 2, 3, 4, 5, 6]),    # one: the OR
    ([[0, 1, 2, 3]], [3], [], [3]),
    ([[0, 1, 2, 3]], [2], [], [1, 2, 3, 4, 5, 6]),
    ([[0, 1, 2]], [2], [1], [4]),                  # minus the docs of {2,3,5}
    ([[3], [0, 1, 2]], [1, 2], [], []),            # {1,6,7} & 2 of ...: no doc
    ([[0], [1, 2, 3]], [1, 2], [], [3]),           # {1,2,3,4} & 2 of ({2,3,5}, {3,4,5,6}, {1,6,7})
    ([[0, 4, 7]], [2], [], []),                    # id 7 is absent (an empty list that still counts) and 9 is alone
    ([[0, 1, 4]], [2], [], [2, 3]),
])
def test_hand_written_answers(groups, mins, excl, want):
    assert mr.match_docs(TINY, groups, excl, mins=mins).tolist() == want
    assert mr.count([TINY], groups, excl, mins=mins) == len(want)


def test_deleted_docs_and_filter():
    mask = np.array([True, False, True, True, True, True, True, True, True])   # row 1 = doc 2 fails the filter
    assert mr.match_docs(TINY, [[0, 1, 2]], deleted=u(4), mask=mask, mins=[2]).tolist() == [3, 5]


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.default_rng(77)
    n = 20_000
    norms = rng.integers(1, 200, n).astype(np.uint32)
    seg = orc.Segment(n, has_wand=True)
    seg.set_norms(norms)
    lists = []
    for p in (0.4, 0.25, 0.1, 0.05, 0.5, 0.01, 0.003, 0.2):
        d = (np.flatnonzero(rng.random(n) < p) + 1).astype(np.uint32)
        seg.add_term(d, rng.integers(1, 5, len(d)).astype(np.uint32))
        lists.append(d)
    vals, valid = rng.integers(0, 1000, n).astype(np.int64), rng.random(n) < 0.7
    seg.add_column(4, vals, cr.validity_words(valid))
    ttf = int(norms.astype(np.uint64).sum())
    terms = []
    for t, d in enumerate(lists):
        st = orc.bm25_stats(n, ttf, len(d))
        x = orc.BM25Term()
        x.idf, x.norm_const, x.norm_length, x.boost, x.term = st.idf, st.norm_const, st.norm_length, 1.0, t
        terms.append(x)
    return dict(seg=seg, n=n, lists=lists, terms=terms, col=(vals, valid))


CASES = [
    ([[0, 1, 2]], [2], []),
    ([[0, 1, 2, 3]], [3], [5]),
    ([[0, 1, 2, 3]], [2], []),
    ([[7], [0, 1, 2]], [1, 2], [3]),
    ([[4, 7], [0, 1, 2, 3, 5]], [1, 3], []),
    ([[0, 1, 2, 3, 4, 5, 6, 7]], [4], []),
]


def _groups(c, gids):
    return [[c["terms"][t] for t in g] for g in gids]


@pytest.mark.parametrize("gids,mins,excl", CASES)
@pytest.mark.parametrize("filt", [None, (4, "BETWEEN", 100, 899)], ids=["nofilter", "between"])
@pytest.mark.parametrize("deleted", [False, True], ids=["live", "deleted"])
def test_reference_matches_numpy_statement(corpus, gids, mins, excl, filt, deleted):
    c = corpus
    dele = np.arange(3, c["n"] + 1, 11, dtype=np.uint32) if deleted else None
    ofilt = orc.make_pred(*filt) if filt else None
    mask = None if filt is None else cr.pred_mask(c["col"][0], c["col"][1], filt[1], filt[2], filt[3])
    c["seg"].set_docs_mask(dele if dele is not None else np.zeros(0, np.uint32))
    try:
        hits, total = mr.topk_groups([c["seg"]], _groups(c, gids), excl, c["n"], filt=ofilt, mode=0, deleted=[dele], mins=mins)
        want = mr.match_docs(c["lists"], gids, excl, dele, mask, mins=mins)
        assert np.array_equal(np.sort(hits["doc"]), want) and total == len(want) > 0
        flat = [t for g in _groups(c, gids) for t in g]
        allh, _, _ = orc.bm25_topk([c["seg"]], "OR", flat, c["n"], filt=ofilt, mode=0)
        kept = allh[np.isin(allh["doc"], want)]
        assert np.array_equal(hits["doc"], kept["doc"])
        assert np.array_equal(hits["score"].view(np.uint32), kept["score"].view(np.uint32))
    finally:
        c["seg"].set_docs_mask(np.zeros(0, np.uint32))


def test_one_is_the_groups_statement_and_all_is_the_and(corpus):
    c = corpus
    for gids, excl in (([[0], [1, 2]], [3]), ([[4, 7], [1, 2, 3], [0]], [5]), ([[0, 1, 2]], [])):
        ones = [1] * len(gids)
        assert np.array_equal(mr.match_docs(c["lists"], gids, excl, mins=ones), gr.match_docs(c["lists"], gids, excl))
        h1, t1 = mr.topk_groups([c["seg"]], _groups(c, gids), excl, 100, mode=0, mins=ones)
        h0, t0 = gr.topk_groups([c["seg"]], _groups(c, gids), excl, 100, mode=0)
        assert t1 == t0 and np.array_equal(h1, h0)
    gids = [[0, 4, 7], [2]]
    assert mr.count([c["lists"]], gids, [5], mins=[3, 1]) == cr.count([c["lists"]], "AND", [0, 4, 7, 2], [5])
    h, t = mr.topk_groups([c["seg"]], _groups(c, [[0, 4, 7]]), [], 100, mode=0, mins=[3])
    oh, ot, _ = orc.bm25_topk([c["seg"]], "AND", _groups(c, [[0, 4, 7]])[0], 100, mode=0)
    assert t == ot and np.array_equal(h["doc"], oh["doc"]) and np.array_equal(h["score"].view(np.uint32), oh["score"].view(np.uint32))


def test_batch_takes_per_query_minimums(corpus):
    c = corpus
    qs = [_groups(c, g) for g, _, _ in CASES]
    xs = [x for _, _, x in CASES]
    ms = [m for _, m, _ in CASES]
    hits, n_out, total = mr.topk_batch_groups([c["seg"]], qs, xs, 50, min_match=ms, mode=0)
    for q in range(len(qs)):
        h, t = mr.topk_groups([c["seg"]], qs[q], xs[q], 50, mode=0, mins=ms[q])
        assert n_out[q] == len(h) and total[q] == t
        assert np.array_equal(hits[q, :n_out[q]], h)
