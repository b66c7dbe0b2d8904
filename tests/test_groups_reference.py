"""The reference for conjunctions of OR groups (`a & (b | c) & !d`, tests/groups_reference.py) against a NumPy statement of
the semantics built from the raw doc lists: the intersection over the groups of each group's union, minus the excluded
lists, the deleted docs and the rows the filter rejects (NULL never passes), each doc scored as the flat OR of the
positive terms scores it. No GPU needed."""
import numpy as np
import pytest

import count_reference as cr
import groups_reference as gr
import orc


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.default_rng(53)
    n = 20_000
    norms = rng.integers(1, 200, n).astype(np.uint32)
    seg = orc.Segment(n, has_wand=True)
    seg.set_norms(norms)
    lists = []
    for p in (0.4, 0.25, 0.1, 0.05, 0.5, 0.01, 0.003, 0.2):
        d = (np.flatnonzero(rng.random(n) < p) + 1).astype(np.uint32)
        seg.add_term(d, rng.integers(1, 5, len(d)).astype(np.uint32))
        lists.append(d)
    vals, valid = rng.integers(0, 1000, n).astype(np.int64), rng.random(n) < 0.7     # nullable column
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
    ([[0], [1, 2]], []),                  # a & (b | c)
    ([[0], [1, 2]], [3]),                 # a & (b | c) & !d
    ([[4, 7], [1, 2, 3], [0]], [5]),
    ([[1, 2], [3, 5, 6]], []),
    ([[0], [1, 2]], [2]),                 # a term of a group also excluded: the group keeps its other terms
    ([[6], [0, 1]], [999]),               # absent excluded id: excludes nothing
    ([[0, 1, 2]], []),                    # one group: the flat OR
    ([[0], [4], [7]], []),                # single-term groups: the AND
]
FILTERS = [None, (4, "BETWEEN", 100, 899), (4, "IS_NULL", 0, 0)]


def _groups(c, gids):
    return [[c["terms"][t] for t in g] for g in gids]


def _mask(c, filt):
    return None if filt is None else cr.pred_mask(c["col"][0], c["col"][1], filt[1], filt[2], filt[3])


@pytest.mark.parametrize("gids,excl", CASES)
@pytest.mark.parametrize("filt", FILTERS, ids=lambda f: "nofilter" if f is None else f[1])
@pytest.mark.parametrize("deleted", [False, True], ids=["live", "deleted"])
def test_groups_reference_matches_numpy_statement(corpus, gids, excl, filt, deleted):
    c = corpus
    dele = np.arange(3, c["n"] + 1, 11, dtype=np.uint32) if deleted else None
    ofilt = orc.make_pred(filt[0], filt[1], filt[2], filt[3]) if filt else None
    c["seg"].set_docs_mask(dele if dele is not None else np.zeros(0, np.uint32))
    try:
        for mode in (0, 1):
            hits, total = gr.topk_groups([c["seg"]], _groups(c, gids), excl, c["n"], filt=ofilt, mode=mode, deleted=[dele])
            want = gr.match_docs(c["lists"], gids, excl, dele, _mask(c, filt))
            assert np.array_equal(np.sort(hits["doc"]), want)
            assert total == len(want) == gr.count([c["lists"]], gids, excl, [dele], [_mask(c, filt)])
        # scores are the flat OR's own, bit for bit: the same docs out of the flat OR of every positive term
        flat = [t for g in _groups(c, gids) for t in g]
        allh, _, _ = orc.bm25_topk([c["seg"]], "OR", flat, c["n"], filt=ofilt, mode=0)
        kept = allh[np.isin(allh["doc"], want)]
        assert np.array_equal(hits["doc"], kept["doc"])
        assert np.array_equal(hits["score"].view(np.uint32), kept["score"].view(np.uint32))
    finally:
        c["seg"].set_docs_mask(np.zeros(0, np.uint32))


def test_degenerate_forms_are_the_flat_queries(corpus):
    c = corpus
    assert gr.count([c["lists"]], [[0, 1, 2]], [3]) == cr.count([c["lists"]], "OR", [0, 1, 2], [3])
    assert gr.count([c["lists"]], [[0], [4], [7]], [5]) == cr.count([c["lists"]], "AND", [0, 4, 7], [5])
    h, t = gr.topk_groups([c["seg"]], _groups(c, [[0], [4]]), [], 100, mode=0)
    oh, ot, _ = orc.bm25_topk([c["seg"]], "AND", [c["terms"][0], c["terms"][4]], 100, mode=0)
    assert t == ot and np.array_equal(h["doc"], oh["doc"]) and np.array_equal(h["score"].view(np.uint32), oh["score"].view(np.uint32))


def test_batch_matches_single_queries_and_restores_the_mask(corpus):
    c = corpus
    qs = [_groups(c, g) for g, _ in CASES]
    xs = [x for _, x in CASES]
    hits, n_out, total = gr.topk_batch_groups([c["seg"]], qs, xs, 50, mode=0)
    for q, (groups, excl) in enumerate(zip(qs, xs)):
        h, t = gr.topk_groups([c["seg"]], groups, excl, 50, mode=0)
        assert n_out[q] == len(h) and total[q] == t
        assert np.array_equal(hits[q, :n_out[q]], h)
    _, ptotal, _ = orc.bm25_topk([c["seg"]], "OR", [c["terms"][0]], 10, mode=0)
    assert ptotal == len(c["lists"][0])
