"""The reference for excluded terms (`a & b & !c`, tests/excl_reference.py) against a NumPy statement of the semantics
built from the raw doc lists: the positive part's matches (union for OR, intersection for AND) minus the union of the
excluded lists, each doc scored by the positive terms alone. No GPU needed."""
import numpy as np
import pytest

import orc
from excl_reference import topk_batch_excl, topk_excl


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.default_rng(31)
    n = 20_000
    norms = rng.integers(1, 200, n).astype(np.uint32)
    seg = orc.Segment(n, has_wand=True)
    seg.set_norms(norms)
    lists = []
    for p in (0.4, 0.25, 0.1, 0.05, 0.5, 0.01, 0.003):
        d = (np.flatnonzero(rng.random(n) < p) + 1).astype(np.uint32)
        f = rng.integers(1, 5, len(d)).astype(np.uint32)
        seg.add_term(d, f)
        lists.append(d)
    ttf = int(norms.astype(np.uint64).sum())
    terms = []
    for t, d in enumerate(lists):
        st = orc.bm25_stats(n, ttf, len(d))
        x = orc.BM25Term()
        x.idf, x.norm_const, x.norm_length, x.boost, x.term = st.idf, st.norm_const, st.norm_length, 1.0, t
        terms.append(x)
    return dict(seg=seg, n=n, lists=lists, terms=terms)


def _expected_docs(c, kind, pos, excl):
    sets = [set(c["lists"][t].tolist()) for t in pos]
    keep = set.union(*sets) if kind == "OR" else set.intersection(*sets)
    for t in excl:
        if t < len(c["lists"]):                 # an id the segment does not hold excludes nothing
            keep -= set(c["lists"][t].tolist())
    return keep


CASES = [
    ("OR", [0, 2], [3]),
    ("OR", [1, 3, 5], [4, 6]),
    ("AND", [0, 4], [2]),
    ("AND", [0, 1, 4], [3, 5, 6]),
    ("OR", [2, 3], [2]),                # excluded and positive: only the other term's docs that are not in it
    ("AND", [0, 4], [4]),               # excluded and positive: empty
    ("OR", [0], [999]),                 # absent term id: excludes nothing
    ("AND", [1, 2], []),                # empty set: the query without exclusions
]


@pytest.mark.parametrize("kind,pos,excl", CASES)
@pytest.mark.parametrize("mode", [0, 1])
def test_exclusion_matches_numpy_statement(corpus, kind, pos, excl, mode):
    c = corpus
    terms = [c["terms"][t] for t in pos]
    want = _expected_docs(c, kind, pos, excl)
    hits, total = topk_excl([c["seg"]], kind, terms, excl, c["n"], mode=mode)
    assert set(hits["doc"].tolist()) == want
    assert total == len(want)
    # the scores are the positive part's own, bit for bit: the same docs out of the query without exclusions
    allh, _, _ = orc.bm25_topk([c["seg"]], kind, terms, c["n"], mode=0)
    kept = allh[np.isin(allh["doc"], np.fromiter(want, np.uint32, len(want)))]
    assert np.array_equal(hits["doc"], kept["doc"])
    assert np.array_equal(hits["score"].view(np.uint32), kept["score"].view(np.uint32))


def test_deleted_docs_and_exclusions_combine_and_the_mask_is_restored(corpus):
    c = corpus
    deleted = np.arange(5, c["n"] + 1, 7, dtype=np.uint32)
    c["seg"].set_docs_mask(deleted)
    try:
        terms = [c["terms"][t] for t in (0, 2)]
        want = _expected_docs(c, "OR", [0, 2], [3]) - set(deleted.tolist())
        hits, total = topk_excl([c["seg"]], "OR", terms, [3], c["n"], deleted=[deleted])
        assert set(hits["doc"].tolist()) == want and total == len(want)
        plain, ptotal, _ = orc.bm25_topk([c["seg"]], "OR", terms, c["n"], mode=0)   # the segment's own mask is back
        assert ptotal == len(_expected_docs(c, "OR", [0, 2], []) - set(deleted.tolist()))
    finally:
        c["seg"].set_docs_mask(np.zeros(0, np.uint32))


def test_exclusion_batch_matches_single_queries(corpus):
    c = corpus
    ors = [(pos, excl) for kind, pos, excl in CASES if kind == "OR"]
    qs = [[c["terms"][t] for t in pos] for pos, _ in ors]
    xs = [excl for _, excl in ors]
    hits, n_out, total = topk_batch_excl([c["seg"]], "OR", qs, xs, 50, mode=0)
    for q, (terms, excl) in enumerate(zip(qs, xs)):
        h, t = topk_excl([c["seg"]], "OR", terms, excl, 50, mode=0)
        assert n_out[q] == len(h) and total[q] == t
        assert np.array_equal(hits[q, :n_out[q]], h)
