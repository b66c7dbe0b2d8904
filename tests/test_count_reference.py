"""The NumPy statement of the Count mode (tests/count_reference.py) against the oracle's exhaustive total_matches
(orc.bm25_topk mode 0; tests/excl_reference.py for excluded terms): OR and AND, the hybrid filter on int32 / int64 /
float64 columns and on a nullable column (IS_NULL / IS_NOT_NULL included), deleted docs and exclusions. No GPU needed."""
import numpy as np
import pytest

import count_reference as cr
import orc
from excl_reference import topk_excl


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.default_rng(77)
    n = 20_000
    norms = rng.integers(1, 200, n).astype(np.uint32)
    seg = orc.Segment(n, has_wand=True)
    seg.set_norms(norms)
    lists = []
    for p in (0.4, 0.25, 0.1, 0.05, 0.5, 0.01, 0.003):
        d = (np.flatnonzero(rng.random(n) < p) + 1).astype(np.uint32)
        seg.add_term(d, rng.integers(1, 5, len(d)).astype(np.uint32))
        lists.append(d)
    cols = {
        1: (rng.integers(0, 1000, n).astype(np.int32), None),
        2: (rng.integers(-10**12, 10**12, n).astype(np.int64), None),
        3: (rng.random(n) * 100.0, None),
        4: (rng.integers(0, 1000, n).astype(np.int64), rng.random(n) < 0.7),    # nullable
    }
    for f, (v, valid) in cols.items():
        seg.add_column(f, v, cr.validity_words(valid) if valid is not None else None)
    ttf = int(norms.astype(np.uint64).sum())
    terms = []
    for t, d in enumerate(lists):
        st = orc.bm25_stats(n, ttf, len(d))
        x = orc.BM25Term()
        x.idf, x.norm_const, x.norm_length, x.boost, x.term = st.idf, st.norm_const, st.norm_length, 1.0, t
        terms.append(x)
    return dict(seg=seg, n=n, lists=lists, terms=terms, cols=cols)


QUERIES = [("OR", [0]), ("OR", [2, 3]), ("OR", [1, 3, 5, 6]), ("AND", [0, 4]), ("AND", [0, 1, 4]), ("AND", [2, 5])]
FILTERS = [
    None,
    (1, "BETWEEN", 250, 749, False),
    (2, "LT", 0, 0, False),
    (3, "GE", 42.5, 0, True),
    (4, "GT", 500, 0, False),
    (4, "IS_NULL", 0, 0, False),
    (4, "IS_NOT_NULL", 0, 0, False),
]


def _oracle_total(c, kind, pos, excl, filt):
    ofilt = orc.make_pred(filt[0], filt[1], filt[2], filt[3], is_float=filt[4]) if filt else None
    terms = [c["terms"][t] for t in pos]
    if excl:
        return topk_excl([c["seg"]], kind, terms, excl, 10, filt=ofilt, mode=0)[1]
    return orc.bm25_topk([c["seg"]], kind, terms, 10, filt=ofilt, mode=0)[1]


def _mask(c, filt):
    if filt is None:
        return None
    v, valid = c["cols"][filt[0]]
    return cr.pred_mask(v, valid, filt[1], filt[2], filt[3])


@pytest.mark.parametrize("kind,pos", QUERIES)
@pytest.mark.parametrize("filt", FILTERS, ids=lambda f: "nofilter" if f is None else "%d_%s" % (f[0], f[1]))
def test_count_statement_matches_oracle_total(corpus, kind, pos, filt):
    c = corpus
    want = cr.count([c["lists"]], kind, pos, masks=[_mask(c, filt)])
    assert want == _oracle_total(c, kind, pos, [], filt)


@pytest.mark.parametrize("kind,pos,excl", [("OR", [0, 2], [3]), ("OR", [2, 3], [2]), ("AND", [0, 4], [4]),
                                           ("AND", [0, 1, 4], [3, 5, 6]), ("OR", [0], [999]), ("OR", [1, 5], [0, 2, 3, 4, 6])])
def test_exclusions_and_deleted_docs(corpus, kind, pos, excl):
    c = corpus
    deleted = np.arange(3, c["n"] + 1, 11, dtype=np.uint32)
    filt = (4, "BETWEEN", 100, 899, False)
    for dele in (None, deleted):
        c["seg"].set_docs_mask(dele if dele is not None else np.zeros(0, np.uint32))
        try:
            for f in (None, filt):
                want = cr.count([c["lists"]], kind, pos, excl, deleted=[dele], masks=[_mask(c, f)])
                ofilt = orc.make_pred(f[0], f[1], f[2], f[3]) if f else None
                got = topk_excl([c["seg"]], kind, [c["terms"][t] for t in pos], excl, 10, filt=ofilt, mode=0, deleted=[dele])[1]
                assert want == got, (kind, pos, excl, dele is not None, f)
        finally:
            c["seg"].set_docs_mask(np.zeros(0, np.uint32))


def test_self_exclusion_semantics(corpus):
    c = corpus
    assert cr.count([c["lists"]], "AND", [0, 4], [4]) == 0
    assert cr.count([c["lists"]], "OR", [2, 3], [2]) == len(np.setdiff1d(c["lists"][3], c["lists"][2]))
