"""Block-max pruning over several segments whose average field lengths differ from the corpus-wide one.

The writer picks each block's (freq, norm) pair under the segment's own average length; a query scores with the
corpus-wide average. Pruned top-k must still equal the exhaustive oracle bit for bit (DESIGN §4.3), and the scores must
agree with BM25 computed from first principles in float64."""
import numpy as np
import pytest

import orc
import serenedb_b200 as sdb
from gpu_util import assert_hits_equal, ctx, oracle_terms, to_gpu
from shape_corpora import (B, K1, Corpus, adversarial_segments, bm25_f64, natural_segments, stored_pair,
                           uniform_segments, writer_avg_dl)

pytestmark = pytest.mark.gpu


def _reader(corpus):
    gsegs = [to_gpu(o) for o in corpus.osegs]
    return sdb.IndexReader(gsegs, corpus.docs_with_field, corpus.total_term_freq, corpus.docs_with_term)


def _kind(kind):
    return sdb.AND if kind == "AND" else sdb.OR


@pytest.fixture(params=[1, 2])
def wand(request):
    ctx().set_wand(request.param)
    yield request.param
    ctx().set_wand(0)


@pytest.fixture(scope="module")
def adversarial():
    dlA, lA, dlB, lB, pair_docs, best_docs = adversarial_segments()
    corpus = Corpus([(dlA, lA), (dlB, lB)])
    return dict(corpus=corpus, reader=_reader(corpus), dlA=dlA, lA=lA, pair_docs=pair_docs, best_docs=best_docs)


def test_adversarial_corpus_shape(adversarial):
    """The corpus really holds the flaw the tests below are about: the block's stored pair is (1, 1), and at the query's
    constants it scores below the block's (10, 20) posting."""
    c, dlA, (docs, freqs) = adversarial["corpus"], adversarial["dlA"], adversarial["lA"][0]
    a_s = writer_avg_dl(dlA)
    b0 = adversarial["pair_docs"][0] - 6
    assert stored_pair(freqs[b0:b0 + 128], dlA[b0:b0 + 128], a_s) == (1, 1)
    sk = c.osegs[0].skip_level0(0)
    assert (int(sk["wand_freq"][7]), int(sk["wand_norm"][7])) == (1, 1)
    st = adversarial["reader"].stats(sdb.BM25(), 0)
    c0 = sdb.BM25().num(st)
    s11, s1020 = orc.bm25_score([1, 10], [1, 20], orc.BM25Stats(st.idf, st.norm_const, st.norm_length))
    assert s11 < s1020 and c0 > 0


QUERIES = [("OR", [0]), ("OR", [0, 1]), ("OR", [0, 1, 2]), ("OR", [0, 1, 2, 3]), ("OR", [0, 1, 2, 3, 4, 5]),
           ("AND", [0, 1]), ("AND", [0, 1, 2, 3])]


@pytest.mark.parametrize("kind,tis", QUERIES)
def test_seeded_threshold_between_stored_pair_and_block_best(adversarial, wand, kind, tis):
    """A threshold seeded strictly between the stored pair's score (plus the most the other terms can add) and the
    (10, 20) posting's score: a bound taken from the stored pair with the query's constants skips the block and loses
    the best hits."""
    reader, corpus = adversarial["reader"], adversarial["corpus"]
    scorer = sdb.BM25()
    st = reader.stats(scorer, 0)
    ost = orc.BM25Stats(st.idf, st.norm_const, st.norm_length)
    s11, s1020 = (float(x) for x in orc.bm25_score([1, 10], [1, 20], ost))
    others = sum(float(scorer.num(reader.stats(scorer, t))) for t in tis[1:])   # any term scores below its c0
    lo, hi = s11 + others, s1020
    assert lo < hi, (lo, hi)
    thr = float(np.float32((lo + hi) / 2))
    hits, total = sdb.ExecuteTopK(reader, tis, _kind(kind), scorer, 10, threshold=thr)
    oh, ototal, _ = orc.bm25_topk(corpus.osegs, kind, oracle_terms(reader, scorer, tis), 10, threshold_in=np.float32(thr), mode=1)
    assert_hits_equal(hits, oh)
    if kind == "OR" and len(tis) == 1:      # the eight (10, 20) postings lead the result
        assert sorted(hits["doc"][:8].tolist()) == adversarial["best_docs"] and np.all(hits["seg"][:8] == 0)
    assert total <= ototal if kind == "OR" else total == ototal


@pytest.mark.parametrize("kind,tis,k", [("OR", [0], 10), ("OR", [0], 8), ("OR", [0, 1], 10), ("OR", [0, 1, 2, 3, 4, 5], 10)])
def test_threshold_raised_inside_the_segment(adversarial, wand, kind, tis, k):
    """No seed: the (tf 2, dl 2) blocks before every bad block raise the threshold above the stored pair's score."""
    reader, corpus = adversarial["reader"], adversarial["corpus"]
    scorer = sdb.BM25()
    hits, total = sdb.ExecuteTopK(reader, tis, sdb.OR, scorer, k)
    oh, ototal, _ = orc.bm25_topk(corpus.osegs, kind, oracle_terms(reader, scorer, tis), k, mode=1)
    assert_hits_equal(hits, oh)
    assert total <= ototal
    if tis == [0]:
        assert set(adversarial["best_docs"][:k]) <= set(hits["doc"].tolist())


@pytest.fixture(scope="module")
def natural():
    corpus = Corpus(natural_segments())
    return dict(corpus=corpus, reader=_reader(corpus))


def _random_queries(rng, n, n_terms, max_terms=4):
    return [sorted(int(t) for t in rng.choice(n_terms, size=int(rng.integers(1, max_terms + 1)), replace=False)) for _ in range(n)]


def test_natural_corpus_pruned_equals_exhaustive(natural, wand):
    reader, corpus = natural["reader"], natural["corpus"]
    scorer = sdb.BM25()
    rng = np.random.default_rng(wand)
    for kind in ("OR", "AND"):
        for tis in _random_queries(rng, 24, corpus.n_terms):
            for k in (10, 100):
                hits, total = sdb.ExecuteTopK(reader, tis, _kind(kind), scorer, k)
                oh, ototal, _ = orc.bm25_topk(corpus.osegs, kind, oracle_terms(reader, scorer, tis), k, mode=1)
                assert_hits_equal(hits, oh)
                assert total <= ototal if kind == "OR" else total == ototal, (kind, tis, k)
    # the lead-mode shape: [long, short], long >= 4x short in every segment
    for tis in ([0, 6], [7, 5], [0, 9], [1, 6]):
        hits, total = sdb.ExecuteTopK(reader, tis, sdb.OR, scorer, 10)
        oh, ototal, _ = orc.bm25_topk(corpus.osegs, "OR", oracle_terms(reader, scorer, tis), 10, mode=1)
        assert_hits_equal(hits, oh)
        assert total <= ototal


def test_natural_corpus_batch(natural, wand):
    reader, corpus = natural["reader"], natural["corpus"]
    scorer = sdb.BM25()
    queries = _random_queries(np.random.default_rng(100 + wand), 64, corpus.n_terms)
    bh, bn, bt = sdb.ExecuteTopKBatch(reader, queries, sdb.OR, scorer, 50)
    for qi, tis in enumerate(queries):
        oh, ototal, _ = orc.bm25_topk(corpus.osegs, "OR", oracle_terms(reader, scorer, tis), 50, mode=1)
        assert_hits_equal(bh[qi, :bn[qi]], oh)
        assert bt[qi] <= ototal


def test_natural_corpus_scores_from_first_principles(natural):
    """The top hits' scores recomputed in float64 from tf, dl, k, b, idf and the corpus average: a check that does not
    lean on the oracle, so it would see a mistake the GPU and the oracle share."""
    reader, corpus = natural["reader"], natural["corpus"]
    scorer = sdb.BM25(K1, B)
    ctx().set_wand(2)
    try:
        for tis in ([0], [3, 5], [0, 2, 8], [1, 4, 6, 9]):
            hits, _ = sdb.ExecuteTopK(reader, tis, sdb.OR, scorer, 50)
            assert len(hits) == 50
            for h in hits:
                seg, doc = int(h["seg"]), int(h["doc"])
                exp = 0.0
                for t in tis:
                    d, f = corpus.lists[seg][t]
                    i = np.searchsorted(d, doc)
                    if i < len(d) and d[i] == doc:
                        exp += float(bm25_f64(f[i], corpus.norms[seg][doc - 1], corpus.docs_with_field,
                                              corpus.total_term_freq, corpus.docs_with_term[t]))
                assert exp > 0 and abs(float(h["score"]) - exp) <= 1e-5 * exp, (tis, seg, doc, float(h["score"]), exp)
    finally:
        ctx().set_wand(0)


def test_split_corpus_equals_whole(wand):
    """Sanity baseline: segments that share one length distribution give the same pruned top-k as the whole corpus in
    one segment, and as the oracle."""
    (norms, lists), parts, cuts = uniform_segments()
    whole, split = Corpus([(norms, lists)]), Corpus(parts)
    assert whole.docs_with_term == split.docs_with_term and whole.total_term_freq == split.total_term_freq
    r1, r3 = _reader(whole), _reader(split)
    scorer = sdb.BM25()
    for kind, tis, k in (("OR", [0], 10), ("OR", [0, 1], 100), ("OR", [1, 2, 3], 100), ("OR", [0, 4, 5, 2], 20),
                         ("AND", [0, 4], 100), ("OR", [0, 5], 10)):
        h1, _ = sdb.ExecuteTopK(r1, tis, _kind(kind), scorer, k)
        h3, t3 = sdb.ExecuteTopK(r3, tis, _kind(kind), scorer, k)
        glob = h3["doc"] + np.array(cuts[:-1], np.uint32)[h3["seg"]]
        assert np.array_equal(glob, h1["doc"]) and np.array_equal(h3["score"].view(np.uint32), h1["score"].view(np.uint32))
        oh, ototal, _ = orc.bm25_topk(split.osegs, kind, oracle_terms(r3, scorer, tis), k, mode=1)
        assert_hits_equal(h3, oh)
        assert t3 <= ototal if kind == "OR" else t3 == ototal
