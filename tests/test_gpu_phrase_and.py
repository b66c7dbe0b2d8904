"""Conjunctions of phrases, terms and negated phrases on the GPU (sdbg_phrase_and_{count,topk,topk_by_column,
facet_counts,aggregate,scan}_batch) against the NumPy statement (tests/phrase_and_reference.py), bit for bit: counts,
hits (doc, segment, order, fp32 score bits), sorted hits, facet and aggregate cells, scan pages and totals. Over
token-sequence segments where one lacks a term of a positive clause and one a term of a negated clause, with deleted
docs, filter chains of 1..4 predicates, exclusions, one-slot and multi-slot negated clauses, every scorer, pruning levels
0..2, k above the match count and ties at the cut, a query of exactly 16 slots, doc ids past 2^31; the two identities
(one positive clause: the phrase entries; one-slot clauses of distinct terms: the flat AND entries); the error codes."""
import ctypes as C

import numpy as np
import pytest

import count_reference as cr
import orc
import phrase_and_reference as par
import phrase_reference as pr
import serenedb_b200 as sdb
from serenedb_b200 import _native as N
from gpu_util import ctx, to_gpu

pytestmark = pytest.mark.gpu

V = 12                       # vocabulary: term 11 never occurs in segment 1, term 10 never in segment 2
SIZES = (3000, 2500, 4000)
I32, F64, KEY, FILT = 1, 3, 5, 4
SCORERS = [sdb.BM25(), sdb.BM25(1.2, 0.0), sdb.BM25(0.0, 0.75), sdb.TFIDF(False), sdb.TFIDF(True)]
SCORER_IDS = ["bm25", "bm15", "bm1", "tfidf", "tfidf_norm"]


def _token_segment(rng, n, missing=()):
    p = 1.0 / np.arange(1, V + 1)
    for t in missing:
        p[t] = 0
    p /= p.sum()
    docs = [rng.choice(V, size=int(rng.integers(1, 40)), p=p).tolist() for _ in range(n)]
    post = pr.postings(docs, V)
    oseg = orc.Segment(n, has_wand=True)
    norms = np.array([len(d) for d in docs], np.uint32)
    oseg.set_norms(norms)
    for d, f, _ in post:
        oseg.add_term(d, f)
    return docs, post, norms, oseg


@pytest.fixture(scope="module")
def pa():
    rng = np.random.default_rng(777)
    segs, docs, norms, cols = [], [], [], []
    for i, n in enumerate(SIZES):
        d, post, nm, oseg = _token_segment(rng, n, missing={1: (11,), 2: (10,)}.get(i, ()))
        c = {I32: (rng.integers(-1000, 1000, n).astype(np.int32), rng.random(n) < 0.85),
             F64: (rng.random(n) * 200.0 - 100.0, rng.random(n) < 0.8),
             KEY: (rng.integers(-5, 20, n).astype(np.int32), rng.random(n) < 0.9),
             FILT: (rng.integers(0, 50, n).astype(np.int32), None)}
        g = to_gpu(oseg, columns={f: (v, None if m is None else cr.validity_words(m)) for f, (v, m) in c.items()})
        g.stage_positions(*pr.staged_positions(post))
        segs.append(g); docs.append(d); norms.append(nm); cols.append(c)
    deleted = [rng.choice(np.arange(1, SIZES[0] + 1), 300, replace=False).astype(np.uint32), None, None]
    segs[0].stage_docs_mask(deleted[0])
    dwt = [sum(sum(1 for x in d if t in x) for d in docs) for t in range(V)]
    reader = sdb.IndexReader(segs, sum(SIZES), int(sum(int(n.sum()) for n in norms)), dwt)
    return dict(segs=segs, docs=docs, norms=norms, cols=cols, deleted=deleted, reader=reader)


def _cut(t, rng, L):
    seq = t["docs"][int(rng.integers(0, 3))][int(rng.integers(0, 2500))]
    if len(seq) < L:
        return rng.integers(0, 4, L).tolist(), seq
    s = int(rng.integers(0, len(seq) - L + 1))
    return seq[s:s + L], seq


def _queries(t, rng, n):
    """(positive clauses, negated clauses) per query: `"w1 w2" & t` with t from the phrase's doc, the same with a
    negated phrase or term, two phrases, and a phrase with a gap; plus queries on the missing terms."""
    qs = []
    for i in range(n):
        ph, seq = _cut(t, rng, 2 + i % 2)
        term = [int(seq[int(rng.integers(0, len(seq)))])]
        neg = []
        if i % 3 == 1:
            neg = [_cut(t, rng, 2)[0]]
        elif i % 3 == 2:
            neg = [[int(rng.integers(3, 10))]]
        pos = [ph, term]
        if i % 4 == 3:
            pos.append((_cut(t, rng, 2)[0][:1] + [int(rng.integers(0, 4))], [0, 2]))
        qs.append((pos, neg))
    qs += [([[0, 1], [11]], []), ([[0, 1], [2]], [[10, 0]]), ([[0], [1]], [[10]]), ([[1, 0], [0]], [[0, 1]]),
           ([[0, 0], [0]], [[1, 2], [3]])]
    return qs


def _clauses(q):
    pos, neg = q
    c = lambda x, n: (list(x[0]), list(x[1]), n) if isinstance(x, tuple) else (list(x), None, n)
    return [c(x, False) for x in pos] + [c(x, True) for x in neg]


def _consts(t, q, scorer):
    return [None if n else pr.consts(t["reader"].phrase_stats(scorer, terms), scorer.k, scorer.b) for terms, _, n in _clauses(q)]


def _same_sorted(a, b):
    assert np.array_equal(a["n_out"], b["n_out"])
    for f in ("docs", "segs", "values", "nulls"):
        assert all(np.array_equal(x, y) for x, y in zip(a[f], b[f])), f


def _want(t, q, excl=(), masks=None):
    return par.matches(t["docs"], _clauses(q), excl, t["deleted"], masks)


def _col(t, f):
    return [c[f] for c in t["cols"]]


def _check(t, queries, scorer=None, k=10, excl=None, filt=None, masks=None, levels=(0,), passes=True):
    excl = excl or [[]] * len(queries)
    Q, X = [q[0] for q in queries], [q[1] for q in queries]
    kw = dict(filt=filt, exclude=excl, exclude_phrases=X)
    wants = [_want(t, q, x, masks) for q, x in zip(queries, excl)]
    counts = sdb.ExecutePhraseAndCountBatch(t["reader"], Q, **kw)
    assert counts.tolist() == [par.count(w) for w in wants]
    if scorer is not None:
        for lv in levels:
            ctx().set_wand(lv)
            hits, n_out, total = sdb.ExecutePhraseAndTopKBatch(t["reader"], Q, scorer, k, **kw)
            assert np.array_equal(total, counts)
            for i, (q, w) in enumerate(zip(queries, wants)):
                ref, _ = par.topk(t["docs"], _clauses(q), w, t["norms"], _consts(t, q, scorer), k)
                got = hits[i, :n_out[i]]
                assert len(got) == len(ref), (q, lv)
                assert np.array_equal(got["doc"], ref["doc"]) and np.array_equal(got["seg"], ref["seg"]), (q, lv)
                assert np.array_equal(got["score"].view(np.uint32), ref["score"].view(np.uint32)), (q, lv)
            ctx().set_wand(False)
    if not passes:
        return counts
    got = sdb.ExecutePhraseAndTopKByColumnBatch(t["reader"], Q, I32, k, True, False, **kw)
    for i, w in enumerate(wants):
        ref = par.sorted_hits(w, _col(t, I32), True, False, k)
        assert np.array_equal(got["docs"][i], ref["docs"]) and np.array_equal(got["segs"][i], ref["segs"]), queries[i]
        assert np.array_equal(got["values"][i], ref["values"]) and np.array_equal(got["nulls"][i], ref["nulls"])
    got = sdb.ExecutePhraseAndFacetCountsBatch(t["reader"], Q, KEY, -5, 25, **kw)
    for i, w in enumerate(wants):
        c, nulls = par.facet_counts(w, _col(t, KEY), -5, 25)
        assert got["counts"][i].tolist() == c.tolist() and int(got["nulls"][i]) == nulls, queries[i]
    got = sdb.ExecutePhraseAndMatchAggregatesBatch(t["reader"], Q, I32, KEY, -5, 25, **kw)
    for i, w in enumerate(wants):
        cells, null_cell = par.aggregate(w, _col(t, KEY), _col(t, I32), -5, 25)
        for j, cell in enumerate(cells):
            assert int(got["count"][i][j]) == cell["count"] and int(got["count_value"][i][j]) == cell["count_value"]
            if cell["count_value"]:
                assert int(got["sum"][i][j]) == cell["sum"] and int(got["min"][i][j]) == cell["min"]
                assert int(got["max"][i][j]) == cell["max"]
        assert int(got["null"]["count"][i]) == null_cell["count"]
    sc = scorer or sdb.BM25()
    for offs, limit in ((None, 1 << 14), (np.array([c // 2 for c in counts], np.uint64), 7)):
        got = sdb.ExecutePhraseAndMatchScanBatch(t["reader"], Q, sc, limit, offs, **kw)
        for i, (q, w) in enumerate(zip(queries, wants)):
            (segs, docs, scores), total = got[i]
            (rs, rd, rsc), rt = par.scan(t["docs"], _clauses(q), w, t["norms"], _consts(t, q, sc),
                                         0 if offs is None else int(offs[i]), limit)
            assert total == rt and np.array_equal(segs, rs) and np.array_equal(docs, rd), q
            assert np.array_equal(scores.view(np.uint32), rsc.view(np.uint32)), q
    return counts


# ---------------------------------------------------------------- the passes
@pytest.mark.parametrize("scorer", SCORERS, ids=SCORER_IDS)
def test_every_pass_every_scorer(pa, scorer):
    rng = np.random.default_rng(3)
    counts = _check(pa, _queries(pa, rng, 12), scorer, k=15)
    assert int(np.count_nonzero(counts[:12])) >= 8


def test_pruning_levels_large_k_and_ties(pa):
    rng = np.random.default_rng(4)
    qs = _queries(pa, rng, 8)
    counts = _check(pa, qs, sdb.BM25(), k=4096, levels=(0, 1, 2), passes=False)
    assert counts.min() < 4096 < counts.max()             # k above some match counts, below others
    for k in (1, 2, 3, 7):                                # ties at the cut: equal (freqs, length) give equal scores
        _check(pa, qs[:6], sdb.BM25(), k=k, levels=(0, 2), passes=False)
    hits, n_out, total = sdb.ExecutePhraseAndTopKBatch(pa["reader"], [q[0] for q in qs], sdb.BM25(), 4096,
                                                       exclude_phrases=[q[1] for q in qs])
    assert total.tolist() == counts.tolist() and n_out.tolist() == np.minimum(counts, 4096).tolist()


def test_missing_terms_per_segment(pa):
    """Segment 1 lacks term 11 (a positive clause with it matches nothing there) and segment 2 lacks term 10 (a negated
    clause with it excludes nothing there)."""
    qs = [([[11], [0]], []), ([[0, 1]], [[10]]), ([[0, 1]], [[10, 0]]), ([[0]], [[11, 1]])]
    _check(pa, qs, sdb.BM25(), k=50)
    alone = par.matches(pa["docs"], [([0, 1], None, False)], (), pa["deleted"])
    assert _want(pa, qs[1])[2][0].tolist() == alone[2][0].tolist() and _want(pa, qs[2])[2][0].tolist() == alone[2][0].tolist()
    assert _want(pa, qs[0])[1][0].size == 0 and par.count(_want(pa, qs[0])) > 0


@pytest.mark.parametrize("n_preds", [1, 2, 3, 4])
def test_filter_chains_and_exclusions(pa, n_preds):
    rng = np.random.default_rng(20 + n_preds)
    chain = [(FILT, "LT", 35), (I32, "GT", -500), (F64, "LE", 60.0), (KEY, "NE", 3)][:n_preds]
    filt = [sdb.pred(f, op, v) for f, op, v in chain]
    masks = [np.logical_and.reduce([cr.pred_mask(c[f][0], c[f][1], op, v) for f, op, v in chain]) for c in pa["cols"]]
    qs = _queries(pa, rng, 9)
    excl = [[int(rng.integers(4, 11))] if i % 2 else [] for i in range(len(qs))]
    _check(pa, qs, sdb.BM25(), k=20, excl=excl, filt=filt, masks=masks)


def test_sixteen_slots(pa):
    rng = np.random.default_rng(6)
    qs = []
    for _ in range(6):
        ph, seq = _cut(pa, rng, 7)
        qs.append(([ph, [int(seq[0])], (ph[:2] + [ph[4]], [0, 1, 4])], [_cut(pa, rng, 5)[0]]))   # 7 + 1 + 3 + 5
    assert all(sum(len(c[0]) for c in _clauses(q)) == 16 for q in qs)
    counts = _check(pa, qs, sdb.BM25(), k=10)
    assert counts.max() > 0
    with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
        sdb.ExecutePhraseAndCountBatch(pa["reader"], [qs[0][0] + [[0]]], exclude_phrases=[qs[0][1]])


def test_batch_of_4096(pa):
    rng = np.random.default_rng(7)
    base = _queries(pa, rng, 6)
    qs = [base[i % len(base)] for i in range(4096)]
    counts = sdb.ExecutePhraseAndCountBatch(pa["reader"], [q[0] for q in qs], exclude_phrases=[q[1] for q in qs])
    ref = [par.count(_want(pa, q)) for q in base]
    assert counts.tolist() == [ref[i % len(base)] for i in range(4096)]


# ---------------------------------------------------------------- the identities
def test_identity_one_positive_clause_is_the_phrase(pa):
    r = pa["reader"]
    rng = np.random.default_rng(8)
    phrases = [_cut(pa, rng, L)[0] for L in (1, 2, 3, 5) for _ in range(3)] + [[0, 11], [0, 0]]
    excl = [[int(rng.integers(4, 11))] if i % 2 else [] for i in range(len(phrases))]
    Q = [[p] for p in phrases]
    for lv in (0, 2):
        ctx().set_wand(lv)
        for sc in (sdb.BM25(), sdb.TFIDF(True)):
            a = sdb.ExecutePhraseAndTopKBatch(r, Q, sc, 30, exclude=excl)
            b = sdb.ExecutePhraseTopKBatch(r, phrases, sc, 30, exclude=excl)
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    ctx().set_wand(False)
    assert np.array_equal(sdb.ExecutePhraseAndCountBatch(r, Q, exclude=excl), sdb.ExecutePhraseCountBatch(r, phrases, exclude=excl))
    a = sdb.ExecutePhraseAndTopKByColumnBatch(r, Q, I32, 40, False, True, exclude=excl)
    b = sdb.ExecutePhraseTopKByColumnBatch(r, phrases, I32, 40, False, True, exclude=excl)
    _same_sorted(a, b)
    a = sdb.ExecutePhraseAndFacetCountsBatch(r, Q, KEY, -5, 25, exclude=excl)
    b = sdb.ExecutePhraseFacetCountsBatch(r, phrases, KEY, -5, 25, exclude=excl)
    assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["nulls"], b["nulls"])
    a = sdb.ExecutePhraseAndMatchAggregatesBatch(r, Q, F64, KEY, -5, 25, exclude=excl)
    b = sdb.ExecutePhraseMatchAggregatesBatch(r, phrases, F64, KEY, -5, 25, exclude=excl)
    for f in ("count", "count_value", "min", "max"):   # a float64 SUM is added in atomic order: equal up to rounding
        assert np.array_equal(np.asarray(a[f]).view(np.uint64), np.asarray(b[f]).view(np.uint64)), f
    assert np.allclose(np.asarray(a["sum"], np.float64), np.asarray(b["sum"], np.float64), rtol=1e-12, atol=1e-9)
    a = sdb.ExecutePhraseAndMatchScanBatch(r, Q, sdb.BM25(), 1 << 13, exclude=excl)
    b = sdb.ExecutePhraseMatchScanBatch(r, phrases, sdb.BM25(), 1 << 13, exclude=excl)
    for ((sa, da, xa), ta), ((sb, db, xb), tb) in zip(a, b):
        assert ta == tb and np.array_equal(sa, sb) and np.array_equal(da, db) and np.array_equal(xa.view(np.uint32), xb.view(np.uint32))


def test_identity_one_slot_clauses_are_the_flat_and(pa):
    r = pa["reader"]
    qs = [[0, 1], [2, 0], [1, 3, 0], [4, 0, 2, 1], [5], [0, 11], [6, 1]]
    excl = [[], [7], [], [8, 9], [], [], [3]]
    Q = [[[t] for t in q] for q in qs]
    ctx().set_wand(0)
    for sc in SCORERS:
        a = sdb.ExecutePhraseAndTopKBatch(r, Q, sc, 100, exclude=excl)
        b = sdb.ExecuteTopKBatch(r, qs, sdb.AND, sc, 100, exclude=excl)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
        for i in range(len(qs)):
            h1, h2 = a[0][i, :a[1][i]], b[0][i, :b[1][i]]
            assert np.array_equal(h1["doc"], h2["doc"]) and np.array_equal(h1["seg"], h2["seg"]), qs[i]
            assert np.array_equal(h1["score"].view(np.uint32), h2["score"].view(np.uint32)), qs[i]
    ctx().set_wand(False)
    assert np.array_equal(sdb.ExecutePhraseAndCountBatch(r, Q, exclude=excl), sdb.ExecuteCountBatch(r, qs, sdb.AND, exclude=excl))
    a = sdb.ExecutePhraseAndTopKByColumnBatch(r, Q, I32, 40, True, True, exclude=excl)
    b = sdb.ExecuteTopKByColumnBatch(r, qs, sdb.AND, I32, 40, True, True, exclude=excl)
    _same_sorted(a, b)
    a = sdb.ExecutePhraseAndFacetCountsBatch(r, Q, KEY, -5, 25, exclude=excl)
    b = sdb.ExecuteFacetCountsBatch(r, qs, sdb.AND, KEY, -5, 25, exclude=excl)
    assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["nulls"], b["nulls"])
    a = sdb.ExecutePhraseAndMatchAggregatesBatch(r, Q, F64, KEY, -5, 25, exclude=excl)
    b = sdb.ExecuteMatchAggregatesBatch(r, qs, sdb.AND, F64, KEY, -5, 25, exclude=excl)
    for f in ("count", "count_value", "min", "max"):
        assert np.array_equal(np.asarray(a[f]).view(np.uint64), np.asarray(b[f]).view(np.uint64)), f
    for sc in (sdb.BM25(), sdb.TFIDF(False)):
        a = sdb.ExecutePhraseAndMatchScanBatch(r, Q, sc, 1 << 13, exclude=excl)
        b = sdb.ExecuteMatchScanBatch(r, qs, sdb.AND, sc, limit=1 << 13, exclude=excl)
        for ((sa, da, xa), ta), ((sb, db, xb), tb) in zip(a, b):
            assert ta == tb and np.array_equal(sa, sb) and np.array_equal(da, db)
            assert np.array_equal(xa.view(np.uint32), xb.view(np.uint32))


# ---------------------------------------------------------------- doc ids past 2^31
def test_doc_ids_past_2_31():
    n = (1 << 32) - 2
    rng = np.random.default_rng(41)
    top = np.sort(rng.choice(np.arange(n - 5_000_000, n + 1, dtype=np.int64), 3000, replace=False)).astype(np.uint32)
    low = np.sort(rng.choice(np.arange(1, 1 << 20), 500, replace=False)).astype(np.uint32)
    a = np.unique(np.concatenate([low, top, [1 << 31, (1 << 31) + 1, n]])).astype(np.uint32)
    b = np.unique(np.concatenate([a[rng.random(len(a)) < 0.6], [1 << 31, n]])).astype(np.uint32)
    c = np.unique(np.concatenate([a[rng.random(len(a)) < 0.3], [n]])).astype(np.uint32)
    fa = rng.integers(1, 4, len(a)).astype(np.uint32)
    posts = [(a, fa, np.concatenate([np.arange(0, 2 * int(x), 2, dtype=np.uint32) for x in fa])),
             (b, np.ones(len(b), np.uint32), (2 * rng.integers(0, 3, len(b)) + 1).astype(np.uint32)),
             (c, np.ones(len(c), np.uint32), (2 * rng.integers(0, 3, len(c))).astype(np.uint32))]
    oseg = orc.Segment(n, has_wand=True)
    for d, f, _ in posts:
        oseg.add_term(d, f)
    g = to_gpu(oseg)
    g.stage_positions(*pr.staged_positions(posts))
    dels = [n, int(top[5])]
    g.stage_docs_mask(np.array(dels, np.uint32))
    reader = sdb.IndexReader([g], n, n, [len(a), len(b), len(c)])
    qs = [([[0, 1], [2]], []), ([[0], [1]], [[2, 1]]), ([[0, 1]], [[1, 0]]), ([[0, 0], [1]], [[2]])]
    sc = sdb.BM25()
    counts = sdb.ExecutePhraseAndCountBatch(reader, [q[0] for q in qs], exclude_phrases=[q[1] for q in qs])
    hits, n_out, _ = sdb.ExecutePhraseAndTopKBatch(reader, [q[0] for q in qs], sc, 100, exclude_phrases=[q[1] for q in qs])
    high = 0
    for i, q in enumerate(qs):
        cl = _clauses(q)
        # match over postings: a doc's positions per term, then the clause frequencies
        by_term = []
        for d, f, pos in posts:
            ends = np.cumsum(f.astype(np.int64))
            by_term.append({int(x): set(pos[e - k:e].tolist()) for x, k, e in zip(d, f, ends)})
        ds, fs = [], []
        for doc in sorted(set(by_term[0]) | set(by_term[1]) | set(by_term[2])):
            if doc in dels:
                continue
            fr = []
            for terms, rel, _ in cl:
                rel = list(range(len(terms))) if rel is None else rel
                anchors = by_term[terms[0]].get(doc, set())
                fr.append(sum(1 for p in anchors if all(p + r in by_term[t].get(doc, set()) for t, r in zip(terms, rel))))
            if all((x > 0) != neg for x, (_, _, neg) in zip(fr, cl)):
                ds.append(doc); fs.append(fr)
        assert counts[i] == len(ds), q
        dc = [len(p[0]) for p in posts]
        order = sorted([j for j in range(len(cl)) if not cl[j][2]], key=lambda j: min(dc[t] for t in cl[j][0]))
        consts = [None if neg else pr.consts(reader.phrase_stats(sc, terms), sc.k, sc.b) for terms, _, neg in cl]
        rows = []
        for d, fr in zip(ds, fs):
            s = np.float32(0)
            for j in order:
                s = np.float32(s + pr.score(fr[j], 1, *consts[j]))
            rows.append((s, d))
        rows.sort(key=lambda x: (-x[0], x[1]))
        got = hits[i, :n_out[i]]
        assert got["doc"].tolist() == [d for _, d in rows[:100]], q
        assert got["score"].view(np.uint32).tolist() == np.array([s for s, _ in rows[:100]], np.float32).view(np.uint32).tolist()
        high += sum(1 for d in ds if d > (1 << 31))
        (_, docs, _), total = sdb.ExecutePhraseAndMatchScan(reader, q[0], None, 1 << 14, exclude_phrases=q[1])
        assert total == len(ds) and docs.tolist() == ds
    assert high > 0


# ---------------------------------------------------------------- errors
def _rc(t, terms, clause_off, qoff, neg=None, rel=None, excl=None, excl_off=None):
    arr = lambda a, dt: None if a is None else np.ascontiguousarray(a, dt)
    terms, clause_off, qoff, neg, rel = arr(terms, np.uint32), arr(clause_off, np.uint32), arr(qoff, np.uint32), arr(neg, np.uint8), arr(rel, np.uint32)
    nq = len(qoff) - 1 if qoff is not None else 1
    counts = np.zeros(max(nq, 1), np.uint64)
    segs = (C.c_void_p * len(t["segs"]))(*[s._h.value for s in t["segs"]])
    p = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    return N.lib().sdbg_phrase_and_count_batch(segs, len(t["segs"]), p(terms), p(rel), p(clause_off), p(neg), p(qoff), nq,
                                               p(excl), p(excl_off), None, p(counts))


def test_errors_then_a_valid_call(pa):
    inval, unsup, notfound = -1, -7, -5
    launches = ctx().launches
    assert _rc(pa, [0, 1], [0, 0, 2], [0, 2]) == inval                       # an empty clause
    assert _rc(pa, [0, 1], [0, 2], [0, 0, 1]) == inval                       # a query without a clause
    assert _rc(pa, [0, 1], [0, 1, 2], [0, 2], neg=[1, 1]) == inval           # a query without a positive clause
    assert _rc(pa, [0, 1], [0, 2], [0, 1], rel=[1, 2]) == inval              # rel_pos not starting at 0
    assert _rc(pa, [0, 1, 2], [0, 2, 3], [0, 2], rel=[0, 0, 0]) == inval     # rel_pos not increasing
    assert _rc(pa, [0, 1], [0, 2, 1], [0, 2]) == inval                       # decreasing clause offsets
    assert _rc(pa, [0, 1], [0, 1, 2], [0, 2, 1]) == inval                    # decreasing query offsets
    assert _rc(pa, None, [0, 2], [0, 1]) == inval                            # NULL terms
    assert _rc(pa, [0, 1], None, [0, 1]) == inval                            # NULL clause_off
    assert _rc(pa, [0, 1], [0, 2], None) == inval                            # NULL query_clause_off
    assert _rc(pa, [0, 99], [0, 2], [0, 1]) == inval                         # a positive term id out of range
    assert _rc(pa, list(range(9)) * 2, [0, 9, 18], [0, 2], neg=[0, 1]) == unsup   # 18 slots, 9 of them negated
    assert _rc(pa, [0], [0, 1], [0, 1], excl=np.arange(17, dtype=np.uint32) % V, excl_off=np.array([0, 17], np.uint32)) == unsup
    # NULL clause_stats in a top-k and in a scored scan; k > 4096
    segs = (C.c_void_p * 3)(*[s._h.value for s in pa["segs"]])
    terms, coff, qoff = np.array([0, 1], np.uint32), np.array([0, 2], np.uint32), np.array([0, 1], np.uint32)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    hits, n_out, total = np.zeros(5000, sdb.engine.HIT_DTYPE), np.zeros(1, np.uint32), np.zeros(1, np.uint64)
    assert N.lib().sdbg_phrase_and_topk_batch(segs, 3, p(terms), None, p(coff), None, p(qoff), 1, None, None, None, 1.2, 0.75,
                                              None, 10, 0.0, p(hits), p(n_out), p(total)) == inval
    assert N.lib().sdbg_phrase_and_scan_batch(segs, 3, p(terms), None, p(coff), None, p(qoff), 1, None, None, None, None, 1.2,
                                              0.75, None, 10, 1, p(hits), p(n_out), p(total)) == inval
    st = (N.BM25Term * 1)(pa["reader"].phrase_stats(sdb.BM25(), [0, 1]))
    assert N.lib().sdbg_phrase_and_topk_batch(segs, 3, p(terms), None, p(coff), None, p(qoff), 1, None, None, st, 1.2, 0.75,
                                              None, 4097, 0.0, p(hits), p(n_out), p(total)) == unsup
    assert ctx().launches == launches                                        # nothing was queued
    # a segment without positions
    oseg = orc.Segment(100, has_wand=True)
    oseg.add_term(np.array([1, 2], np.uint32), np.array([1, 1], np.uint32))
    g = to_gpu(oseg, columns={I32: (np.arange(100, dtype=np.int32), None)})
    r2 = sdb.IndexReader([g], 100, 100, [2])
    for call in (lambda: sdb.ExecutePhraseAndCountBatch(r2, [[[0]]]),
                 lambda: sdb.ExecutePhraseAndTopKBatch(r2, [[[0]]], sdb.BM25(), 5),
                 lambda: sdb.ExecutePhraseAndTopKByColumnBatch(r2, [[[0]]], I32, 5),
                 lambda: sdb.ExecutePhraseAndFacetCountsBatch(r2, [[[0]]], I32, 0, 100),
                 lambda: sdb.ExecutePhraseAndMatchAggregatesBatch(r2, [[[0]]], I32),
                 lambda: sdb.ExecutePhraseAndMatchScanBatch(r2, [[[0]]])):
        with pytest.raises(N.SdbgError, match="ENOTFOUND"):
            call()
    # the same context serves valid calls afterwards
    _check(pa, _queries(pa, np.random.default_rng(9), 4), sdb.BM25(), k=10)


# ---------------------------------------------------------------- adapters
def _selftest_corpus(n_docs):
    """The token corpus of adapter_selftest's "phrase" modes, rebuilt from its generator."""
    state, docs = 12345, []

    def nxt():
        nonlocal state
        state = (state * 1664525 + 1013904223) & 0xFFFFFFFF
        return state >> 16
    for _ in range(n_docs):
        n = 1 + nxt() % 16
        docs.append([nxt() % 6 for _ in range(n)])
    return docs


def test_adapters_phrase_and_mode():
    """All six phrase adapters with clause_sizes / clause_negated against the reference; each positive clause scored
    with its statistics computed here by hand: its slots' BM25 idfs summed in float32, the first slot's norm constants."""
    import json
    import subprocess
    from serenedb_b200 import build as b

    exe = b.build_adapters()
    n = 20_000
    res = subprocess.run([exe, str(n), "phrase", "and"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = [json.loads(l) for l in res.stdout.strip().splitlines()]
    assert len(lines) == 3
    docs = _selftest_corpus(n)
    norms = np.array([len(d) for d in docs], np.uint32)
    post = pr.postings(docs, 6)
    sc = sdb.BM25()
    d = np.arange(1, n + 1, dtype=np.int64)
    cols = [((d * 7919) % 23 - 11, d % 5 != 0)]
    for x in lines:
        off = np.concatenate([[0], np.cumsum(x["sizes"])])
        cl = [(x["slots"][off[j]:off[j + 1]], x["rel"][off[j]:off[j + 1]], bool(x["neg"][j])) for j in range(len(x["sizes"]))]
        consts = []
        for terms, _, neg in cl:
            idf = np.float32(0)
            for t in terms:
                idf = np.float32(idf + np.float32(sc.collect(n, int(norms.sum()), len(post[t][0])).idf))
            st = sc.collect(n, int(norms.sum()), len(post[terms[0]][0]))
            c0 = np.float32(np.float32(np.float32(1.0) * np.float32(np.float32(1.2) + np.float32(1))) * idf)
            consts.append(None if neg else (c0, np.float32(st.norm_const), np.float32(st.norm_length)))
        w = par.matches([docs], cl, x["excl"])
        n_match = par.count(w)
        assert x["count"] == x["total"] == x["scan_total"] == n_match > 0, x["slots"]
        ref, _ = par.topk([docs], cl, w, [norms], consts, 50)
        assert [h[0] for h in x["topk"]] == ref["doc"].tolist(), x["slots"]
        assert np.array_equal(np.array([h[1] for h in x["topk"]], np.float32).view(np.uint32), ref["score"].view(np.uint32))
        assert x["sorted_docs"] == par.sorted_hits(w, cols, True, False, 30)["docs"].tolist()
        counts, nulls = par.facet_counts(w, cols, -11, 23)
        assert x["facet_keys"] == [k - 11 for k in np.nonzero(counts)[0].tolist()] + ([0] if nulls else [])
        assert x["facet_counts"] == counts[counts > 0].tolist() + ([nulls] if nulls else [])
        assert x["agg_count"] == [n_match]
        (_, rd, rsc), _ = par.scan([docs], cl, w, [norms], consts)
        assert x["scan_docs"] == rd.tolist()
        assert np.array_equal(np.array(x["scan_scores"], np.float32).view(np.uint32), rsc.view(np.uint32))


def test_three_clauses_with_a_cost_tie():
    """Terms 0..3 occur in the same docs, so the clauses "0 1" and "2 3" tie in cost behind the cheaper term 4: their
    order, the query's, decides the fp32 sum's last bits, which the two query orders below show."""
    rng = np.random.default_rng(61)
    n = 3000
    docs = []
    for _ in range(n):
        if rng.random() < 0.5:
            seq = rng.permutation(4).tolist() + rng.choice([0, 1, 2, 3, 5], int(rng.integers(0, 12))).tolist()
        else:
            seq = [5] * int(rng.integers(1, 8))
        if rng.random() < 0.4:
            seq.insert(int(rng.integers(0, len(seq) + 1)), 4)
        docs.append(seq)
    post = pr.postings(docs, 6)
    oseg = orc.Segment(n, has_wand=True)
    norms = np.array([len(d) for d in docs], np.uint32)
    oseg.set_norms(norms)
    for d, f, _ in post:
        oseg.add_term(d, f)
    g = to_gpu(oseg)
    g.stage_positions(*pr.staged_positions(post))
    reader = sdb.IndexReader([g], n, int(norms.sum()), [len(p[0]) for p in post])
    sc = sdb.BM25()
    qs = [[[0, 1], [2, 3], [4]], [[2, 3], [0, 1], [4]], [[1, 0], [3, 2], [4]], [[3, 2], [1, 0], [4]]]
    hits, n_out, total = sdb.ExecutePhraseAndTopKBatch(reader, qs, sc, 4096)
    scans = sdb.ExecutePhraseAndMatchScanBatch(reader, qs, sc, 1 << 13)
    by_doc = []
    for i, q in enumerate(qs):
        cl = [(c, None, False) for c in q]
        consts = [pr.consts(reader.phrase_stats(sc, c), sc.k, sc.b) for c in q]
        w = par.matches([docs], cl)
        assert par.cost_order(docs, cl)[0] == 2 and total[i] == par.count(w) > 0
        ref, _ = par.topk([docs], cl, w, [norms], consts, 4096)
        got = hits[i, :n_out[i]]
        assert np.array_equal(got["doc"], ref["doc"]) and np.array_equal(got["score"].view(np.uint32), ref["score"].view(np.uint32))
        (_, rd, rsc), _ = par.scan([docs], cl, w, [norms], consts)
        (_, sd, ss), _ = scans[i]
        assert np.array_equal(sd, rd) and np.array_equal(ss.view(np.uint32), rsc.view(np.uint32))
        by_doc.append(dict(zip(rd.tolist(), rsc.view(np.uint32).tolist())))
    # the tie order matters here: the same clauses in the other query order give other bits for some docs
    assert any(by_doc[0][d] != by_doc[1][d] for d in by_doc[0]) or any(by_doc[2][d] != by_doc[3][d] for d in by_doc[2])
