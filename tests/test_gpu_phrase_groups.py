"""Conjunctions of OR groups of phrases and terms on the GPU (sdbg_phrase_groups_{count,topk,topk_by_column,
facet_counts,aggregate,scan}_batch) against the NumPy statement (tests/phrase_groups_reference.py), bit for bit: counts,
hits (doc, segment, order, fp32 score bits), sorted hits, facet and aggregate cells, scan pages and totals. Over
token-sequence segments where one lacks a term of a positive alternative and one a term of a negated one, with deleted
docs, filter chains of 1..4 predicates, exclusions, every scorer, pruning levels 0..2, k above the match count and ties
at the cut, exactly 16 slots and 16 groups, a batch of 4096 mixing the three candidate shapes, proxy collisions, doc ids
past 2^31; the three identities (groups of one alternative: the clause conjunction entries; one-slot alternatives of
distinct terms: the OR-group entries; one group of them: the flat OR entries); the error codes."""
import ctypes as C

import numpy as np
import pytest

import count_reference as cr
import orc
import phrase_groups_reference as pgr
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
def pg():
    rng = np.random.default_rng(778)
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


def _other(t, rng):
    """A token of another doc."""
    seq = t["docs"][int(rng.integers(0, 3))][int(rng.integers(0, 2500))]
    return int(seq[int(rng.integers(0, len(seq)))])


def _queries(t, rng, n):
    """(groups, negated alternatives) per query: `("w1 w2" | s) & t`, `"w1 w2" | s`, `("w1 w2" | s) & t & !"w3 w4"`,
    two phrase groups, and a group with a gapped phrase; plus queries on the missing terms and proxy collisions."""
    qs = []
    for i in range(n):
        ph, seq = _cut(t, rng, 2 + i % 2)
        term = [int(seq[int(rng.integers(0, len(seq)))])]
        s = [_other(t, rng)]
        kind = i % 5
        if kind == 0:
            qs.append(([[ph, s], [term]], []))
        elif kind == 1:
            qs.append(([[ph, s]], []))
        elif kind == 2:
            qs.append(([[ph, s], [term]], [_cut(t, rng, 2)[0]]))
        elif kind == 3:
            qs.append(([[ph, s], [_cut(t, rng, 2)[0], term]], [[int(rng.integers(3, 10))]]))
        else:
            qs.append(([[(ph[:1] + [int(rng.integers(0, 4))], [0, 2]), ph], [term, s]], []))
    qs += [([[[0, 1], [11]], [[2]]], []), ([[[0, 1], [10, 2]]], [[10, 0]]), ([[[11, 0], [1]]], [[1, 2]]),
           ([[[0, 1]], [[0, 2], [3]]], []),                  # "0 1" & ("0 2" | 3): the proxy of "0 2" must avoid 0
           ([[[0]], [[0], [1]]], []),                        # 0 & (0 | 1): the group repeats 0, left out of the candidates
           ([[[0, 0], [1]], [[1, 0], [1]]], [[2, 3]])]       # repeated terms, duplicate alternatives
    return qs


def _groups(q):
    pos, neg = q
    alt = lambda x: (list(x[0]), list(x[1])) if isinstance(x, tuple) else (list(x), None)
    return [([alt(a) for a in g], False) for g in pos] + [([alt(a)], True) for a in neg]


def _consts(t, q, scorer):
    return [None if n else pr.consts(t["reader"].phrase_stats(scorer, terms), scorer.k, scorer.b)
            for terms, _, n in pgr.flat(_groups(q))]


def _same_sorted(a, b):
    assert np.array_equal(a["n_out"], b["n_out"])
    for f in ("docs", "segs", "values", "nulls"):
        assert all(np.array_equal(x, y) for x, y in zip(a[f], b[f])), f


def _want(t, q, excl=(), masks=None):
    return pgr.matches(t["docs"], _groups(q), excl, t["deleted"], masks)


def _col(t, f):
    return [c[f] for c in t["cols"]]


def _check(t, queries, scorer=None, k=10, excl=None, filt=None, masks=None, levels=(0,), passes=True):
    excl = excl or [[]] * len(queries)
    Q, X = [q[0] for q in queries], [q[1] for q in queries]
    kw = dict(filt=filt, exclude=excl, exclude_phrases=X)
    wants = [_want(t, q, x, masks) for q, x in zip(queries, excl)]
    counts = sdb.ExecutePhraseGroupsCountBatch(t["reader"], Q, **kw)
    assert counts.tolist() == [pgr.count(w) for w in wants]
    if scorer is not None:
        for lv in levels:
            ctx().set_wand(lv)
            hits, n_out, total = sdb.ExecutePhraseGroupsTopKBatch(t["reader"], Q, scorer, k, **kw)
            assert np.array_equal(total, counts)
            for i, (q, w) in enumerate(zip(queries, wants)):
                ref, _ = pgr.topk(t["docs"], _groups(q), w, t["norms"], _consts(t, q, scorer), k)
                got = hits[i, :n_out[i]]
                assert len(got) == len(ref), (q, lv)
                assert np.array_equal(got["doc"], ref["doc"]) and np.array_equal(got["seg"], ref["seg"]), (q, lv)
                assert np.array_equal(got["score"].view(np.uint32), ref["score"].view(np.uint32)), (q, lv)
            ctx().set_wand(False)
    if not passes:
        return counts
    got = sdb.ExecutePhraseGroupsTopKByColumnBatch(t["reader"], Q, I32, k, True, False, **kw)
    for i, w in enumerate(wants):
        ref = pgr.sorted_hits(w, _col(t, I32), True, False, k)
        assert np.array_equal(got["docs"][i], ref["docs"]) and np.array_equal(got["segs"][i], ref["segs"]), queries[i]
        assert np.array_equal(got["values"][i], ref["values"]) and np.array_equal(got["nulls"][i], ref["nulls"])
    got = sdb.ExecutePhraseGroupsFacetCountsBatch(t["reader"], Q, KEY, -5, 25, **kw)
    for i, w in enumerate(wants):
        c, nulls = pgr.facet_counts(w, _col(t, KEY), -5, 25)
        assert got["counts"][i].tolist() == c.tolist() and int(got["nulls"][i]) == nulls, queries[i]
    got = sdb.ExecutePhraseGroupsMatchAggregatesBatch(t["reader"], Q, I32, KEY, -5, 25, **kw)
    for i, w in enumerate(wants):
        cells, null_cell = pgr.aggregate(w, _col(t, KEY), _col(t, I32), -5, 25)
        for j, cell in enumerate(cells):
            assert int(got["count"][i][j]) == cell["count"] and int(got["count_value"][i][j]) == cell["count_value"]
            if cell["count_value"]:
                assert int(got["sum"][i][j]) == cell["sum"] and int(got["min"][i][j]) == cell["min"]
                assert int(got["max"][i][j]) == cell["max"]
        assert int(got["null"]["count"][i]) == null_cell["count"]
    sc = scorer or sdb.BM25()
    for offs, limit in ((None, 1 << 14), (np.array([c // 2 for c in counts], np.uint64), 7)):
        got = sdb.ExecutePhraseGroupsMatchScanBatch(t["reader"], Q, sc, limit, offs, **kw)
        for i, (q, w) in enumerate(zip(queries, wants)):
            (segs, docs, scores), total = got[i]
            (rs, rd, rsc), rt = pgr.scan(t["docs"], _groups(q), w, t["norms"], _consts(t, q, sc),
                                         0 if offs is None else int(offs[i]), limit)
            assert total == rt and np.array_equal(segs, rs) and np.array_equal(docs, rd), q
            assert np.array_equal(scores.view(np.uint32), rsc.view(np.uint32)), q
    return counts


# ---------------------------------------------------------------- the passes
@pytest.mark.parametrize("scorer", SCORERS, ids=SCORER_IDS)
def test_every_pass_every_scorer(pg, scorer):
    rng = np.random.default_rng(3)
    counts = _check(pg, _queries(pg, rng, 15), scorer, k=15)
    assert int(np.count_nonzero(counts[:15])) >= 10


def test_pruning_levels_large_k_and_ties(pg):
    rng = np.random.default_rng(4)
    qs = _queries(pg, rng, 10)
    counts = _check(pg, qs, sdb.BM25(), k=4096, levels=(0, 1, 2), passes=False)
    assert counts.min() < 4096 < counts.max()
    for k in (1, 2, 3, 7):
        _check(pg, qs[:8], sdb.BM25(), k=k, levels=(0, 2), passes=False)


def test_missing_terms_per_segment(pg):
    """Segment 1 lacks term 11 (a positive alternative with it matches nothing there, and a group of such alternatives
    nothing at all) and segment 2 lacks term 10 (a negated alternative with it excludes nothing there)."""
    qs = [([[[11], [0, 1]], [[2]]], []), ([[[11]], [[0]]], []), ([[[0, 1], [2]]], [[10]]), ([[[0, 1], [3]]], [[10, 0]])]
    _check(pg, qs, sdb.BM25(), k=50)
    assert _want(pg, qs[1])[1][0].size == 0 and pgr.count(_want(pg, qs[1])) > 0


@pytest.mark.parametrize("n_preds", [1, 2, 3, 4])
def test_filter_chains_and_exclusions(pg, n_preds):
    rng = np.random.default_rng(20 + n_preds)
    chain = [(FILT, "LT", 35), (I32, "GT", -500), (F64, "LE", 60.0), (KEY, "NE", 3)][:n_preds]
    filt = [sdb.pred(f, op, v) for f, op, v in chain]
    masks = [np.logical_and.reduce([cr.pred_mask(c[f][0], c[f][1], op, v) for f, op, v in chain]) for c in pg["cols"]]
    qs = _queries(pg, rng, 10)
    excl = [[int(rng.integers(4, 11))] if i % 2 else [] for i in range(len(qs))]
    _check(pg, qs, sdb.BM25(), k=20, excl=excl, filt=filt, masks=masks)


def test_sixteen_slots_and_sixteen_groups(pg):
    rng = np.random.default_rng(6)
    qs = []
    for _ in range(4):
        ph, seq = _cut(pg, rng, 5)
        qs.append(([[ph, [int(seq[0])]], [(ph[:2] + [ph[4]], [0, 1, 4]), [_other(pg, rng)]], [_cut(pg, rng, 3)[0]]],
                   [_cut(pg, rng, 3)[0]]))                                       # 5 + 1 + 3 + 1 + 3 + 3
    assert all(sum(len(a[0]) for a in pgr.flat(_groups(q))) == 16 for q in qs)
    qs.append(([[[t]] for t in (0, 1, 2, 3)], [[t] for t in range(4, 16)]))   # 16 groups of one slot, ids past V negated
    assert len(_groups(qs[-1])) == 16
    counts = _check(pg, qs, sdb.BM25(), k=10)
    assert counts[:4].max() > 0
    with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
        sdb.ExecutePhraseGroupsCountBatch(pg["reader"], [qs[0][0] + [[[0]]]], exclude_phrases=[qs[0][1]])
    with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
        sdb.ExecutePhraseGroupsCountBatch(pg["reader"], [[[[t % V]] for t in range(17)]])


def test_batch_of_4096_mixes_the_candidate_shapes(pg):
    """Groups of one alternative (the AND), one group (the flat OR) and several groups, in one batch of 4096 whose
    results are scattered back to the queries' places."""
    rng = np.random.default_rng(7)
    base = _queries(pg, rng, 10) + [([[_cut(pg, rng, 2)[0]], [[1]]], [])]
    qs = [base[(i * 7) % len(base)] for i in range(4096)]
    Q, X = [q[0] for q in qs], [q[1] for q in qs]
    counts = sdb.ExecutePhraseGroupsCountBatch(pg["reader"], Q, exclude_phrases=X)
    ref = [pgr.count(_want(pg, q)) for q in base]
    assert counts.tolist() == [ref[(i * 7) % len(base)] for i in range(4096)]
    sc = sdb.BM25()
    hits, n_out, total = sdb.ExecutePhraseGroupsTopKBatch(pg["reader"], Q, sc, 5, exclude_phrases=X)
    assert np.array_equal(total, counts)
    for i in range(0, 4096, 97):
        q = qs[i]
        r, _ = pgr.topk(pg["docs"], _groups(q), _want(pg, q), pg["norms"], _consts(pg, q, sc), 5)
        got = hits[i, :n_out[i]]
        assert np.array_equal(got["doc"], r["doc"]) and np.array_equal(got["score"].view(np.uint32), r["score"].view(np.uint32))
    f = sdb.ExecutePhraseGroupsFacetCountsBatch(pg["reader"], Q, KEY, -5, 25, exclude_phrases=X)
    scans = sdb.ExecutePhraseGroupsMatchScanBatch(pg["reader"], Q, None, 3, exclude_phrases=X)
    for i in range(0, 4096, 131):
        w = _want(pg, qs[i])
        c, nulls = pgr.facet_counts(w, _col(pg, KEY), -5, 25)
        assert f["counts"][i].tolist() == c.tolist() and int(f["nulls"][i]) == nulls
        (rs, rd, _), rt = pgr.scan(pg["docs"], _groups(qs[i]), w, limit=3)
        (ss, sd, _), st = scans[i]
        assert st == rt and np.array_equal(sd, rd) and np.array_equal(ss, rs)


def test_proxy_collisions(pg):
    """`"0 1" & ("0 2" | 3)`: the phrase's proxy avoids the used 0; `0 & (0 | 1)`: the group cannot avoid 0 and is checked
    per doc only; `("0 1" | 0) & ("1 0" | 1)`: the second group's phrase finds no unused term."""
    qs = [([[[0, 1]], [[0, 2], [3]]], []), ([[[0]], [[0], [1]]], []), ([[[0, 1], [0]], [[1, 0], [1]]], []),
          ([[[0, 1], [2]], [[0, 2], [1]], [[2, 1], [0]]], []), ([[[1, 2]], [[1, 2], [4]]], [[0]])]
    counts = _check(pg, qs, sdb.BM25(), k=30)
    assert counts.min() > 0


# ---------------------------------------------------------------- the identities
def test_identity_groups_of_one_alternative_are_the_clause_conjunction(pg):
    r = pg["reader"]
    rng = np.random.default_rng(8)
    clause_qs = [([_cut(pg, rng, 2)[0], [int(rng.integers(0, 6))]], [_cut(pg, rng, 2)[0]]) for _ in range(6)]
    clause_qs += [([[0, 11]], []), ([[0, 0], [1]], [[10]]), ([_cut(pg, rng, 3)[0]], [])]
    Q, X = [q[0] for q in clause_qs], [q[1] for q in clause_qs]
    G = [[[c] for c in q] for q in Q]
    excl = [[int(rng.integers(4, 11))] if i % 2 else [] for i in range(len(Q))]
    for lv in (0, 2):
        ctx().set_wand(lv)
        for sc in (sdb.BM25(), sdb.TFIDF(True)):
            a = sdb.ExecutePhraseGroupsTopKBatch(r, G, sc, 30, exclude=excl, exclude_phrases=X)
            b = sdb.ExecutePhraseAndTopKBatch(r, Q, sc, 30, exclude=excl, exclude_phrases=X)
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    ctx().set_wand(False)
    kw = dict(exclude=excl, exclude_phrases=X)
    assert np.array_equal(sdb.ExecutePhraseGroupsCountBatch(r, G, **kw), sdb.ExecutePhraseAndCountBatch(r, Q, **kw))
    _same_sorted(sdb.ExecutePhraseGroupsTopKByColumnBatch(r, G, I32, 40, False, True, **kw),
                 sdb.ExecutePhraseAndTopKByColumnBatch(r, Q, I32, 40, False, True, **kw))
    a = sdb.ExecutePhraseGroupsFacetCountsBatch(r, G, KEY, -5, 25, **kw)
    b = sdb.ExecutePhraseAndFacetCountsBatch(r, Q, KEY, -5, 25, **kw)
    assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["nulls"], b["nulls"])
    a = sdb.ExecutePhraseGroupsMatchAggregatesBatch(r, G, I32, KEY, -5, 25, **kw)
    b = sdb.ExecutePhraseAndMatchAggregatesBatch(r, Q, I32, KEY, -5, 25, **kw)
    for f in ("count", "count_value", "sum", "min", "max"):
        assert np.array_equal(np.asarray(a[f]), np.asarray(b[f])), f
    a = sdb.ExecutePhraseGroupsMatchScanBatch(r, G, sdb.BM25(), 1 << 13, **kw)
    b = sdb.ExecutePhraseAndMatchScanBatch(r, Q, sdb.BM25(), 1 << 13, **kw)
    for ((sa, da, xa), ta), ((sb, db, xb), tb) in zip(a, b):
        assert ta == tb and np.array_equal(sa, sb) and np.array_equal(da, db) and np.array_equal(xa.view(np.uint32), xb.view(np.uint32))


def test_identity_one_slot_alternatives_are_the_or_groups(pg):
    """Distinct one-slot alternatives: the *_groups(_min) entries with every minimum 1, bit for bit at pruning level 0;
    one group of them: the flat OR entries."""
    r = pg["reader"]
    gq = [[[0, 1], [2]], [[3], [1, 4, 0]], [[5, 2], [0, 6], [1]], [[0, 11], [2]], [[7, 8, 9]], [[0, 1, 2, 3]]]
    excl = [[], [7], [], [8, 9], [], [10]]
    G = [[[[t] for t in g] for g in q] for q in gq]
    ones = [[1] * len(q) for q in gq]
    ctx().set_wand(0)
    for sc in SCORERS:
        a = sdb.ExecutePhraseGroupsTopKBatch(r, G, sc, 100, exclude=excl)
        b = sdb.ExecuteTopKGroupsBatch(r, gq, sc, 100, exclude=excl, min_match=ones)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
        for i in range(len(gq)):
            h1, h2 = a[0][i, :a[1][i]], b[0][i, :b[1][i]]
            assert np.array_equal(h1["doc"], h2["doc"]) and np.array_equal(h1["seg"], h2["seg"]), gq[i]
            assert np.array_equal(h1["score"].view(np.uint32), h2["score"].view(np.uint32)), gq[i]
    ctx().set_wand(False)
    assert np.array_equal(sdb.ExecutePhraseGroupsCountBatch(r, G, exclude=excl), sdb.ExecuteCountGroupsBatch(r, gq, exclude=excl, min_match=ones))
    _same_sorted(sdb.ExecutePhraseGroupsTopKByColumnBatch(r, G, I32, 40, True, True, exclude=excl),
                 sdb.ExecuteTopKByColumnGroupsBatch(r, gq, I32, 40, True, True, exclude=excl, min_match=ones))
    a = sdb.ExecutePhraseGroupsFacetCountsBatch(r, G, KEY, -5, 25, exclude=excl)
    b = sdb.ExecuteFacetCountsGroupsBatch(r, gq, KEY, -5, 25, exclude=excl, min_match=ones)
    assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["nulls"], b["nulls"])
    for sc in (sdb.BM25(), sdb.TFIDF(False)):
        for ((sa, da, xa), ta), ((sb, db, xb), tb) in zip(sdb.ExecutePhraseGroupsMatchScanBatch(r, G, sc, 1 << 13, exclude=excl),
                                                          sdb.ExecuteMatchScanGroupsBatch(r, gq, sc, limit=1 << 13, exclude=excl,
                                                                                          min_match=ones)):
            assert ta == tb and np.array_equal(sa, sb) and np.array_equal(da, db)
            assert np.array_equal(xa.view(np.uint32), xb.view(np.uint32))
    # one group of one-slot alternatives: the flat OR
    flat = [q[0] for q in gq if len(q) == 1]
    FG = [[[[t] for t in g]] for g in flat]
    for sc in (sdb.BM25(), sdb.TFIDF(False)):
        a = sdb.ExecutePhraseGroupsTopKBatch(r, FG, sc, 100)
        b = sdb.ExecuteTopKBatch(r, flat, sdb.OR, sc, 100)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
        for i in range(len(flat)):
            h1, h2 = a[0][i, :a[1][i]], b[0][i, :b[1][i]]
            assert np.array_equal(h1["doc"], h2["doc"]) and np.array_equal(h1["score"].view(np.uint32), h2["score"].view(np.uint32))
    assert np.array_equal(sdb.ExecutePhraseGroupsCountBatch(r, FG), sdb.ExecuteCountBatch(r, flat, sdb.OR))
    for ((sa, da, xa), ta), ((sb, db, xb), tb) in zip(sdb.ExecutePhraseGroupsMatchScanBatch(r, FG, sdb.BM25(), 1 << 13),
                                                      sdb.ExecuteMatchScanBatch(r, flat, sdb.OR, sdb.BM25(), limit=1 << 13)):
        assert ta == tb and np.array_equal(da, db) and np.array_equal(xa.view(np.uint32), xb.view(np.uint32))


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
    qs = [([[[0, 1], [2]]], []), ([[[0, 1], [2, 0]], [[1]]], [[2, 1]]), ([[[0, 1]], [[2], [1]]], []), ([[[2, 0], [1, 0]]], [[0, 1]])]
    sc = sdb.BM25()
    counts = sdb.ExecutePhraseGroupsCountBatch(reader, [q[0] for q in qs], exclude_phrases=[q[1] for q in qs])
    hits, n_out, _ = sdb.ExecutePhraseGroupsTopKBatch(reader, [q[0] for q in qs], sc, 100, exclude_phrases=[q[1] for q in qs])
    by_term = []
    for d, f, pos in posts:
        ends = np.cumsum(f.astype(np.int64))
        by_term.append({int(x): set(pos[e - k:e].tolist()) for x, k, e in zip(d, f, ends)})
    dc = [len(p[0]) for p in posts]
    high = 0
    for i, q in enumerate(qs):
        groups = _groups(q)
        alts = pgr.flat(groups)
        ds, fs = [], []
        for doc in sorted(set(by_term[0]) | set(by_term[1]) | set(by_term[2])):
            if doc in dels:
                continue
            fr = []
            for terms, rel, _ in alts:
                rel = list(range(len(terms))) if rel is None else rel
                anchors = by_term[terms[0]].get(doc, set())
                fr.append(sum(1 for p in anchors if all(p + r in by_term[t].get(doc, set()) for t, r in zip(terms, rel))))
            j, ok = 0, True
            for ga, neg in groups:
                gf = fr[j:j + len(ga)]
                j += len(ga)
                ok = ok and (not any(gf) if neg else any(gf))
            if ok:
                ds.append(doc); fs.append(fr)
        assert counts[i] == len(ds), q
        order = sorted([j for j in range(len(alts)) if not alts[j][2]], key=lambda j: min(dc[t] for t in alts[j][0]))
        consts = [None if neg else pr.consts(reader.phrase_stats(sc, terms), sc.k, sc.b) for terms, _, neg in alts]
        rows = []
        for d, fr in zip(ds, fs):
            s = np.float32(0)
            for j in order:
                if fr[j]:
                    s = np.float32(s + pr.score(fr[j], 1, *consts[j]))
            rows.append((s, d))
        rows.sort(key=lambda x: (-x[0], x[1]))
        got = hits[i, :n_out[i]]
        assert got["doc"].tolist() == [d for _, d in rows[:100]], q
        assert got["score"].view(np.uint32).tolist() == np.array([s for s, _ in rows[:100]], np.float32).view(np.uint32).tolist()
        high += sum(1 for d in ds if d > (1 << 31))
        (_, docs, _), total = sdb.ExecutePhraseGroupsMatchScan(reader, q[0], None, 1 << 14, exclude_phrases=q[1])
        assert total == len(ds) and docs.tolist() == ds
    assert high > 0


# ---------------------------------------------------------------- errors
def _rc(t, terms, coff, goff, qoff, neg=None, rel=None, excl=None, excl_off=None):
    arr = lambda a, dt: None if a is None else np.ascontiguousarray(a, dt)
    terms, coff, goff, qoff = arr(terms, np.uint32), arr(coff, np.uint32), arr(goff, np.uint32), arr(qoff, np.uint32)
    neg, rel, excl, excl_off = arr(neg, np.uint8), arr(rel, np.uint32), arr(excl, np.uint32), arr(excl_off, np.uint32)
    nq = len(qoff) - 1 if qoff is not None else 1
    counts = np.zeros(max(nq, 1), np.uint64)
    segs = (C.c_void_p * len(t["segs"]))(*[s._h.value for s in t["segs"]])
    p = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    return N.lib().sdbg_phrase_groups_count_batch(segs, len(t["segs"]), p(terms), p(rel), p(coff), p(goff), p(neg), p(qoff), nq,
                                                  p(excl), p(excl_off), None, p(counts))


def test_errors_then_a_valid_call(pg):
    inval, unsup, notfound = -1, -7, -5
    launches = ctx().launches
    assert _rc(pg, [0, 1], [0, 0, 2], [0, 2], [0, 1]) == inval                 # an empty clause
    assert _rc(pg, [0, 1], [0, 1, 2], [0, 0, 2], [0, 2]) == inval              # an empty group
    assert _rc(pg, [0, 1], [0, 2], [0, 1], [0, 0, 1]) == inval                 # a query without a group
    assert _rc(pg, [0, 1], [0, 1, 2], [0, 2], [0, 1], neg=[1]) == inval        # a query without a positive group
    assert _rc(pg, [0, 1], [0, 2], [0, 1], [0, 1], rel=[1, 2]) == inval        # rel_pos not starting at 0
    assert _rc(pg, [0, 1, 2], [0, 3], [0, 1], [0, 1], rel=[0, 2, 2]) == inval  # rel_pos not increasing
    assert _rc(pg, [0, 1], [0, 2, 1], [0, 2], [0, 1]) == inval                 # decreasing clause offsets
    assert _rc(pg, [0, 1], [0, 1, 2], [0, 2, 1], [0, 2]) == inval              # decreasing group offsets
    assert _rc(pg, [0, 1], [0, 1, 2], [0, 1, 2], [0, 2, 1]) == inval           # decreasing query offsets
    assert _rc(pg, None, [0, 2], [0, 1], [0, 1]) == inval                      # NULL terms
    assert _rc(pg, [0, 1], None, [0, 1], [0, 1]) == inval                      # NULL clause_off
    assert _rc(pg, [0, 1], [0, 2], None, [0, 1]) == inval                      # NULL group_off
    assert _rc(pg, [0, 1], [0, 2], [0, 1], None) == inval                      # NULL query_group_off
    assert _rc(pg, [0, 1], [0, 1, 2], [0, 2], [0, 1], excl=None, excl_off=[0, 2]) == inval   # NULL excl_terms
    assert _rc(pg, [0, 99], [0, 1, 2], [0, 2], [0, 1]) == inval                # a positive term id out of range
    assert _rc(pg, list(range(9)) * 2, [0, 9, 18], [0, 1, 2], [0, 2], neg=[0, 1]) == unsup   # 18 slots
    assert _rc(pg, list(range(17)), list(range(18)), list(range(18)), [0, 17]) == unsup       # 17 groups
    assert _rc(pg, [0], [0, 1], [0, 1], [0, 1], excl=np.arange(17) % V, excl_off=[0, 17]) == unsup
    segs = (C.c_void_p * 3)(*[s._h.value for s in pg["segs"]])
    terms, coff, goff, qoff = (np.array(x, np.uint32) for x in ([0, 1, 2], [0, 2, 3], [0, 2], [0, 1]))
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    hits, n_out, total = np.zeros(5000, sdb.engine.HIT_DTYPE), np.zeros(1, np.uint32), np.zeros(1, np.uint64)
    assert N.lib().sdbg_phrase_groups_topk_batch(segs, 3, p(terms), None, p(coff), p(goff), None, p(qoff), 1, None, None, None, 1.2,
                                                 0.75, None, 10, 0.0, p(hits), p(n_out), p(total)) == inval
    assert N.lib().sdbg_phrase_groups_scan_batch(segs, 3, p(terms), None, p(coff), p(goff), None, p(qoff), 1, None, None, None, None,
                                                 1.2, 0.75, None, 10, 1, p(hits), p(n_out), p(total)) == inval
    st = (N.BM25Term * 2)(pg["reader"].phrase_stats(sdb.BM25(), [0, 1]), pg["reader"].phrase_stats(sdb.BM25(), [2]))
    assert N.lib().sdbg_phrase_groups_topk_batch(segs, 3, p(terms), None, p(coff), p(goff), None, p(qoff), 1, None, None, st, 1.2,
                                                 0.75, None, 4097, 0.0, p(hits), p(n_out), p(total)) == unsup
    assert ctx().launches == launches                                          # nothing was queued
    oseg = orc.Segment(100, has_wand=True)
    oseg.add_term(np.array([1, 2], np.uint32), np.array([1, 1], np.uint32))
    g = to_gpu(oseg, columns={I32: (np.arange(100, dtype=np.int32), None)})
    r2 = sdb.IndexReader([g], 100, 100, [2])
    for call in (lambda: sdb.ExecutePhraseGroupsCountBatch(r2, [[[[0]]]]),
                 lambda: sdb.ExecutePhraseGroupsTopKBatch(r2, [[[[0]]]], sdb.BM25(), 5),
                 lambda: sdb.ExecutePhraseGroupsTopKByColumnBatch(r2, [[[[0]]]], I32, 5),
                 lambda: sdb.ExecutePhraseGroupsFacetCountsBatch(r2, [[[[0]]]], I32, 0, 100),
                 lambda: sdb.ExecutePhraseGroupsMatchAggregatesBatch(r2, [[[[0]]]], I32),
                 lambda: sdb.ExecutePhraseGroupsMatchScanBatch(r2, [[[[0]]]])):
        with pytest.raises(N.SdbgError, match="ENOTFOUND"):
            call()
    _check(pg, _queries(pg, np.random.default_rng(9), 5), sdb.BM25(), k=10)


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


def test_adapters_phrase_groups_mode():
    """All six phrase adapters with clause_sizes / clause_negated / clause_group_sizes against the reference; each positive
    alternative scored with its statistics computed here by hand: its slots' BM25 idfs summed in float32, the first slot's
    norm constants."""
    import json
    import subprocess
    from serenedb_b200 import build as b

    exe = b.build_adapters()
    n = 20_000
    res = subprocess.run([exe, str(n), "phrase", "groups"], capture_output=True, text=True, timeout=300)
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
        off = np.concatenate([[0], np.cumsum(x["sizes"])]).astype(int)
        goff = np.concatenate([[0], np.cumsum(x["gsizes"])]).astype(int)
        alts = [(x["slots"][off[j]:off[j + 1]], x["rel"][off[j]:off[j + 1]]) for j in range(len(x["sizes"]))]
        groups = [(alts[goff[g]:goff[g + 1]], bool(x["neg"][goff[g]])) for g in range(len(x["gsizes"]))]
        consts = []
        for terms, _, neg in pgr.flat(groups):
            idf = np.float32(0)
            for t in terms:
                idf = np.float32(idf + np.float32(sc.collect(n, int(norms.sum()), len(post[t][0])).idf))
            st = sc.collect(n, int(norms.sum()), len(post[terms[0]][0]))
            c0 = np.float32(np.float32(np.float32(1.0) * np.float32(np.float32(1.2) + np.float32(1))) * idf)
            consts.append(None if neg else (c0, np.float32(st.norm_const), np.float32(st.norm_length)))
        w = pgr.matches([docs], groups, x["excl"])
        n_match = pgr.count(w)
        assert x["count"] == x["total"] == x["scan_total"] == n_match > 0, x["slots"]
        ref, _ = pgr.topk([docs], groups, w, [norms], consts, 50)
        assert [h[0] for h in x["topk"]] == ref["doc"].tolist(), x["slots"]
        assert np.array_equal(np.array([h[1] for h in x["topk"]], np.float32).view(np.uint32), ref["score"].view(np.uint32))
        assert x["sorted_docs"] == pgr.sorted_hits(w, cols, True, False, 30)["docs"].tolist()
        counts, nulls = pgr.facet_counts(w, cols, -11, 23)
        assert x["facet_keys"] == [k - 11 for k in np.nonzero(counts)[0].tolist()] + ([0] if nulls else [])
        assert x["facet_counts"] == counts[counts > 0].tolist() + ([nulls] if nulls else [])
        assert x["agg_count"] == [n_match]
        (_, rd, rsc), _ = pgr.scan([docs], groups, w, [norms], consts)
        assert x["scan_docs"] == rd.tolist()
        assert np.array_equal(np.array(x["scan_scores"], np.float32).view(np.uint32), rsc.view(np.uint32))
