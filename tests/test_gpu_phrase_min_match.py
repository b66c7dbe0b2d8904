"""Minimum match counts over OR groups of phrases and terms on the GPU (sdbg_phrase_groups_{count,topk,topk_by_column,
facet_counts,aggregate,scan}_batch_min) against the NumPy statement (tests/phrase_min_match_reference.py), bit for bit:
counts, hits (doc, segment, order, fp32 score bits), sorted hits, facet and aggregate cells, scan pages and totals. Over
token-sequence segments where one lacks a term of a positive alternative and one a term of a negated one, with deleted
docs, filter chains of 1..4 predicates, exclusions, every scorer, pruning levels 0..2, k above the match count and ties at
the cut; candidate minimums of 2 and more (distinct proxies), minimums lowered by shared proxies, two minimum groups, a
minimum group next to a negated phrase, a group left out of the candidates, exactly 16 slots with a 16-alternative group
at m = 15 (4 counter planes), the top-k at k = 4096 with 4 planes, a batch of 4096 mixing minimum groups with the three
candidate shapes; the three identities (every minimum 1: the OR-group entries; m equal to the group's size: the clause
conjunction entries; one-slot alternatives of distinct terms: the term *_groups_min entries); the error codes; the C++
adapters."""
import ctypes as C

import numpy as np
import pytest

import count_reference as cr
import orc
import phrase_min_match_reference as pmr
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
def pm():
    rng = np.random.default_rng(991)
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


def _tok(t, rng):
    """A token of some doc."""
    seq = t["docs"][int(rng.integers(0, 3))][int(rng.integers(0, 2500))]
    return int(seq[int(rng.integers(0, len(seq)))])


# A query: (positive groups, negated alternatives, one minimum per positive group)
def _queries(t, rng, n):
    """`2 of ("w1 w2" | s | t)`, `2 of ("w1 w2" | s | t) & u`, `2 of ("w1 w2" | s | "w3 w4")`, two minimum groups, a
    minimum group next to a negated phrase, and `3 of` a group of four; plus fixed queries on the missing terms, shared
    proxies and a group left out of the candidates."""
    qs = []
    for i in range(n):
        ph, _ = _cut(t, rng, 2 + i % 2)
        s, u, v = [_tok(t, rng)], [_tok(t, rng)], [_tok(t, rng)]
        kind = i % 6
        if kind == 0:
            qs.append(([[ph, s, v]], [], [2]))
        elif kind == 1:
            qs.append(([[ph, s, v], [u]], [], [2, 1]))
        elif kind == 2:
            qs.append(([[ph, s, _cut(t, rng, 2)[0]]], [], [2]))
        elif kind == 3:
            qs.append(([[ph, s, v], [_cut(t, rng, 2)[0], u, [_tok(t, rng)]]], [], [2, 2]))
        elif kind == 4:
            qs.append(([[ph, s, v]], [_cut(t, rng, 2)[0]], [2]))
        else:
            qs.append(([[ph, s, v, u], [[_tok(t, rng)], [_tok(t, rng)]]], [], [3, 1]))
    qs += [([[[0, 1], [11], [2]]], [], [2]),                        # segment 1 lacks 11: needs "0 1" and 2 there
           ([[[0, 1], [1, 2], [3]]], [], [2]),                      # both phrases may stand on 1: m' lowered to 1
           ([[[0, 1], [1, 0], [0]]], [[2, 3]], [2]),                # every alternative on one list
           ([[[0]], [[0], [1], [2]]], [], [1, 2]),                  # the group repeats 0: only checked per doc
           ([[[0], [0], [1]]], [], [2]),                            # duplicate alternatives: 0 alone is two of them
           ([[[3], [4], [5]], [[0, 1], [6], [7]]], [[10]], [2, 2]),  # a guaranteed minimum group (m' == m) and a phrase one
           ([[[1, 2], [2, 3], [3, 4], [5]]], [], [3])]
    return qs


def _groups(q):
    pos, neg, _ = q
    alt = lambda x: (list(x[0]), list(x[1])) if isinstance(x, tuple) else (list(x), None)
    return [([alt(a) for a in g], False) for g in pos] + [([alt(a)], True) for a in neg]


def _mins(q):
    return list(q[2]) + [1] * len(q[1])


def _consts(t, q, scorer):
    return [None if n else pr.consts(t["reader"].phrase_stats(scorer, terms), scorer.k, scorer.b)
            for terms, _, n in pmr.flat(_groups(q))]


def _want(t, q, excl=(), masks=None):
    return pmr.matches(t["docs"], _groups(q), excl, t["deleted"], masks, _mins(q))


def _col(t, f):
    return [c[f] for c in t["cols"]]


def _same_hits(a, b, ctx_=None):
    assert np.array_equal(a["doc"], b["doc"]) and np.array_equal(a["seg"], b["seg"]), ctx_
    assert np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)), ctx_


def _check(t, queries, scorer=None, k=10, excl=None, filt=None, masks=None, levels=(0,), passes=True):
    excl = excl or [[]] * len(queries)
    Q, X, M = [q[0] for q in queries], [q[1] for q in queries], [q[2] for q in queries]
    kw = dict(filt=filt, exclude=excl, exclude_phrases=X, min_match=M)
    wants = [_want(t, q, x, masks) for q, x in zip(queries, excl)]
    counts = sdb.ExecutePhraseGroupsCountBatch(t["reader"], Q, **kw)
    assert counts.tolist() == [pmr.count(w) for w in wants]
    if scorer is not None:
        for lv in levels:
            ctx().set_wand(lv)
            hits, n_out, total = sdb.ExecutePhraseGroupsTopKBatch(t["reader"], Q, scorer, k, **kw)
            assert np.array_equal(total, counts)
            for i, (q, w) in enumerate(zip(queries, wants)):
                ref, _ = pmr.topk(t["docs"], _groups(q), w, t["norms"], _consts(t, q, scorer), k)
                got = hits[i, :n_out[i]]
                assert len(got) == len(ref), (q, lv)
                _same_hits(got, ref, (q, lv))
            ctx().set_wand(False)
    if not passes:
        return counts
    got = sdb.ExecutePhraseGroupsTopKByColumnBatch(t["reader"], Q, I32, k, True, False, **kw)
    for i, w in enumerate(wants):
        ref = pmr.sorted_hits(w, _col(t, I32), True, False, k)
        assert np.array_equal(got["docs"][i], ref["docs"]) and np.array_equal(got["segs"][i], ref["segs"]), queries[i]
        assert np.array_equal(got["values"][i], ref["values"]) and np.array_equal(got["nulls"][i], ref["nulls"])
    got = sdb.ExecutePhraseGroupsFacetCountsBatch(t["reader"], Q, KEY, -5, 25, **kw)
    for i, w in enumerate(wants):
        c, nulls = pmr.facet_counts(w, _col(t, KEY), -5, 25)
        assert got["counts"][i].tolist() == c.tolist() and int(got["nulls"][i]) == nulls, queries[i]
    got = sdb.ExecutePhraseGroupsMatchAggregatesBatch(t["reader"], Q, I32, KEY, -5, 25, **kw)
    for i, w in enumerate(wants):
        cells, null_cell = pmr.aggregate(w, _col(t, KEY), _col(t, I32), -5, 25)
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
            (rs, rd, rsc), rt = pmr.scan(t["docs"], _groups(q), w, t["norms"], _consts(t, q, sc),
                                         0 if offs is None else int(offs[i]), limit)
            assert total == rt and np.array_equal(segs, rs) and np.array_equal(docs, rd), q
            assert np.array_equal(scores.view(np.uint32), rsc.view(np.uint32)), q
    return counts


# ---------------------------------------------------------------- the passes
@pytest.mark.parametrize("scorer", SCORERS, ids=SCORER_IDS)
def test_every_pass_every_scorer(pm, scorer):
    rng = np.random.default_rng(3)
    counts = _check(pm, _queries(pm, rng, 18), scorer, k=15)
    assert int(np.count_nonzero(counts)) >= 15


def test_pruning_levels_large_k_and_ties(pm):
    rng = np.random.default_rng(4)
    qs = _queries(pm, rng, 12)
    counts = _check(pm, qs, sdb.BM25(), k=4096, levels=(0, 1, 2), passes=False)
    assert counts.min() < 4096 < counts.max()
    for k in (1, 2, 3, 7):
        _check(pm, qs[:8], sdb.BM25(), k=k, levels=(0, 2), passes=False)


@pytest.mark.parametrize("n_preds", [1, 2, 3, 4])
def test_filter_chains_and_exclusions(pm, n_preds):
    rng = np.random.default_rng(20 + n_preds)
    chain = [(FILT, "LT", 35), (I32, "GT", -500), (F64, "LE", 60.0), (KEY, "NE", 3)][:n_preds]
    filt = [sdb.pred(f, op, v) for f, op, v in chain]
    masks = [np.logical_and.reduce([cr.pred_mask(c[f][0], c[f][1], op, v) for f, op, v in chain]) for c in pm["cols"]]
    qs = _queries(pm, rng, 12)
    excl = [[int(rng.integers(4, 11))] if i % 2 else [] for i in range(len(qs))]
    _check(pm, qs, sdb.BM25(), k=20, excl=excl, filt=filt, masks=masks)


def test_sixteen_slots_and_four_planes(pm):
    """Groups of 16 one-slot alternatives at m = 13 and m = 15 over the 12 terms (the four repeated terms stand twice on
    their lists: candidate minimums 9 and 11, 4 counter planes), every alternative one of four terms, and 16 slots of
    phrases with a minimum group; the top-k at k = 4096 with the planes behind the phrase sink's 128 KB of keys."""
    rng = np.random.default_rng(6)
    wide = [[t % V] for t in range(16)]                               # 12 distinct terms, 4 repeated: m' < 15
    qs = [([[[t] for t in range(V)] + [[0], [1], [2], [3]]], [], [13]),
          ([wide], [], [15]),
          ([[[t % 4] for t in range(16)]], [], [9]),
          ([[[t] for t in range(10)]], [[10, 11], [11], [10, 0, 1]], [3])]
    for _ in range(3):
        ph, seq = _cut(pm, rng, 5)
        qs.append(([[ph, [int(seq[0])], _cut(pm, rng, 3)[0], [_tok(pm, rng)]], [_cut(pm, rng, 2)[0], [_tok(pm, rng)]]],
                   [_cut(pm, rng, 3)[0]], [2, 1]))                     # 5 + 1 + 3 + 1 + 2 + 1 + 3
    assert all(sum(len(a[0]) for a in pmr.flat(_groups(q))) == 16 for q in qs)
    counts = _check(pm, qs, sdb.BM25(), k=10)
    assert counts[2] > 0 and counts[3] > 0
    _check(pm, qs, sdb.BM25(), k=4096, levels=(0, 2), passes=False)


def test_batch_of_4096_mixes_minimum_groups_and_the_shapes(pm):
    """Minimum groups next to the AND, flat OR and OR-group shapes in one batch of 4096; each query's result is its
    result alone."""
    rng = np.random.default_rng(7)
    base = _queries(pm, rng, 12) + [([[_cut(pm, rng, 2)[0]], [[1]]], [], [1, 1]), ([[[0, 1], [2]]], [], [1]),
                                    ([[[0, 1], [2]], [[3], [4, 5]]], [[6]], [1, 1])]
    qs = [base[(i * 7) % len(base)] for i in range(4096)]
    Q, X, M = [q[0] for q in qs], [q[1] for q in qs], [q[2] for q in qs]
    counts = sdb.ExecutePhraseGroupsCountBatch(pm["reader"], Q, exclude_phrases=X, min_match=M)
    alone = [int(sdb.ExecutePhraseGroupsCount(pm["reader"], q[0], exclude_phrases=q[1], min_match=q[2])) for q in base]
    assert alone == [pmr.count(_want(pm, q)) for q in base]
    assert counts.tolist() == [alone[(i * 7) % len(base)] for i in range(4096)]
    sc = sdb.BM25()
    hits, n_out, total = sdb.ExecutePhraseGroupsTopKBatch(pm["reader"], Q, sc, 5, exclude_phrases=X, min_match=M)
    assert np.array_equal(total, counts)
    for i in range(0, 4096, 97):
        q = qs[i]
        h1, n1 = sdb.ExecutePhraseGroupsTopK(pm["reader"], q[0], sc, 5, exclude_phrases=q[1], min_match=q[2])
        _same_hits(hits[i, :n_out[i]], h1, q)
        r, _ = pmr.topk(pm["docs"], _groups(q), _want(pm, q), pm["norms"], _consts(pm, q, sc), 5)
        _same_hits(h1, r, q)
    f = sdb.ExecutePhraseGroupsFacetCountsBatch(pm["reader"], Q, KEY, -5, 25, exclude_phrases=X, min_match=M)
    s = sdb.ExecutePhraseGroupsTopKByColumnBatch(pm["reader"], Q, I32, 5, exclude_phrases=X, min_match=M)
    scans = sdb.ExecutePhraseGroupsMatchScanBatch(pm["reader"], Q, None, 3, exclude_phrases=X, min_match=M)
    for i in range(0, 4096, 131):
        w = _want(pm, qs[i])
        c, nulls = pmr.facet_counts(w, _col(pm, KEY), -5, 25)
        assert f["counts"][i].tolist() == c.tolist() and int(f["nulls"][i]) == nulls
        assert np.array_equal(s["docs"][i], pmr.sorted_hits(w, _col(pm, I32), False, False, 5)["docs"])
        (rs, rd, _), rt = pmr.scan(pm["docs"], _groups(qs[i]), w, limit=3)
        (ss, sd, _), st = scans[i]
        assert st == rt and np.array_equal(sd, rd) and np.array_equal(ss, rs)


# ---------------------------------------------------------------- the identities
def _all_passes(r, Q, kw, kw2, fa, fb):
    """The six passes of the phrase groups functions (fa: keyword arguments kw) and of another family (fb, kw2)."""
    for sc in (sdb.BM25(), sdb.TFIDF(True)):
        for lv in (0, 2):
            ctx().set_wand(lv)
            a = fa["topk"](r, Q[0], sc, 30, **kw)
            b = fb["topk"](r, Q[1], sc, 30, **kw2)
            assert all(np.array_equal(x, y) for x, y in zip(a, b)), lv
        ctx().set_wand(False)
    assert np.array_equal(fa["count"](r, Q[0], **kw), fb["count"](r, Q[1], **kw2))
    a, b = fa["sorted"](r, Q[0], I32, 40, False, True, **kw), fb["sorted"](r, Q[1], I32, 40, False, True, **kw2)
    for f in ("n_out", "docs", "segs", "values", "nulls"):
        assert all(np.array_equal(x, y) for x, y in zip(a[f], b[f])), f
    a, b = fa["facet"](r, Q[0], KEY, -5, 25, **kw), fb["facet"](r, Q[1], KEY, -5, 25, **kw2)
    assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["nulls"], b["nulls"])
    a, b = fa["agg"](r, Q[0], I32, KEY, -5, 25, **kw), fb["agg"](r, Q[1], I32, KEY, -5, 25, **kw2)
    for f in ("count", "count_value", "sum", "min", "max"):
        assert np.array_equal(np.asarray(a[f]), np.asarray(b[f])), f
    a, b = fa["scan"](r, Q[0], sdb.BM25(), 1 << 13, **kw), fb["scan"](r, Q[1], sdb.BM25(), 1 << 13, **kw2)
    for ((sa, da, xa), ta), ((sb, db, xb), tb) in zip(a, b):
        assert ta == tb and np.array_equal(sa, sb) and np.array_equal(da, db)
        assert np.array_equal(xa.view(np.uint32), xb.view(np.uint32))


PHRASE_GROUPS = dict(topk=sdb.ExecutePhraseGroupsTopKBatch, count=sdb.ExecutePhraseGroupsCountBatch,
                     sorted=sdb.ExecutePhraseGroupsTopKByColumnBatch, facet=sdb.ExecutePhraseGroupsFacetCountsBatch,
                     agg=sdb.ExecutePhraseGroupsMatchAggregatesBatch, scan=sdb.ExecutePhraseGroupsMatchScanBatch)


def test_identity_every_minimum_one_is_the_or_groups(pm):
    rng = np.random.default_rng(8)
    qs = _queries(pm, rng, 12)
    Q, X = [q[0] for q in qs], [q[1] for q in qs]
    ones = [[1] * len(q[0]) for q in qs]
    _all_passes(pm["reader"], (Q, Q), dict(exclude_phrases=X, min_match=ones), dict(exclude_phrases=X), PHRASE_GROUPS,
                PHRASE_GROUPS)


def test_identity_minimum_equal_to_size_is_the_clause_conjunction(pm):
    """`3 of (A | B | C) & D & !E` is `A & B & C & D & !E`, score bits included."""
    rng = np.random.default_rng(9)
    qs = []
    for _ in range(8):
        alts = [_cut(pm, rng, 2)[0], [_tok(pm, rng)], _cut(pm, rng, 3)[0]]
        qs.append((alts, [_tok(pm, rng)], [_cut(pm, rng, 2)[0]]))
    G = [[q[0], [q[1]]] for q in qs]
    M = [[3, 1] for _ in qs]
    A = [q[0] + [q[1]] for q in qs]
    X = [q[2] for q in qs]
    PHRASE_AND = dict(topk=sdb.ExecutePhraseAndTopKBatch, count=sdb.ExecutePhraseAndCountBatch,
                      sorted=sdb.ExecutePhraseAndTopKByColumnBatch, facet=sdb.ExecutePhraseAndFacetCountsBatch,
                      agg=sdb.ExecutePhraseAndMatchAggregatesBatch, scan=sdb.ExecutePhraseAndMatchScanBatch)
    _all_passes(pm["reader"], (G, A), dict(exclude_phrases=X, min_match=M), dict(exclude_phrases=X), PHRASE_GROUPS,
                PHRASE_AND)


def test_identity_one_slot_alternatives_are_the_min_match_groups(pm):
    """Distinct one-slot alternatives with any minimums: the term *_groups_min entries, the top-k bit for bit at pruning
    level 0."""
    r = pm["reader"]
    gq = [[[0, 1, 2], [3]], [[3, 1, 4, 0], [5, 2]], [[0, 1, 2, 3, 4, 5]], [[0, 6], [1, 2, 3]], [[7, 8, 9, 11]], [[0, 11, 2]]]
    mins = [[2, 1], [3, 2], [4], [1, 2], [2], [2]]
    excl = [[], [7], [], [8, 9], [], [10]]
    G = [[[[t] for t in g] for g in q] for q in gq]
    ctx().set_wand(0)
    for sc in SCORERS:
        a = sdb.ExecutePhraseGroupsTopKBatch(r, G, sc, 100, exclude=excl, min_match=mins)
        b = sdb.ExecuteTopKGroupsBatch(r, gq, sc, 100, exclude=excl, min_match=mins)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
        for i in range(len(gq)):
            _same_hits(a[0][i, :a[1][i]], b[0][i, :b[1][i]], gq[i])
    ctx().set_wand(False)
    kw = dict(exclude=excl, min_match=mins)
    assert np.array_equal(sdb.ExecutePhraseGroupsCountBatch(r, G, **kw), sdb.ExecuteCountGroupsBatch(r, gq, **kw))
    a = sdb.ExecutePhraseGroupsTopKByColumnBatch(r, G, I32, 40, True, True, **kw)
    b = sdb.ExecuteTopKByColumnGroupsBatch(r, gq, I32, 40, True, True, **kw)
    for f in ("n_out", "docs", "segs", "values", "nulls"):
        assert all(np.array_equal(x, y) for x, y in zip(a[f], b[f])), f
    a = sdb.ExecutePhraseGroupsFacetCountsBatch(r, G, KEY, -5, 25, **kw)
    b = sdb.ExecuteFacetCountsGroupsBatch(r, gq, KEY, -5, 25, **kw)
    assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["nulls"], b["nulls"])
    a = sdb.ExecutePhraseGroupsMatchAggregatesBatch(r, G, I32, KEY, -5, 25, **kw)
    b = sdb.ExecuteMatchAggregatesGroupsBatch(r, gq, I32, KEY, -5, 25, **kw)
    for f in ("count", "count_value", "sum", "min", "max"):
        assert np.array_equal(np.asarray(a[f]), np.asarray(b[f])), f
    for sc in (sdb.BM25(), sdb.TFIDF(False)):
        for ((sa, da, xa), ta), ((sb, db, xb), tb) in zip(sdb.ExecutePhraseGroupsMatchScanBatch(r, G, sc, 1 << 13, **kw),
                                                          sdb.ExecuteMatchScanGroupsBatch(r, gq, sc, limit=1 << 13, **kw)):
            assert ta == tb and np.array_equal(sa, sb) and np.array_equal(da, db)
            assert np.array_equal(xa.view(np.uint32), xb.view(np.uint32))


# ---------------------------------------------------------------- errors
def test_errors_then_a_valid_call(pm):
    inval, unsup = -1, -7
    launches = ctx().launches
    segs = (C.c_void_p * 3)(*[s._h.value for s in pm["segs"]])
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
    u32 = lambda a: np.array(a, np.uint32)
    # ("0 1" | 2 | 3) & !(4 | 5)
    terms, coff, goff, qoff = u32([0, 1, 2, 3, 4, 5]), u32([0, 2, 3, 4, 5, 6]), u32([0, 3, 5]), u32([0, 2])
    neg = np.array([0, 1], np.uint8)
    counts = np.zeros(1, np.uint64)
    rc = lambda gmin: N.lib().sdbg_phrase_groups_count_batch_min(segs, 3, p(terms), None, p(coff), p(goff), p(neg), p(gmin),
                                                                 p(qoff), 1, None, None, None, p(counts))
    assert rc(u32([0, 1])) == inval                 # m = 0
    assert rc(u32([4, 1])) == inval                 # m above the group's size
    assert rc(u32([2, 2])) == unsup                 # a negated group with m != 1
    assert rc(u32([2, 0])) == inval
    hits, n_out, total = np.zeros(16, sdb.engine.HIT_DTYPE), np.zeros(1, np.uint32), np.zeros(1, np.uint64)
    st = (N.BM25Term * 5)()
    assert N.lib().sdbg_phrase_groups_topk_batch_min(segs, 3, p(terms), None, p(coff), p(goff), p(neg), p(u32([2, 2])), p(qoff), 1,
                                                     None, None, st, 1.2, 0.75, None, 10, 0.0, p(hits), p(n_out), p(total)) == unsup
    assert N.lib().sdbg_phrase_groups_scan_batch_min(segs, 3, p(terms), None, p(coff), p(goff), p(neg), p(u32([0, 1])), p(qoff), 1,
                                                     None, None, None, None, 1.2, 0.75, None, 10, 0, p(hits), p(n_out),
                                                     p(total)) == inval
    assert ctx().launches == launches               # nothing was queued
    assert rc(u32([2, 1])) == 0
    q = ([[[0, 1], [2], [3]]], [[4], [5]], [2])
    assert int(counts[0]) == pmr.count(_want(pm, q))
    with pytest.raises(ValueError):
        sdb.ExecutePhraseGroupsCountBatch(pm["reader"], [q[0]], min_match=[[2, 1]])
    with pytest.raises(N.SdbgError, match="EINVAL"):
        sdb.ExecutePhraseGroupsCountBatch(pm["reader"], [q[0]], min_match=[[4]])


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


def test_adapters_count_and_topk_take_the_minimums(pm):
    """GpuCountScan and GpuTopKIterator with phrase_positions and group_min_match return the minimum-match result (the
    adapters used to drop the minimums); a minimum per clause group, a size mismatch refused."""
    import json
    import subprocess
    from serenedb_b200 import build as b

    exe = b.build_adapters()
    n = 20_000
    res = subprocess.run([exe, str(n), "phrase", "min"], capture_output=True, text=True, timeout=300)
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
        for terms, _, neg in pmr.flat(groups):
            idf = np.float32(0)
            for t in terms:
                idf = np.float32(idf + np.float32(sc.collect(n, int(norms.sum()), len(post[t][0])).idf))
            st = sc.collect(n, int(norms.sum()), len(post[terms[0]][0]))
            c0 = np.float32(np.float32(np.float32(1.0) * np.float32(np.float32(1.2) + np.float32(1))) * idf)
            consts.append(None if neg else (c0, np.float32(st.norm_const), np.float32(st.norm_length)))
        w = pmr.matches([docs], groups, x["excl"], mins=x["gmin"])
        n_match = pmr.count(w)
        # the minimums matter here: with every minimum 1 the query matches more
        assert n_match < pmr.count(pmr.matches([docs], groups, x["excl"])), x["slots"]
        assert x["count"] == x["total"] == x["scan_total"] == n_match > 0, x["slots"]
        ref, _ = pmr.topk([docs], groups, w, [norms], consts, 50)
        assert [h[0] for h in x["topk"]] == ref["doc"].tolist(), x["slots"]
        assert np.array_equal(np.array([h[1] for h in x["topk"]], np.float32).view(np.uint32), ref["score"].view(np.uint32))
        assert x["sorted_docs"] == pmr.sorted_hits(w, cols, True, False, 30)["docs"].tolist()
        counts, nulls = pmr.facet_counts(w, cols, -11, 23)
        assert x["facet_keys"] == [k - 11 for k in np.nonzero(counts)[0].tolist()] + ([0] if nulls else [])
        assert x["facet_counts"] == counts[counts > 0].tolist() + ([nulls] if nulls else [])
        assert x["agg_count"] == [n_match]
        (_, rd, rsc), _ = pmr.scan([docs], groups, w, [norms], consts)
        assert x["scan_docs"] == rd.tolist()
        assert np.array_equal(np.array(x["scan_scores"], np.float32).view(np.uint32), rsc.view(np.uint32))
