"""The sorted scan, facet counts, aggregates and match scan of exact phrase queries on the GPU
(sdbg_phrase_topk_by_column_batch, sdbg_phrase_facet_counts_batch, sdbg_phrase_aggregate_batch, sdbg_phrase_scan_batch)
against the NumPy statement (tests/phrase_column_reference.py), bit for bit, over token-sequence segments (one missing a
term) with nullable int and float columns and deleted docs: every sort type, direction and NULL placement, k from 1 to
4096 and pruning levels 0..2; default and explicit key ranges and the out-of-range report; grouped and ungrouped
aggregates with exact 128-bit sums; scan pages, totals and scores under every scorer (equal to the phrase top-k's);
filter chains, exclusions, gaps, repeated terms, phrase lengths 1..16, doc ids past 2^31, a batch of 4096 phrases;
one-slot phrases against the flat AND entries; the error codes; and the adapters' phrase variants."""
import ctypes as C
import json
import subprocess

import numpy as np
import pytest

import count_reference as cr
import orc
import phrase_column_reference as pc
import phrase_reference as pr
import serenedb_b200 as sdb
from serenedb_b200 import _native as N
from gpu_util import ctx, to_gpu

pytestmark = pytest.mark.gpu

V = 12                       # vocabulary: term 11 never occurs in segment 1
SIZES = (3000, 2500, 4000)
I32, I64, F64, KEY, FILT, BIG = 1, 2, 3, 5, 4, 6   # column fields
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


def _columns(rng, n):
    """Per field (values, valid bool or None): nullable int32 / int64 / float64 sort columns, a nullable small-range key,
    a NOT NULL filter column and an int64 column of values near +-2^62 (their sum needs 128 bits)."""
    f = rng.random(n) * 200.0 - 100.0
    f[rng.random(n) < 0.02] = -0.0
    return {I32: (rng.integers(-1000, 1000, n).astype(np.int32), rng.random(n) < 0.85),
            I64: (rng.integers(-10**15, 10**15, n).astype(np.int64), rng.random(n) < 0.9),
            F64: (f, rng.random(n) < 0.8),
            KEY: (rng.integers(-5, 20, n).astype(np.int32), rng.random(n) < 0.9),
            FILT: (rng.integers(0, 50, n).astype(np.int32), None),
            BIG: (rng.integers(2**62 - 2**40, 2**62, n).astype(np.int64) * np.where(rng.random(n) < 0.3, -1, 1), rng.random(n) < 0.95)}


@pytest.fixture(scope="module")
def ph():
    rng = np.random.default_rng(4242)
    segs, docs, norms, cols = [], [], [], []
    for i, n in enumerate(SIZES):
        d, post, nm, oseg = _token_segment(rng, n, missing=(11,) if i == 1 else ())
        c = _columns(rng, n)
        g = to_gpu(oseg, columns={f: (v, None if m is None else cr.validity_words(m)) for f, (v, m) in c.items()})
        g.stage_positions(*pr.staged_positions(post))
        segs.append(g); docs.append(d); norms.append(nm); cols.append(c)
    deleted = [rng.choice(np.arange(1, SIZES[0] + 1), 300, replace=False).astype(np.uint32), None, None]
    segs[0].stage_docs_mask(deleted[0])
    dwt = [sum(int(np.count_nonzero([t in set(x) for x in d])) for d in docs) for t in range(V)]
    reader = sdb.IndexReader(segs, sum(SIZES), int(sum(int(n.sum()) for n in norms)), dwt)
    return dict(segs=segs, docs=docs, norms=norms, cols=cols, deleted=deleted, reader=reader)


def _phrases(t, rng, n, lengths):
    """Phrases cut from the corpus's own docs (so that they match), of the given lengths."""
    out = []
    for L in lengths:
        for _ in range(n):
            seq = t["docs"][int(rng.integers(0, 3))][int(rng.integers(0, 2500))]
            if len(seq) >= L:
                s = int(rng.integers(0, len(seq) - L + 1))
                out.append(seq[s:s + L])
            else:
                out.append(rng.integers(0, 4, L).tolist())
    return out


def _want(t, phrase, rel=None, excl=(), masks=None):
    return pc.matches(t["docs"], phrase, rel, excl, t["deleted"], masks)


def _col(t, f):
    return [c[f] for c in t["cols"]]


# ---------------------------------------------------------------- per-pass checks against the reference
def _check_sorted(t, phrases, field, k, desc, nf, rels=None, excl=None, filt=None, masks=None, wants=None):
    rels = rels or [None] * len(phrases)
    excl = excl or [[]] * len(phrases)
    wants = wants or [_want(t, p, r, x, masks) for p, r, x in zip(phrases, rels, excl)]
    got = sdb.ExecutePhraseTopKByColumnBatch(t["reader"], phrases, field, k, desc, nf, rel_pos=rels, filt=filt, exclude=excl)
    for q, w in enumerate(wants):
        ref = pc.sorted_hits(w, _col(t, field), desc, nf, k)
        assert got["n_out"][q] == len(ref["docs"]), (phrases[q], field, k)
        assert np.array_equal(got["docs"][q], ref["docs"]) and np.array_equal(got["segs"][q], ref["segs"]), (phrases[q], field)
        assert np.array_equal(got["nulls"][q], ref["nulls"])
        v, r = np.asarray(got["values"][q]), np.asarray(ref["values"])
        assert np.array_equal(v.view(np.uint64) if v.dtype == np.float64 else v, r.view(np.uint64) if r.dtype == np.float64 else r)
    return wants


def _check_facets(t, phrases, key_min=None, key_span=None, rels=None, excl=None, filt=None, masks=None, wants=None):
    rels = rels or [None] * len(phrases)
    excl = excl or [[]] * len(phrases)
    wants = wants or [_want(t, p, r, x, masks) for p, r, x in zip(phrases, rels, excl)]
    got = sdb.ExecutePhraseFacetCountsBatch(t["reader"], phrases, KEY, key_min, key_span, rel_pos=rels, filt=filt, exclude=excl)
    span = got["counts"].shape[1]
    for q, w in enumerate(wants):
        counts, nulls = pc.facet_counts(w, _col(t, KEY), got["key_min"], span)
        assert got["counts"][q].tolist() == counts.tolist() and int(got["nulls"][q]) == nulls, phrases[q]
        assert int(got["counts"][q].sum()) + int(got["nulls"][q]) == sum(len(ds) for ds, _ in w)
    return wants


def _cells_equal(got, q, i, cell, is_float, where):
    assert int(got["count"][q][i]) == cell["count"] and int(got["count_value"][q][i]) == cell["count_value"], where
    if not cell["count_value"]:
        return
    if is_float:
        assert np.isclose(float(got["sum"][q][i]), cell["sum"], rtol=1e-12, atol=1e-9), where
        assert np.float64(got["min"][q][i]).view(np.uint64) == np.float64(cell["min"]).view(np.uint64), where
        assert np.float64(got["max"][q][i]).view(np.uint64) == np.float64(cell["max"]).view(np.uint64), where
    else:
        assert int(got["sum"][q][i]) == cell["sum"], where
        assert int(got["min"][q][i]) == cell["min"] and int(got["max"][q][i]) == cell["max"], where


def _check_aggs(t, phrases, value, grouped, rels=None, excl=None, filt=None, masks=None, wants=None):
    rels = rels or [None] * len(phrases)
    excl = excl or [[]] * len(phrases)
    wants = wants or [_want(t, p, r, x, masks) for p, r, x in zip(phrases, rels, excl)]
    got = sdb.ExecutePhraseMatchAggregatesBatch(t["reader"], phrases, value, KEY if grouped else None, rel_pos=rels, filt=filt,
                                                exclude=excl)
    is_float = value == F64
    span = got["count"].shape[1]
    null = {f: [[x] for x in got["null"][f]] for f in ("count", "count_value", "sum", "min", "max")}
    for q, w in enumerate(wants):
        cells, null_cell = pc.aggregate(w, _col(t, KEY) if grouped else None, _col(t, value), got["key_min"], span)
        for i, c in enumerate(cells):
            _cells_equal(got, q, i, c, is_float, (phrases[q], value, i))
        if grouped:
            _cells_equal(null, q, 0, null_cell, is_float, (phrases[q], value, None))
        assert int(got["count"][q].sum()) + int(got["null"]["count"][q]) == sum(len(ds) for ds, _ in w)
    return wants


def _check_scan(t, phrases, scorer=None, limit=1 << 16, offsets=None, rels=None, excl=None, filt=None, masks=None, wants=None):
    rels = rels or [None] * len(phrases)
    excl = excl or [[]] * len(phrases)
    wants = wants or [_want(t, p, r, x, masks) for p, r, x in zip(phrases, rels, excl)]
    got = sdb.ExecutePhraseMatchScanBatch(t["reader"], phrases, scorer, limit, offsets, rel_pos=rels, filt=filt, exclude=excl)
    for q, (w, ((segs, docs, scores), total)) in enumerate(zip(wants, got)):
        c = None if scorer is None else pr.consts(t["reader"].phrase_stats(scorer, phrases[q]), scorer.k, scorer.b)
        (rs, rd, rsc), rt = pc.scan(w, t["norms"], c, 0 if offsets is None else int(offsets[q]), limit)
        assert total == rt and np.array_equal(segs, rs) and np.array_equal(docs, rd), (phrases[q], offsets)
        assert np.array_equal(scores.view(np.uint32), rsc.view(np.uint32)), (phrases[q], scorer)
    return got, wants


# ---------------------------------------------------------------- the passes
@pytest.mark.parametrize("field", [I32, I64, F64], ids=["int32", "int64", "float64"])
def test_sorted_every_type_direction_and_k(ph, field):
    rng = np.random.default_rng(field)
    phrases = _phrases(ph, rng, 3, (1, 2, 3)) + [[0, 0], [0, 11]]
    wants = None
    for desc in (False, True):
        for nf in (False, True):
            for k in (1, 10, 4096):
                wants = _check_sorted(ph, phrases, field, k, desc, nf, wants=wants)
    counts = sdb.ExecutePhraseCountBatch(ph["reader"], phrases)
    assert counts.tolist() == [sum(len(ds) for ds, _ in w) for w in wants]
    assert any(0 < c < 4096 for c in counts) and counts.max() > 1000      # k = 4096 lies above some phrases' counts


def test_sorted_ties_and_pruning_levels(ph):
    """The small-range key column makes long runs of equal values: ties go by (segment, doc); levels 0..2 agree."""
    rng = np.random.default_rng(11)
    phrases = _phrases(ph, rng, 4, (1, 2))
    wants = None
    for lv in (0, 1, 2):
        ctx().set_wand(lv)
        for desc, nf in ((False, False), (True, True), (True, False)):
            for k in (1, 5, 100):
                wants = _check_sorted(ph, phrases, KEY, k, desc, nf, wants=wants)
                _check_sorted(ph, phrases, FILT, k, desc, nf, wants=wants)
    ctx().set_wand(False)


def test_facets_ranges_nulls_and_out_of_range(ph):
    rng = np.random.default_rng(12)
    phrases = _phrases(ph, rng, 4, (1, 2, 3))
    wants = _check_facets(ph, phrases)                                      # the column's own range
    _check_facets(ph, phrases, -40, 100, wants=wants)                       # an explicit wider range
    assert sum(int(pc.facet_counts(w, _col(ph, KEY), -5, 25)[1]) for w in wants) > 0   # NULL keys among the matches
    with pytest.raises(N.SdbgError, match="outside"):
        sdb.ExecutePhraseFacetCountsBatch(ph["reader"], phrases[:1], KEY, 0, 10)


@pytest.mark.parametrize("value", [I32, F64, BIG], ids=["int32", "float64", "int64_wide"])
def test_aggregates(ph, value):
    rng = np.random.default_rng(13 + value)
    phrases = _phrases(ph, rng, 3, (1, 2, 3))
    wants = _check_aggs(ph, phrases, value, grouped=True)
    _check_aggs(ph, phrases, value, grouped=False, wants=wants)
    if value == BIG:   # the exact sum of values near +-2^62 leaves int64
        got = sdb.ExecutePhraseMatchAggregatesBatch(ph["reader"], [[0]], BIG)
        assert abs(int(got["sum"][0][0])) > 2**63


def test_scan_pages_and_totals(ph):
    rng = np.random.default_rng(14)
    phrases = _phrases(ph, rng, 3, (1, 2, 3))
    (_, wants) = _check_scan(ph, phrases)
    totals = [sum(len(ds) for ds, _ in w) for w in wants]
    assert sdb.ExecutePhraseCountBatch(ph["reader"], phrases).tolist() == totals
    for offs in ([0] * len(phrases), [n // 2 for n in totals], [max(n - 1, 0) for n in totals], [n for n in totals],
                 [n + 7 for n in totals]):
        for limit in (1, 13, max(totals) + 5):
            _check_scan(ph, phrases, None, limit, np.array(offs, np.uint64), wants=wants)


@pytest.mark.parametrize("scorer", SCORERS, ids=SCORER_IDS)
def test_scan_scores_equal_the_phrase_topk(ph, scorer):
    rng = np.random.default_rng(15)
    phrases = [p for p in _phrases(ph, rng, 4, (2, 3, 4))]
    got, wants = _check_scan(ph, phrases, scorer)
    hits, n_out, total = sdb.ExecutePhraseTopKBatch(ph["reader"], phrases, scorer, 4096)
    for q, ((segs, docs, scores), tot) in enumerate(got):
        assert tot == total[q]
        if tot > 4096:
            continue
        # the top-k holds the scores above its threshold (BM1 scores every match 0: none); every one of them is in the page
        h = hits[q, :n_out[q]]
        by = {(int(s), int(d)): np.float32(x) for s, d, x in zip(h["seg"], h["doc"], h["score"])}
        assert n_out[q] == int(np.count_nonzero(scores > 0))
        page = {(int(s), int(d)): np.float32(x) for s, d, x in zip(segs, docs, scores)}
        assert all(page[key].view(np.uint32) == x.view(np.uint32) for key, x in by.items())


@pytest.mark.parametrize("n_preds", [1, 2, 3, 4])
def test_filter_chains_and_exclusions(ph, n_preds):
    rng = np.random.default_rng(20 + n_preds)
    chain = [(FILT, "LT", 35), (I64, "GT", -5 * 10**14), (F64, "LE", 60.0), (I32, "NE", 3)][:n_preds]
    filt = [sdb.pred(f, op, v) for f, op, v in chain]
    masks = [np.logical_and.reduce([cr.pred_mask(c[f][0], c[f][1], op, v) for f, op, v in chain]) for c in ph["cols"]]
    phrases = _phrases(ph, rng, 3, (1, 2, 3))
    excl = [[int(rng.integers(4, 11))] if i % 2 else [] for i in range(len(phrases))]
    kw = dict(excl=excl, filt=filt, masks=masks)
    wants = _check_sorted(ph, phrases, I32, 50, False, True, **kw)
    _check_facets(ph, phrases, wants=wants, **kw)
    _check_aggs(ph, phrases, F64, True, wants=wants, **kw)
    _check_scan(ph, phrases, sdb.BM25(), wants=wants, **kw)


def test_gaps_repeated_terms_and_lengths_1_to_16(ph):
    rng = np.random.default_rng(30)
    phrases, rels = [], []
    for _ in range(10):
        seq = ph["docs"][0][int(rng.integers(0, 3000))]
        if len(seq) < 6:
            continue
        idx = sorted(rng.choice(len(seq), 3, replace=False).tolist())
        phrases.append([seq[i] for i in idx])
        rels.append([i - idx[0] for i in idx])
    phrases += _phrases(ph, rng, 1, range(1, 17)) + [[0, 0], [0, 0, 0], [1, 0, 1, 0]]
    rels += [None] * (len(phrases) - len(rels))
    wants = _check_sorted(ph, phrases, I64, 20, True, False, rels=rels)
    _check_facets(ph, phrases, rels=rels, wants=wants)
    _check_aggs(ph, phrases, I32, True, rels=rels, wants=wants)
    _check_scan(ph, phrases, sdb.BM25(), rels=rels, wants=wants)
    assert sum(1 for w in wants if sum(len(ds) for ds, _ in w)) > 20


def test_batch_of_4096(ph):
    rng = np.random.default_rng(31)
    base = _phrases(ph, rng, 4, (1, 2, 3))
    phrases = [base[i % len(base)] for i in range(4096)]
    ref = [_want(ph, p) for p in base]
    wants = [ref[i % len(base)] for i in range(4096)]
    _check_sorted(ph, phrases, I32, 10, False, False, wants=wants)
    _check_facets(ph, phrases, wants=wants)
    _check_aggs(ph, phrases, I64, False, wants=wants)
    _check_scan(ph, phrases, sdb.BM25(), limit=5, offsets=np.full(4096, 3, np.uint64), wants=wants)


def test_one_slot_equals_flat_and(ph):
    r = ph["reader"]
    sc = sdb.BM25()
    for lv in (0, 2):
        ctx().set_wand(lv)
        for term in range(V):
            a = sdb.ExecutePhraseTopKByColumnBatch(r, [[term]], I32, 30, True, True)
            b = sdb.ExecuteTopKByColumnBatch(r, [[term]], sdb.AND, I32, 30, True, True)
            for f in ("docs", "segs", "values", "nulls"):
                assert np.array_equal(a[f][0], b[f][0]), (term, f)
            a = sdb.ExecutePhraseFacetCountsBatch(r, [[term]], KEY, -5, 25)
            b = sdb.ExecuteFacetCountsBatch(r, [[term]], sdb.AND, KEY, -5, 25)
            assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["nulls"], b["nulls"])
            a = sdb.ExecutePhraseMatchAggregatesBatch(r, [[term]], F64, KEY, -5, 25)
            b = sdb.ExecuteMatchAggregatesBatch(r, [[term]], sdb.AND, F64, KEY, -5, 25)
            for f in ("count", "count_value", "min", "max"):
                assert np.array_equal(np.asarray(a[f]).view(np.uint64), np.asarray(b[f]).view(np.uint64)), (term, f)
            (sa, da, xa), ta = sdb.ExecutePhraseMatchScan(r, [term], sc, limit=1 << 14)
            (sb, db, xb), tb = sdb.ExecuteMatchScanBatch(r, [[term]], sdb.AND, sc, limit=1 << 14)[0]
            assert ta == tb and np.array_equal(sa, sb) and np.array_equal(da, db)
            assert np.array_equal(xa.view(np.uint32), xb.view(np.uint32)), term
    ctx().set_wand(False)


def test_doc_ids_past_2_31():
    """One segment of 2^32 - 2 docs; the columns cover the first 2^20 rows, so the high docs have NULL keys and values."""
    n = (1 << 32) - 2
    rng = np.random.default_rng(41)
    top = np.sort(rng.choice(np.arange(n - 5_000_000, n + 1, dtype=np.int64), 3000, replace=False)).astype(np.uint32)
    low = np.sort(rng.choice(np.arange(1, 1 << 20), 500, replace=False)).astype(np.uint32)
    a = np.unique(np.concatenate([low, top, [1 << 31, (1 << 31) + 1, n]])).astype(np.uint32)
    b = a[rng.random(len(a)) < 0.6]
    b = np.unique(np.concatenate([b, [1 << 31, n]])).astype(np.uint32)
    fa = rng.integers(1, 4, len(a)).astype(np.uint32)
    fb = np.ones(len(b), np.uint32)
    posts = [(a, fa, np.concatenate([np.arange(0, 2 * int(x), 2, dtype=np.uint32) for x in fa])),
             (b, fb, (2 * rng.integers(0, 3, len(b)) + 1).astype(np.uint32))]
    oseg = orc.Segment(n, has_wand=True)
    for d, f, _ in posts:
        oseg.add_term(d, f)
    rows = 1 << 20
    key = rng.integers(0, 8, rows).astype(np.int64)
    g = to_gpu(oseg, columns={KEY: (key, None)})
    g.stage_positions(*pr.staged_positions(posts))
    dels = [n, int(top[5])]
    g.stage_docs_mask(np.array(dels, np.uint32))
    reader = sdb.IndexReader([g], n, n, [len(a), len(b)])
    cols = [(key, None)]
    high = 0
    for p in ([0, 1], [1, 0], [0], [0, 0]):
        w = [pr.match_postings(posts, p, deleted=dels)]
        got = sdb.ExecutePhraseTopKByColumnBatch(reader, [p], KEY, 200, True, True)
        ref = pc.sorted_hits(w, cols, True, True, 200)
        assert np.array_equal(got["docs"][0], ref["docs"]) and np.array_equal(got["values"][0], ref["values"]), p
        f = sdb.ExecutePhraseFacetCountsBatch(reader, [p], KEY, 0, 8)
        counts, nulls = pc.facet_counts(w, cols, 0, 8)
        assert f["counts"][0].tolist() == counts.tolist() and int(f["nulls"][0]) == nulls, p
        agg = sdb.ExecutePhraseMatchAggregatesBatch(reader, [p], KEY)
        cells, _ = pc.aggregate(w, None, cols)
        assert int(agg["count"][0][0]) == cells[0]["count"] and int(agg["sum"][0][0]) == cells[0]["sum"], p
        sc = sdb.BM25()
        (segs, docs, scores), total = sdb.ExecutePhraseMatchScan(reader, p, sc, limit=1 << 14)
        (rs, rd, rsc), rt = pc.scan(w, None, pr.consts(reader.phrase_stats(sc, p), sc.k, sc.b))
        assert total == rt and np.array_equal(docs, rd) and np.array_equal(scores.view(np.uint32), rsc.view(np.uint32)), p
        high += int(np.count_nonzero(docs > (1 << 31)))
    assert high > 0


# ---------------------------------------------------------------- errors
def test_errors_then_a_valid_call(ph):
    r = ph["reader"]
    ph["segs"][0].stage_column(77, np.zeros(SIZES[0], np.int32))                # a sort column the other segments lack
    launches = ctx().launches
    calls = {
        "sorted": lambda p, **kw: sdb.ExecutePhraseTopKByColumnBatch(r, p, kw.get("field", I32), kw.get("k", 10)),
        "facet": lambda p, **kw: sdb.ExecutePhraseFacetCountsBatch(r, p, KEY, kw.get("lo", -5), kw.get("span", 25)),
        "agg": lambda p, **kw: sdb.ExecutePhraseMatchAggregatesBatch(r, p, kw.get("field", I32), KEY, -5, kw.get("span", 25)),
        "scan": lambda p, **kw: sdb.ExecutePhraseMatchScanBatch(r, p, None, kw.get("limit", 10)),
    }
    for name, call in calls.items():
        with pytest.raises(N.SdbgError, match="EINVAL"):
            call([[0, 1], []])                                                  # an empty phrase
        with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
            call([list(range(11)) + [0, 1, 2, 3, 4, 5]])                        # 17 slots
        with pytest.raises(N.SdbgError, match="EINVAL"):
            call([[0, 99]])                                                     # a term id out of range
    with pytest.raises(N.SdbgError, match="EINVAL"):
        calls["sorted"]([[0, 1]], k=0)
    with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
        calls["sorted"]([[0, 1]], k=4097)
    with pytest.raises(N.SdbgError, match="ENOTFOUND"):
        calls["sorted"]([[0, 1]], field=77)
    with pytest.raises(N.SdbgError, match="EINVAL"):
        calls["facet"]([[0, 1]], span=0)
    with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
        calls["facet"]([[0, 1]], span=40000)
    with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
        calls["agg"]([[0, 1]], span=5000)
    with pytest.raises(N.SdbgError, match="EINVAL"):
        calls["scan"]([[0, 1]], limit=0)
    # a scored scan without phrase statistics
    terms, off = np.array([0, 1], np.uint32), np.array([0, 2], np.uint32)
    hits, n_out, total = np.zeros(10, sdb.engine.HIT_DTYPE), np.zeros(1, np.uint32), np.zeros(1, np.uint64)
    segs = (C.c_void_p * 3)(*[s._h.value for s in ph["segs"]])
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    assert N.lib().sdbg_phrase_scan_batch(segs, 3, p(terms), None, p(off), 1, None, None, None, None, 1.2, 0.75, None, 10, 1,
                                          p(hits), p(n_out), p(total)) == -1
    assert ctx().launches == launches                                           # nothing was queued
    # a segment without positions
    oseg = orc.Segment(100, has_wand=True)
    oseg.add_term(np.array([1, 2], np.uint32), np.array([1, 1], np.uint32))
    g = to_gpu(oseg, columns={I32: (np.arange(100, dtype=np.int32), None)})
    r2 = sdb.IndexReader([g], 100, 100, [2])
    for call in (lambda: sdb.ExecutePhraseTopKByColumnBatch(r2, [[0]], I32, 5),
                 lambda: sdb.ExecutePhraseFacetCountsBatch(r2, [[0]], I32, 0, 100),
                 lambda: sdb.ExecutePhraseMatchAggregatesBatch(r2, [[0]], I32),
                 lambda: sdb.ExecutePhraseMatchScanBatch(r2, [[0]])):
        with pytest.raises(N.SdbgError, match="ENOTFOUND"):
            call()
    # the same context serves valid calls afterwards
    rng = np.random.default_rng(50)
    phrases = _phrases(ph, rng, 2, (2,))
    wants = _check_sorted(ph, phrases, I32, 10, False, False)
    _check_facets(ph, phrases, wants=wants)
    _check_aggs(ph, phrases, I32, True, wants=wants)
    _check_scan(ph, phrases, sdb.BM25(), wants=wants)


# ---------------------------------------------------------------- adapters
def _selftest_corpus(n_docs):
    """The token corpus of adapter_selftest's "phrase" mode, rebuilt from its generator."""
    state, docs = 12345, []

    def nxt():
        nonlocal state
        state = (state * 1664525 + 1013904223) & 0xFFFFFFFF
        return state >> 16
    for _ in range(n_docs):
        n = 1 + nxt() % 16
        docs.append([nxt() % 6 for _ in range(n)])
    return docs


def test_adapters_phrase_columns():
    """GpuSortedScan, GpuFacetScan, GpuMatchAggScan and GpuMatchScan with phrase_positions against the reference, the
    scan scored with the phrase's statistics computed here by hand (the slots' BM25 idfs summed in float32)."""
    from serenedb_b200 import build as b

    exe = b.build_adapters()
    n = 20_000
    res = subprocess.run([exe, str(n), "phrase", "columns"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = [json.loads(l) for l in res.stdout.strip().splitlines()]
    assert len(lines) == 2
    docs = _selftest_corpus(n)
    norms = np.array([len(d) for d in docs], np.uint32)
    d = np.arange(1, n + 1, dtype=np.int64)
    cols = [((d * 7919) % 23 - 11, d % 5 != 0)]
    post = pr.postings(docs, 6)
    sc = sdb.BM25()
    for x in lines:
        w = pc.matches([docs], x["slots"], x["rel"], x["excl"])
        n_match = len(w[0][0])
        assert n_match > 0
        ref = pc.sorted_hits(w, cols, True, False, 30)
        assert x["sorted_docs"] == ref["docs"].tolist() and x["sorted_values"] == ref["values"].tolist()
        assert x["sorted_valid"] == [0 if z else 1 for z in ref["nulls"]]
        counts, nulls = pc.facet_counts(w, cols, -11, 23)
        keys = [k - 11 for k in np.nonzero(counts)[0].tolist()]
        assert x["facet_keys"] == keys + ([0] if nulls else [])
        assert x["facet_counts"] == counts[counts > 0].tolist() + ([nulls] if nulls else [])
        assert x["facet_valid"] == [1] * len(keys) + ([0] if nulls else [])
        cells, _ = pc.aggregate(w, None, cols)
        c = cells[0]
        assert x["agg_count"] == [c["count"]] and x["agg_count_value"] == [c["count_value"]]
        assert x["agg_sum_lo"] == [c["sum"]] and x["agg_min"] == [c["min"]] and x["agg_max"] == [c["max"]]
        idf = np.float32(0)
        for t in x["slots"]:
            idf = np.float32(idf + np.float32(sc.collect(n, int(norms.sum()), len(post[t][0])).idf))
        st = sc.collect(n, int(norms.sum()), len(post[x["slots"][0]][0]))
        c0 = np.float32(np.float32(np.float32(1.0) * np.float32(np.float32(1.2) + np.float32(1))) * idf)
        (_, rd, rsc), rt = pc.scan(w, [norms], (c0, np.float32(st.norm_const), np.float32(st.norm_length)))
        assert x["scan_total"] == rt == n_match and x["scan_docs"] == rd.tolist()
        assert np.array_equal(np.array(x["scan_scores"], np.float32).view(np.uint32), rsc.view(np.uint32))
