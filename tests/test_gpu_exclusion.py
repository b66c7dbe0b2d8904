"""Queries with excluded terms (`a & b & !c`, `(a | b) & !c`) on the GPU against the oracle's exhaustive evaluation (with
the excluded docs masked, tests/excl_reference.py), bit for bit (doc, segment, fp32 score), at pruning levels 0, 1 and 2: total_matches exact at level 0 and never above it with
pruning. Covers the stream kernels (OR of 1..4 terms, AND), the legacy window kernel (OR of 5..8 terms, BM15, BM1,
TFIDF), the hybrid filter and deleted docs, every block encoding as the excluded list, several segments, a lead-mode
shaped pair, the streaming scan, the C++ adapter and a 2 M-doc batch."""
import ctypes as C
import json
import subprocess

import numpy as np
import pytest

import orc
import serenedb_b200 as sdb
from serenedb_b200 import _native as N
from excl_reference import topk_batch_excl, topk_excl
from gpu_util import assert_hits_equal, ctx, oracle_terms, to_gpu
from shape_corpora import NORM_WIDTHS, Corpus, natural_segments, shape_segment, uniform_segments

pytestmark = pytest.mark.gpu

LEVELS = (0, 1, 2)


def _okind(kind):
    return "AND" if kind == sdb.AND else "OR"


def check(reader, osegs, kind, queries, excludes, scorer, k, gfilt=None, ofilt=None, deleted=None, levels=LEVELS):
    """GPU batch with exclusions at each pruning level == the exhaustive reference; returns the level-0 totals."""
    oq = [oracle_terms(reader, scorer, q) for q in queries]
    oh, on, ot = topk_batch_excl(osegs, _okind(kind), oq, excludes, k, k1=scorer.k, b=scorer.b, filt=ofilt, deleted=deleted)
    try:
        for lvl in levels:
            ctx().set_wand(lvl)
            gh, gn, gt = sdb.ExecuteTopKBatch(reader, queries, kind, scorer, k, filt=gfilt, exclude=excludes)
            for q in range(len(queries)):
                assert_hits_equal(gh[q, :gn[q]], oh[q, :on[q]])
                if lvl == 0:
                    assert gt[q] == ot[q], (lvl, q)
                else:
                    assert gt[q] <= ot[q], (lvl, q)
    finally:
        ctx().set_wand(0)
    return ot


@pytest.fixture(scope="module")
def synth():
    n = 200_000
    tids = list(range(0, 24))
    oseg, dl, lists = orc.synth_segment(n, tids)
    g = to_gpu(oseg)
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d, _ in lists])
    return dict(oseg=oseg, g=g, reader=reader, n=n, dl=dl, lists=lists)


def _random_queries(rng, n_terms, sizes, n_excl, count):
    qs, xs = [], []
    for _ in range(count):
        q = sorted(int(t) for t in rng.choice(n_terms, size=int(rng.choice(sizes)), replace=False))
        rest = [t for t in range(n_terms) if t not in q]
        xs.append([int(t) for t in rng.choice(rest, size=int(rng.integers(n_excl[0], n_excl[1] + 1)), replace=False)])
        qs.append(q)
    return qs, xs


@pytest.mark.parametrize("kind,sizes", [(sdb.OR, (1, 2, 3, 4)), (sdb.AND, (2, 3, 5, 8, 16)), (sdb.OR, (5, 6, 7, 8))],
                         ids=["or1-4", "and2-16", "or5-8"])
def test_bm25_forms(synth, kind, sizes):
    rng = np.random.default_rng(len(sizes) + kind)
    n_terms = 24 if kind == sdb.AND else 12
    qs, xs = _random_queries(rng, n_terms, sizes, (1, 3), 24)
    if kind == sdb.AND:                       # keep the conjunctions non-empty: dense terms first
        qs = [sorted(rng.choice(6, size=min(len(q), 6), replace=False).tolist()) + [t for t in q if t >= 6][:max(0, len(q) - 6)]
              for q in qs]
        xs = [[t for t in x if t not in q] or [20] for q, x in zip(qs, xs)]
    tot = check(synth["reader"], [synth["oseg"]], kind, qs, xs, sdb.BM25(), 100)
    assert tot.sum() > 0


@pytest.mark.parametrize("scorer", [sdb.BM25(1.2, 0.0), sdb.BM25(0.0, 0.75), sdb.TFIDF(False), sdb.TFIDF(True)],
                         ids=["bm15", "bm1", "tfidf", "tfidf_norm"])
def test_other_scorers_legacy_kernel(synth, scorer):
    rng = np.random.default_rng(3)
    for kind in (sdb.OR, sdb.AND):
        qs, xs = _random_queries(rng, 8, (1, 2, 3), (1, 2), 12)
        check(synth["reader"], [synth["oseg"]], kind, qs, xs, scorer, 50)


def test_filter_and_deleted_docs():
    n = 150_000
    oseg, dl, lists = orc.synth_segment(n, list(range(10)))
    vals = orc.synth_column(2, 1, 1, n).astype(np.int32)
    oseg.add_column(9, vals)
    rng = np.random.default_rng(8)
    deleted = np.unique(rng.integers(1, n + 1, 9000)).astype(np.uint32)
    oseg.set_docs_mask(deleted)
    g = to_gpu(oseg, columns={9: (vals, None)})
    g.stage_docs_mask(deleted)
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d, _ in lists])
    qs = [[0, 3], [1], [2, 5, 7, 9], [0, 1]]
    xs = [[1], [4, 6], [0], [2, 3, 8]]
    for kind in (sdb.OR, sdb.AND):
        check(reader, [oseg], kind, qs, xs, sdb.BM25(), 100, gfilt=sdb.pred(9, "BETWEEN", 200000, 799999),
              ofilt=orc.make_pred(9, "BETWEEN", 200000, 799999), deleted=[deleted])
        check(reader, [oseg], kind, qs, xs, sdb.BM25(), 100, deleted=[deleted])


@pytest.fixture(scope="module", params=NORM_WIDTHS, ids=lambda w: f"norms{w or 0}")
def shapes(request):
    oseg, norms, lists = shape_segment(request.param)
    g = to_gpu(oseg)
    ttf = int(norms.astype(np.uint64).sum()) if norms is not None else oseg.n_docs
    reader = sdb.IndexReader([g], oseg.n_docs, ttf, [len(d) for _, d, _ in lists])
    return dict(oseg=oseg, g=g, reader=reader, lists=lists)


def test_every_encoding_as_excluded_list(shapes):
    """Each shape term excluded from its companion (which shares ~15 % of its docs and adds misses): the companion's
    docs minus the shape's, through OR (alone and with a second term) and AND."""
    lists = shapes["lists"]
    shape_ids = [t for t, (name, _, _) in enumerate(lists) if not name.endswith("+lead")]
    qs_or, xs = [[t + 1] for t in shape_ids], [[t] for t in shape_ids]
    k = max(len(lists[t + 1][1]) for t in shape_ids)
    check(shapes["reader"], [shapes["oseg"]], sdb.OR, qs_or, xs, sdb.BM25(), min(k, 8192))
    qs_or2 = [[t + 1, (t + 3) % len(lists)] for t in shape_ids]
    check(shapes["reader"], [shapes["oseg"]], sdb.OR, qs_or2, xs, sdb.BM25(), 100)
    qs_and = [[t + 1, (t + 3) % len(lists)] for t in shape_ids]
    check(shapes["reader"], [shapes["oseg"]], sdb.AND, qs_and, xs, sdb.BM25(), 100)


def test_dense_excluded_list(synth):
    """Term 0 holds about half of all docs (bitset blocks): most candidates are excluded."""
    qs = [[3], [2, 5], [1, 4, 9, 11], [6, 7]]
    xs = [[0], [0], [0, 1], [0, 2, 3]]
    check(synth["reader"], [synth["oseg"]], sdb.OR, qs, xs, sdb.BM25(), 100)
    check(synth["reader"], [synth["oseg"]], sdb.AND, [[1, 2], [3, 4]], [[0], [0]], sdb.BM25(), 100)


@pytest.mark.parametrize("which", ["natural", "uniform"])
def test_three_segments(which):
    segs = natural_segments() if which == "natural" else uniform_segments()[1]
    corpus = Corpus(segs)
    reader = sdb.IndexReader([to_gpu(o) for o in corpus.osegs], corpus.docs_with_field, corpus.total_term_freq,
                             corpus.docs_with_term)
    nt = corpus.n_terms
    rng = np.random.default_rng(12)
    qs, xs = _random_queries(rng, nt, (1, 2, 3, 4), (1, 2), 20)
    check(reader, corpus.osegs, sdb.OR, qs, xs, sdb.BM25(), 10)
    qs, xs = _random_queries(rng, nt, (2, 3), (1, 1), 10)
    check(reader, corpus.osegs, sdb.AND, qs, xs, sdb.BM25(), 10)


def test_lead_mode_shaped_pair():
    """Long list >= 4x the short one, short >= 3k: without exclusions this pair runs in lead mode; with one it must
    run in the stream kernel with per-doc checks and still equal the exhaustive result."""
    n = 1_000_000
    oseg, dl, lists = orc.synth_segment(n, [0, 40, 3])
    g = to_gpu(oseg)
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d, _ in lists])
    assert len(lists[0][0]) >= 4 * len(lists[1][0]) and len(lists[1][0]) >= 3 * 100
    check(reader, [oseg], sdb.OR, [[0, 1]] * 2, [[2], [1]], sdb.BM25(), 100)


def _scan_excl(g, terms, excl, kind, doc_min, doc_max, cap, docs=None, scores=None):
    x = np.ascontiguousarray(excl, np.uint32)
    n = C.c_uint64(0)
    arr = (N.BM25Term * len(terms))(*terms)
    rc = N.lib().sdbg_bm25_scan_excl(g._h, kind, arr, len(terms), x.ctypes.data_as(C.c_void_p) if len(x) else None, len(x),
                                     1.2, 0.75, None, doc_min, doc_max,
                                     docs.ctypes.data_as(C.c_void_p) if docs is not None else None,
                                     scores.ctypes.data_as(C.c_void_p) if scores is not None else None, cap, C.byref(n))
    return rc, n.value


def test_streaming_scan(synth):
    reader, oseg, g, n = synth["reader"], synth["oseg"], synth["g"], synth["n"]
    scorer = sdb.BM25()
    for kind, q, x in ((sdb.OR, [1, 4], [2]), (sdb.OR, [3, 5, 6, 9], [0, 7]), (sdb.AND, [0, 1, 2], [5]), (sdb.OR, [5], [5])):
        allh, tot = topk_excl([oseg], _okind(kind), oracle_terms(reader, scorer, q), x, n)
        order = np.argsort(allh["doc"], kind="stable")
        ed, es = allh["doc"][order], allh["score"][order]
        d, s = sdb.StreamScoredDocs(reader, 0, q, kind, scorer, exclude=x)
        assert np.array_equal(d, ed) and np.array_equal(s.view(np.uint32), es.view(np.uint32))
        for lo, hi in ((1, 5000), (77_777, 123_457), (150_000, n + 1)):
            d, s = sdb.StreamScoredDocs(reader, 0, q, kind, scorer, doc_min=lo, doc_max=hi, exclude=x)
            m = (ed >= lo) & (ed < hi)
            assert np.array_equal(d, ed[m]) and np.array_equal(s.view(np.uint32), es[m].view(np.uint32))
        rc, cnt = _scan_excl(g, [reader.stats(scorer, t) for t in q], x, kind, 1, 0xFFFFFFFF, 0)
        assert cnt == tot == len(ed) and rc == (-6 if tot else 0)       # count-only form: ECAPACITY with the room needed


def test_empty_set_is_the_plain_query_and_self_exclusion(synth):
    reader, oseg = synth["reader"], synth["oseg"]
    scorer = sdb.BM25()
    qs = [[0, 3], [1], [2, 5, 7], [0, 1, 2, 3, 4, 5]]
    for kind in (sdb.OR, sdb.AND):
        for lvl in LEVELS:
            ctx().set_wand(lvl)
            terms, off = sdb.engine._flatten_queries(reader, qs, scorer)
            xoff = np.zeros(len(qs) + 1, np.uint32)
            outs = []
            for fn in ("sdbg_bm25_topk_batch", "sdbg_bm25_topk_batch_excl"):
                hits = np.zeros((len(qs), 50), sdb.engine.HIT_DTYPE)
                n_out, total = np.zeros(len(qs), np.uint32), np.zeros(len(qs), np.uint64)
                extra = [None, xoff.ctypes.data_as(C.c_void_p)] if fn.endswith("excl") else []
                N.check(getattr(N.lib(), fn)(sdb.engine._seg_array(reader.segments), 1, kind, terms, off.ctypes.data_as(C.c_void_p),
                                             len(qs), *extra, scorer.k, scorer.b, None, 50, sdb.FLT_MIN,
                                             hits.ctypes.data_as(C.c_void_p), n_out.ctypes.data_as(C.c_void_p),
                                             total.ctypes.data_as(C.c_void_p)), ctx()._h)
                outs.append((hits, n_out, total))
            assert np.array_equal(outs[0][1], outs[1][1])
            if lvl == 0:      # with pruning the count depends on when other chains raise the threshold: not repeatable
                assert np.array_equal(outs[0][2], outs[1][2])
            for q in range(len(qs)):
                assert_hits_equal(outs[1][0][q, :outs[1][1][q]], outs[0][0][q, :outs[0][1][q]])
    ctx().set_wand(0)
    # an excluded term that is also positive: AND -> nothing, OR -> the other terms' docs outside its list
    for lvl in LEVELS:
        ctx().set_wand(lvl)
        h, t = sdb.ExecuteTopK(reader, [0, 3], sdb.AND, scorer, 50, exclude=[3])
        assert len(h) == 0 and t == 0
    ctx().set_wand(0)
    tot = check(reader, [oseg], sdb.OR, [[0, 3], [2, 5, 7]], [[3], [2, 5]], scorer, 50)
    d0, d3 = set(synth["lists"][0][0].tolist()), set(synth["lists"][3][0].tolist())
    assert tot[0] == len(d0 - d3)


def test_errors(synth):
    reader = synth["reader"]
    with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
        sdb.ExecuteTopK(reader, [0, 1], sdb.OR, sdb.BM25(), 10, exclude=list(range(2, 19)))
    with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
        sdb.StreamScoredDocs(reader, 0, [0, 1], sdb.OR, sdb.BM25(), exclude=list(range(2, 19)))
    terms, off = sdb.engine._flatten_queries(reader, [[0], [1]], sdb.BM25())
    hits = np.zeros((2, 10), sdb.engine.HIT_DTYPE)
    n_out, total = np.zeros(2, np.uint32), np.zeros(2, np.uint64)
    x = np.array([3, 4], np.uint32)
    for xoff, xp in ((np.array([0, 2, 1], np.uint32), x), (np.array([0, 1, 2], np.uint32), None)):
        rc = N.lib().sdbg_bm25_topk_batch_excl(sdb.engine._seg_array(reader.segments), 1, sdb.OR, terms, off.ctypes.data_as(C.c_void_p),
                                               2, xp.ctypes.data_as(C.c_void_p) if xp is not None else None,
                                               xoff.ctypes.data_as(C.c_void_p), 1.2, 0.75, None, 10, sdb.FLT_MIN,
                                               hits.ctypes.data_as(C.c_void_p), n_out.ctypes.data_as(C.c_void_p),
                                               total.ctypes.data_as(C.c_void_p))
        assert rc == -1                                                                   # EINVAL
    rc, _ = _scan_excl(synth["g"], [reader.stats(sdb.BM25(), 0)], [], sdb.OR, 1, 100, 0)
    assert rc in (0, -6)
    n = C.c_uint64(0)
    t1 = (N.BM25Term * 1)(reader.stats(sdb.BM25(), 0))
    assert N.lib().sdbg_bm25_scan_excl(synth["g"]._h, sdb.OR, t1, 1, None, 2, 1.2, 0.75, None, 1, 100, None, None, 0, C.byref(n)) == -1


def test_adapter_with_excluded_terms():
    from serenedb_b200 import build as b
    exe = b.build_adapters()
    n = 200_000
    res = subprocess.run([exe, str(n), "excl"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = [json.loads(l) for l in res.stdout.strip().splitlines()]
    assert [x["filter"] for x in lines] == [0, 1]
    oseg, dc, sum_dl = orc.synth_segment_mt(n, 0, 8, threads=4)
    oseg.add_column(9, orc.synth_column(2, 1, 1, n).astype(np.int32))
    terms = []
    for t in (2, 5):
        st = orc.bm25_stats(n, sum_dl, int(dc[t]))
        x = orc.BM25Term()
        x.idf, x.norm_const, x.norm_length, x.boost, x.term = st.idf, st.norm_const, st.norm_length, 1.0, t
        terms.append(x)
    for out in lines:
        filt = orc.make_pred(9, "BETWEEN", 250000, 749999) if out["filter"] else None
        oh, ototal = topk_excl([oseg], "OR", terms, [3], 100, filt=filt)
        assert [d for d, _ in out["topk"]] == oh["doc"].tolist()
        assert np.array_equal(np.array([s for _, s in out["topk"]], np.float32), oh["score"])
        assert out["total"] <= ototal                                        # the selftest runs with pruning on
        assert np.float32(out["threshold"]) == oh["score"][-1]
        allh, alltotal = topk_excl([oseg], "OR", terms, [3], n, filt=filt)
        assert out["stream_n"] == alltotal == len(allh)
        assert out["stream_doc_sum"] == int(allh["doc"].astype(np.uint64).sum())
        assert out["stream_score_sum"] == pytest.approx(float(allh["score"].astype(np.float64).sum()), rel=1e-10)


def test_at_scale_pruned_equals_exhaustive():
    """2 M docs, 256 two-term disjunctions with one excluded term each: level 2 == level 0, hits and order."""
    n = 2_000_000
    nt = 64
    g = sdb.Segment(ctx(), n)
    dc, sum_dl = g.synth_corpus(0, 0, nt)
    reader = sdb.IndexReader([g], n, sum_dl, dc)
    rng = np.random.default_rng(2026)
    qs = [sorted(int(t) for t in rng.choice(nt, 2, replace=False)) for _ in range(256)]
    xs = [[int(rng.choice([t for t in range(nt) if t not in q]))] for q in qs]
    res = {}
    try:
        for lvl in (0, 2):
            ctx().set_wand(lvl)
            res[lvl] = sdb.ExecuteTopKBatch(reader, qs, sdb.OR, sdb.BM25(), 100, exclude=xs)
    finally:
        ctx().set_wand(0)
    (h0, n0, t0), (h2, n2, t2) = res[0], res[2]
    assert np.array_equal(n0, n2) and np.all(t2 <= t0)
    for q in range(len(qs)):
        assert_hits_equal(h2[q, :n2[q]], h0[q, :n0[q]])
