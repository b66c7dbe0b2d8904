"""Conjunctions of OR groups (`a & (b | c) & !d`, sdbg_bm25_topk_batch_groups / sdbg_match_count_batch_groups) on the GPU
against the oracle's exhaustive evaluation of the flat OR with the rejected docs masked (tests/groups_reference.py), bit
for bit (doc, segment, fp32 score), at pruning levels 0, 1 and 2: total_matches exact at level 0 and never above it with
pruning; counts equal the NumPy statement and the level-0 totals. Covers the stream kernel (1..4 positive terms) and the
legacy window kernel (5..16 terms, BM15, BM1, TFIDF), the hybrid filter, deleted docs and exclusions, three segments
with a group that is empty in one of them, every block encoding as a group member, count window edges, the flat OR's
scores, the degenerate forms, the error codes, the C++ adapters and a 4096-query batch over 10 M docs."""
import ctypes as C
import json
import subprocess

import numpy as np
import pytest

import groups_reference as gr
import orc
import serenedb_b200 as sdb
from serenedb_b200 import _native as N
from gpu_util import assert_hits_equal, ctx, oracle_terms, to_gpu
from shape_corpora import NORM_WIDTHS, Corpus, natural_segments, shape_segment

pytestmark = pytest.mark.gpu

LEVELS = (0, 1, 2)
W = 1 << 16   # docs per window of the count kernel


def check(reader, osegs, queries, excludes, scorer, k, gfilt=None, ofilt=None, deleted=None, seg_lists=None, masks=None,
          levels=LEVELS):
    """GPU batch at each pruning level == the exhaustive reference; counts == level-0 totals (== the NumPy statement when
    seg_lists is given). Returns the level-0 totals."""
    oq = [[oracle_terms(reader, scorer, g) for g in q] for q in queries]
    oh, on, ot = gr.topk_batch_groups(osegs, oq, excludes, k, k1=scorer.k, b=scorer.b, filt=ofilt, deleted=deleted)
    try:
        for lvl in levels:
            ctx().set_wand(lvl)
            gh, gn, gt = sdb.ExecuteTopKGroupsBatch(reader, queries, scorer, k, filt=gfilt, exclude=excludes)
            for q in range(len(queries)):
                assert_hits_equal(gh[q, :gn[q]], oh[q, :on[q]])
                if lvl == 0:
                    assert gt[q] == ot[q], (lvl, q)
                else:
                    assert gt[q] <= ot[q], (lvl, q)
            counts = sdb.ExecuteCountGroupsBatch(reader, queries, filt=gfilt, exclude=excludes)
            assert np.array_equal(counts, ot), lvl
    finally:
        ctx().set_wand(0)
    if seg_lists is not None:
        want = [gr.count(seg_lists, q, x or [], deleted, masks) for q, x in zip(queries, excludes)]
        assert ot.tolist() == want
    return ot


@pytest.fixture(scope="module")
def synth():
    n = 200_000
    oseg, dl, lists = orc.synth_segment(n, list(range(24)))
    g = to_gpu(oseg)
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d, _ in lists])
    return dict(oseg=oseg, g=g, reader=reader, n=n, lists=[d for d, _ in lists])


def _random_groups(rng, n_terms, total, n_groups):
    ids = [int(t) for t in rng.choice(n_terms, size=total, replace=False)]
    cuts = sorted(rng.choice(np.arange(1, total), size=n_groups - 1, replace=False).tolist())
    return [ids[a:b] for a, b in zip([0] + cuts, cuts + [total])]


def _queries(rng, n_terms, totals, count, excl=(0, 2)):
    qs, xs = [], []
    for _ in range(count):
        total = int(rng.choice(totals))
        q = _random_groups(rng, n_terms, total, int(rng.integers(2, total)))    # fewer groups than terms: nested
        flat = [t for g in q for t in g]
        rest = [t for t in range(n_terms) if t not in flat]
        xs.append([int(t) for t in rng.choice(rest, size=int(rng.integers(excl[0], excl[1] + 1)), replace=False)])
        qs.append(q)
    return qs, xs


@pytest.mark.parametrize("totals", [(3, 4), (5, 6, 8), (9, 12, 16)], ids=["stream", "legacy5-8", "legacy9-16"])
def test_bm25_both_routes(synth, totals):
    rng = np.random.default_rng(sum(totals))
    qs, xs = _queries(rng, 12 if max(totals) <= 8 else 24, totals, 24)
    tot = check(synth["reader"], [synth["oseg"]], qs, xs, sdb.BM25(), 100, seg_lists=[synth["lists"]])
    assert tot.sum() > 0


@pytest.mark.parametrize("scorer", [sdb.BM25(1.2, 0.0), sdb.BM25(0.0, 0.75), sdb.TFIDF(False), sdb.TFIDF(True)],
                         ids=["bm15", "bm1", "tfidf", "tfidf_norm"])
def test_other_scorers_legacy_kernel(synth, scorer):
    rng = np.random.default_rng(3)
    qs, xs = _queries(rng, 8, (3, 4, 5), 12)
    check(synth["reader"], [synth["oseg"]], qs, xs, scorer, 50)


def test_filter_deleted_docs_and_exclusions():
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
    seg_lists = [[d for d, _ in lists]]
    qs = [[[0], [3, 4]], [[1, 2], [5, 6]], [[2], [5, 7], [9, 0, 1]], [[0], [1, 3]], [[4, 5, 6, 7], [8, 9]]]
    xs = [[1], [4, 0], [], [3], [0, 1, 2]]                  # [[0], [1, 3]] & !3: the group keeps term 1
    mask = (vals >= 200000) & (vals <= 799999)
    check(reader, [oseg], qs, xs, sdb.BM25(), 100, gfilt=sdb.pred(9, "BETWEEN", 200000, 799999),
          ofilt=orc.make_pred(9, "BETWEEN", 200000, 799999), deleted=[deleted], seg_lists=seg_lists, masks=[mask])
    check(reader, [oseg], qs, xs, sdb.BM25(), 100, deleted=[deleted], seg_lists=seg_lists)


def test_three_segments_with_a_group_empty_in_one():
    segs = natural_segments()
    norms, lists = segs[1]
    lists[9] = (np.zeros(0, np.uint32), np.zeros(0, np.uint32))          # term 9 holds no doc in segment 1
    corpus = Corpus(segs)
    reader = sdb.IndexReader([to_gpu(o) for o in corpus.osegs], corpus.docs_with_field, corpus.total_term_freq,
                             corpus.docs_with_term)
    seg_lists = [[np.asarray(d, np.uint32) for d, _ in l] for l in corpus.lists]
    rng = np.random.default_rng(12)
    qs, xs = _queries(rng, 9, (3, 4, 6), 16)
    qs += [[[9], [0, 1]], [[0], [9, 6]], [[9], [0], [1, 2, 3]]]
    xs += [[], [2], [4]]
    check(reader, corpus.osegs, qs, xs, sdb.BM25(), 10, seg_lists=seg_lists)


@pytest.fixture(scope="module", params=NORM_WIDTHS, ids=lambda w: f"norms{w or 0}")
def shapes(request):
    oseg, norms, lists = shape_segment(request.param)
    g = to_gpu(oseg)
    ttf = int(norms.astype(np.uint64).sum()) if norms is not None else oseg.n_docs
    reader = sdb.IndexReader([g], oseg.n_docs, ttf, [len(d) for _, d, _ in lists])
    return dict(oseg=oseg, g=g, reader=reader, lists=lists)


def test_every_encoding_as_group_member(shapes):
    """Each shape term in an OR group next to another list, required together with its companion (which shares ~15 % of
    its docs and adds misses), and as the companion's partner through both routes."""
    lists = shapes["lists"]
    L = len(lists)
    seg_lists = [[d for _, d, _ in lists]]
    shape_ids = [t for t, (name, _, _) in enumerate(lists) if not name.endswith("+lead")]
    qs = [[[t + 1], [t, (t + 3) % L]] for t in shape_ids]
    check(shapes["reader"], [shapes["oseg"]], qs, [[]] * len(qs), sdb.BM25(), 100, seg_lists=seg_lists)
    qs = [[[t, (t + 5) % L], [t + 1, (t + 2) % L, (t + 4) % L]] for t in shape_ids]             # 5 terms: legacy kernel
    xs = [[(t + 7) % L] for t in shape_ids]
    check(shapes["reader"], [shapes["oseg"]], qs, xs, sdb.BM25(), 100, seg_lists=seg_lists)


@pytest.mark.parametrize("n", [3 * W + 17, 4 * W + 31])
def test_count_window_edges(n):
    edge = [1, W - 1, W, W + 1, 2 * W - 1, 2 * W, 3 * W, n - 1, n]
    rng = np.random.default_rng(n)
    oseg = orc.Segment(n)
    lists = [np.unique(np.array(edge, np.uint32)),
             np.unique(np.concatenate([edge[::2], rng.integers(1, n + 1, 3000)])).astype(np.uint32),
             np.unique(np.concatenate([np.arange(W - 200, W + 200), np.arange(n - 300, n + 1)])).astype(np.uint32),
             np.unique(np.concatenate([np.flatnonzero(rng.random(n) < 0.4) + 1, edge])).astype(np.uint32)]
    for d in lists:
        oseg.add_term(d, np.ones(len(d), np.uint32))
    g = to_gpu(oseg)
    reader = sdb.IndexReader([g], n, n, [len(d) for d in lists])
    qs = [[[0], [1, 2]], [[1, 2], [3]], [[0, 3], [1, 2]], [[0], [2], [1, 3]], [[2], [0, 1]]]
    for xs in ([[]] * len(qs), [[3], [0], [], [], [1]]):
        want = [gr.count([lists], q, x) for q, x in zip(qs, xs)]
        assert sdb.ExecuteCountGroupsBatch(reader, qs, exclude=xs).tolist() == want
    deleted = np.array([1, W, n], np.uint32)
    g.stage_docs_mask(deleted)
    assert sdb.ExecuteCountGroupsBatch(reader, qs).tolist() == [gr.count([lists], q, deleted=[deleted]) for q in qs]
    g.stage_docs_mask(None)


def test_scores_are_the_flat_or_scores(synth):
    """Every hit scores as the flat OR of the query's terms scores that doc (the streaming scan of that OR)."""
    reader, scorer = synth["reader"], sdb.BM25()
    for q, x in (([[0], [3, 5]], []), ([[1, 2], [4, 7]], [9]), ([[6], [0], [2, 8]], [])):
        flat = [t for g in q for t in g]
        d, s = sdb.StreamScoredDocs(reader, 0, flat, sdb.OR, scorer)
        for lvl in LEVELS:
            ctx().set_wand(lvl)
            hits, _ = sdb.ExecuteTopKGroups(reader, q, scorer, 500, exclude=x)
            idx = np.searchsorted(d, hits["doc"])
            assert len(hits) and np.array_equal(d[idx], hits["doc"])
            assert np.array_equal(s[idx].view(np.uint32), hits["score"].view(np.uint32))
    ctx().set_wand(0)


def test_degenerate_forms_take_the_existing_paths(synth):
    reader, scorer = synth["reader"], sdb.BM25()
    ors = [[0, 3], [1], [2, 5, 7], [0, 1, 2, 3, 4, 5]]
    ands = [[0, 3], [2, 5, 7], [1, 4], [0, 1, 2, 3, 4, 5, 6]]
    nested = [[[0], [3, 4]], [[1, 2], [5, 6, 7]]]
    xs_or = [[4], [], [1], [9, 10]]
    xs_and = [[], [1], [8], []]
    for lvl in LEVELS:
        ctx().set_wand(lvl)
        for flat, kind, xs, as_groups in ((ors, sdb.OR, xs_or, [[q] for q in ors]),
                                          (ands, sdb.AND, xs_and, [[[t] for t in q] for q in ands])):
            eh, en, et = sdb.ExecuteTopKBatch(reader, flat, kind, scorer, 50, exclude=xs)
            gh, gn, gt = sdb.ExecuteTopKGroupsBatch(reader, as_groups, scorer, 50, exclude=xs)
            assert np.array_equal(en, gn)
            if lvl == 0:
                assert np.array_equal(et, gt)
            for q in range(len(flat)):
                assert_hits_equal(gh[q, :gn[q]], eh[q, :en[q]])
            assert np.array_equal(sdb.ExecuteCountGroupsBatch(reader, as_groups, exclude=xs),
                                  sdb.ExecuteCountBatch(reader, flat, kind, exclude=xs))
        # a mixed batch: every query gives what its own shape's batch gives
        mixed = [[ors[0]], nested[0], [[t] for t in ands[1]], nested[1], [ors[2]]]
        mx = [xs_or[0], [], xs_and[1], [2], xs_or[2]]
        mh, mn, mt = sdb.ExecuteTopKGroupsBatch(reader, mixed, scorer, 50, exclude=mx)
        mc = sdb.ExecuteCountGroupsBatch(reader, mixed, exclude=mx)
        for q, (groups, x) in enumerate(zip(mixed, mx)):
            h, t = sdb.ExecuteTopKGroups(reader, groups, scorer, 50, exclude=x)
            assert_hits_equal(mh[q, :mn[q]], h)
            if lvl == 0:
                assert mt[q] == t == mc[q]
            assert mc[q] == sdb.ExecuteCountGroups(reader, groups, exclude=x)
    ctx().set_wand(0)


def _raw(reader, fn, ids, group_off, qgo, nq, excl=None, xoff=None, k=10):
    arr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    segs = sdb.engine._seg_array(reader.segments)
    if fn == "count":
        out = np.zeros(max(nq, 1), np.uint64)
        return N.lib().sdbg_match_count_batch_groups(segs, len(reader.segments), arr(ids), arr(group_off), arr(qgo), nq, arr(excl),
                                                     arr(xoff), None, arr(out))
    terms = None
    if ids is not None:
        terms = (N.BM25Term * max(len(ids), 1))()
        for i, t in enumerate(ids):
            terms[i] = reader.stats(sdb.BM25(), 0)
            terms[i].term = int(t)
    hits = np.zeros((max(nq, 1), k), sdb.engine.HIT_DTYPE)
    n_out, total = np.zeros(max(nq, 1), np.uint32), np.zeros(max(nq, 1), np.uint64)
    return N.lib().sdbg_bm25_topk_batch_groups(segs, len(reader.segments), terms, arr(group_off), arr(qgo), nq, arr(excl), arr(xoff),
                                               1.2, 0.75, None, k, sdb.FLT_MIN, arr(hits), arr(n_out), arr(total))


def test_errors(synth):
    reader = synth["reader"]
    u = lambda *v: np.array(v, np.uint32)
    ids = u(0, 1, 2)
    for fn in ("topk", "count"):
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2), 1) == 0
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2), 0) == -1                        # no query
        assert _raw(reader, fn, None, u(0, 1, 3), u(0, 2), 1) == -1                       # NULL terms
        assert _raw(reader, fn, ids, None, u(0, 2), 1) == -1
        assert _raw(reader, fn, ids, u(0, 1, 3), None, 1) == -1
        assert _raw(reader, fn, ids, u(0, 1, 1, 3), u(0, 3), 1) == -1                     # empty group
        assert _raw(reader, fn, ids, u(0, 2, 1), u(0, 2), 1) == -1                        # decreasing group_off
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2, 1), 2) == -1                     # decreasing query_group_off
        assert _raw(reader, fn, u(0, 1, 0), u(0, 1, 3), u(0, 2), 1) == -1                 # a term twice in a query
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2), 1, None, u(0, 1)) == -1         # NULL excl_terms, non-empty range
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2), 1, u(3, 4), u(2, 1)) == -1      # decreasing excl_off
        g17 = np.arange(18, dtype=np.uint32)
        assert _raw(reader, fn, np.arange(17, dtype=np.uint32), g17, u(0, 17), 1) == -7   # 17 groups
        assert _raw(reader, fn, np.arange(17, dtype=np.uint32), u(0, 1, 17), u(0, 2), 1) == -7   # 17 positive terms
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2), 1, np.arange(3, 20, dtype=np.uint32), u(0, 17)) == -7
        assert _raw(reader, fn, u(0, 10_000), u(0, 1, 2), u(0, 2), 1) == -1               # term id out of range
        # a mixed batch whose shape-2 query has an out-of-range term: the valid shape-0 query is not run either
        before = ctx().launches
        assert _raw(reader, fn, u(0, 1, 2, 3, 10_000), u(0, 2, 3, 5), u(0, 1, 3), 2) == -1
        assert ctx().launches == before, fn
    with pytest.raises(N.SdbgError, match="EINVAL"):
        sdb.ExecuteTopKGroups(reader, [[0], []], sdb.BM25(), 10)
    with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
        sdb.ExecuteCountGroups(reader, [[t] for t in range(17)])


def test_adapters_with_groups():
    from serenedb_b200 import build as b
    exe = b.build_adapters()
    n = 200_000
    res = subprocess.run([exe, str(n), "groups"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = [json.loads(l) for l in res.stdout.strip().splitlines()]
    assert lines[-1] == {"stream_error": -7}                                  # k = 0 has no grouped form
    lines = lines[:-1]
    assert [(x["filter"], x["excl"]) for x in lines] == [(0, 0), (0, 1), (1, 0), (1, 1)]
    oseg, dc, sum_dl = orc.synth_segment_mt(n, 0, 8, threads=4)
    col = orc.synth_column(2, 1, 1, n).astype(np.int32)
    oseg.add_column(9, col)
    terms = {}
    for t in (2, 5, 6):
        st = orc.bm25_stats(n, sum_dl, int(dc[t]))
        x = orc.BM25Term()
        x.idf, x.norm_const, x.norm_length, x.boost, x.term = st.idf, st.norm_const, st.norm_length, 1.0, t
        terms[t] = x
    lists = [oseg.decode_term(t)[0] for t in range(8)]
    mask = (col >= 250000) & (col <= 749999)
    for out in lines:
        filt = orc.make_pred(9, "BETWEEN", 250000, 749999) if out["filter"] else None
        ex = [3] if out["excl"] else []
        oh, ototal = gr.topk_groups([oseg], [[terms[2]], [terms[5], terms[6]]], ex, 100, filt=filt)
        assert [d for d, _ in out["topk"]] == oh["doc"].tolist()
        assert np.array_equal(np.array([s for _, s in out["topk"]], np.float32), oh["score"])
        assert out["total"] <= ototal                                        # the selftest runs with pruning on
        assert np.float32(out["threshold"]) == oh["score"][-1]
        assert out["count"] == ototal == gr.count([lists], [[2], [5, 6]], ex, masks=[mask if out["filter"] else None])
        assert out["rows_after"] == 0


def test_bench_corpus_batch_pruned_equals_exhaustive():
    """The 10 M-doc benchmark corpus (256 terms), 4096 queries `a & (b | c)`, top-1000: level 2 == level 0, hits and order;
    counts == level-0 totals."""
    n = 10_000_000
    nt = 256
    g = sdb.Segment(ctx(), n)
    dc, sum_dl = g.synth_corpus(0, 0, nt, threads=16)
    reader = sdb.IndexReader([g], n, sum_dl, dc)
    rng = np.random.default_rng(20261015)
    qs = []
    for _ in range(4096):
        a, b_, c = (int(t) for t in rng.choice(nt, 3, replace=False))
        qs.append([[a], [b_, c]])
    res = {}
    try:
        for lvl in (0, 2):
            ctx().set_wand(lvl)
            res[lvl] = sdb.ExecuteTopKGroupsBatch(reader, qs, sdb.BM25(), 1000)
        counts = sdb.ExecuteCountGroupsBatch(reader, qs)
    finally:
        ctx().set_wand(0)
    (h0, n0, t0), (h2, n2, t2) = res[0], res[2]
    assert np.array_equal(n0, n2) and np.all(t2 <= t0)
    assert np.array_equal(counts, t0) and t0.sum() > 0
    for q in range(len(qs)):
        assert_hits_equal(h2[q, :n2[q]], h0[q, :n0[q]])
