"""OR groups with a minimum match count (`2 of (a | b | c) & d`, sdbg_bm25_topk_batch_groups_min /
sdbg_match_count_batch_groups_min) on the GPU against the oracle's exhaustive evaluation of the flat OR with the rejected
docs masked (tests/min_match_reference.py), bit for bit (doc, segment, fp32 score), at pruning
levels 0, 1 and 2: hits equal at every level, total_matches exact at level 0 and never above it with pruning; counts equal
the NumPy statement and the level-0 totals. Covers the stream kernel with the pigeonhole lead (`m of n`, n <= 4) and with
a min-match group inside an AND, the legacy window kernel (5..16 terms, BM15, BM1, TFIDF), the hybrid filter, deleted docs
and exclusions, three segments with a group short of non-empty lists in one, every block encoding as a group member,
count window edges, the degenerate forms, the error codes, the C++ adapters and a 4096-query batch over 10 M docs."""
import ctypes as C
import json
import subprocess

import numpy as np
import pytest

import min_match_reference as mr
import orc
import serenedb_b200 as sdb
from serenedb_b200 import _native as N
from gpu_util import assert_hits_equal, ctx, oracle_terms, to_gpu
from shape_corpora import NORM_WIDTHS, Corpus, natural_segments, shape_segment

pytestmark = pytest.mark.gpu

LEVELS = (0, 1, 2)
W = 1 << 16   # docs per window of the count kernel


def check(reader, osegs, queries, mins, excludes, scorer, k, gfilt=None, ofilt=None, deleted=None, seg_lists=None,
          masks=None, levels=LEVELS):
    """GPU batch at each pruning level == the exhaustive reference; counts == level-0 totals (== the NumPy statement when
    seg_lists is given). Returns the level-0 totals."""
    oq = [[oracle_terms(reader, scorer, g) for g in q] for q in queries]
    oh, on, ot = mr.topk_batch_groups(osegs, oq, excludes, k, min_match=mins, k1=scorer.k, b=scorer.b, filt=ofilt,
                                      deleted=deleted)
    try:
        for lvl in levels:
            ctx().set_wand(lvl)
            gh, gn, gt = sdb.ExecuteTopKGroupsBatch(reader, queries, scorer, k, filt=gfilt, exclude=excludes, min_match=mins)
            for q in range(len(queries)):
                assert_hits_equal(gh[q, :gn[q]], oh[q, :on[q]])
                if lvl == 0:
                    assert gt[q] == ot[q], (lvl, q)
                else:
                    assert gt[q] <= ot[q], (lvl, q)
            counts = sdb.ExecuteCountGroupsBatch(reader, queries, filt=gfilt, exclude=excludes, min_match=mins)
            assert np.array_equal(counts, ot), lvl
    finally:
        ctx().set_wand(0)
    if seg_lists is not None:
        want = [mr.count(seg_lists, q, x or [], deleted, masks, mins=m) for q, x, m in zip(queries, excludes, mins)]
        assert ot.tolist() == want
    return ot


@pytest.fixture(scope="module")
def synth():
    n = 200_000
    oseg, dl, lists = orc.synth_segment(n, list(range(24)))
    g = to_gpu(oseg)
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d, _ in lists])
    return dict(oseg=oseg, g=g, reader=reader, n=n, lists=[d for d, _ in lists])


def _queries(rng, n_terms, shapes, count, excl=(0, 2)):
    """Random queries of the given shapes: each shape is a list of (group size, minimum) pairs."""
    qs, ms, xs = [], [], []
    for i in range(count):
        shape = shapes[i % len(shapes)]
        ids = [int(t) for t in rng.choice(n_terms, size=sum(s for s, _ in shape), replace=False)]
        q, o = [], 0
        for s, _ in shape:
            q.append(ids[o:o + s])
            o += s
        rest = [t for t in range(n_terms) if t not in ids]
        xs.append([int(t) for t in rng.choice(rest, size=int(rng.integers(excl[0], excl[1] + 1)), replace=False)])
        qs.append(q)
        ms.append([m for _, m in shape])
    return qs, ms, xs


STREAM = [[(3, 2)], [(4, 2)], [(4, 3)], [(1, 1), (3, 2)], [(2, 1), (2, 1)], [(3, 2), (1, 1)]]
LEGACY = [[(6, 3)], [(5, 2)], [(2, 1), (4, 3)], [(3, 2), (3, 2)], [(1, 1), (7, 4)]]
WIDE = [[(16, 8)], [(9, 5), (3, 1)], [(4, 2), (4, 3), (4, 2)], [(12, 11)]]


@pytest.mark.parametrize("shapes", [STREAM, LEGACY, WIDE], ids=["stream", "legacy5-8", "legacy9-16"])
def test_bm25_both_routes(synth, shapes):
    rng = np.random.default_rng(len(shapes) * 7 + len(shapes[0]))
    qs, ms, xs = _queries(rng, 12 if shapes is not WIDE else 24, shapes, 24)
    tot = check(synth["reader"], [synth["oseg"]], qs, ms, xs, sdb.BM25(), 100, seg_lists=[synth["lists"]])
    assert tot.sum() > 0


def test_pigeonhole_lead_shapes(synth):
    """`2 of 3`, `2 of 4`, `3 of 4` (the stream kernel probes their m - 1 longest lists from the start), and one such group
    inside an AND; top-1000 so that the threshold rises late."""
    qs = [[[0, 1, 2]], [[3, 4, 5, 6]], [[7, 8, 9, 10]], [[11], [12, 13, 14]], [[1, 5, 9]], [[2, 3, 4, 8]]]
    ms = [[2], [2], [3], [1, 2], [2], [3]]
    tot = check(synth["reader"], [synth["oseg"]], qs, ms, [[]] * len(qs), sdb.BM25(), 1000, seg_lists=[synth["lists"]])
    assert np.all(tot > 0)


@pytest.mark.parametrize("scorer", [sdb.BM25(1.2, 0.0), sdb.BM25(0.0, 0.75), sdb.TFIDF(False), sdb.TFIDF(True)],
                         ids=["bm15", "bm1", "tfidf", "tfidf_norm"])
def test_other_scorers_legacy_kernel(synth, scorer):
    rng = np.random.default_rng(3)
    qs, ms, xs = _queries(rng, 8, [[(3, 2)], [(1, 1), (3, 2)], [(5, 3)]], 12)
    check(synth["reader"], [synth["oseg"]], qs, ms, xs, scorer, 50)


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
    qs = [[[0, 3, 4]], [[1, 2], [5, 6, 7]], [[2], [5, 7, 9, 0]], [[0, 1, 3, 4, 6, 8]], [[4, 5, 6, 7], [8, 9]]]
    ms = [[2], [1, 2], [1, 3], [4], [2, 1]]
    xs = [[1], [4, 0], [], [2], [0, 1]]
    mask = (vals >= 200000) & (vals <= 799999)
    check(reader, [oseg], qs, ms, xs, sdb.BM25(), 100, gfilt=sdb.pred(9, "BETWEEN", 200000, 799999),
          ofilt=orc.make_pred(9, "BETWEEN", 200000, 799999), deleted=[deleted], seg_lists=seg_lists, masks=[mask])
    check(reader, [oseg], qs, ms, xs, sdb.BM25(), 100, deleted=[deleted], seg_lists=seg_lists)


def test_three_segments_with_a_group_short_in_one():
    segs = natural_segments()
    norms, lists = segs[1]
    lists[8] = (np.zeros(0, np.uint32), np.zeros(0, np.uint32))          # terms 8 and 9 hold no doc in segment 1
    lists[9] = (np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    corpus = Corpus(segs)
    reader = sdb.IndexReader([to_gpu(o) for o in corpus.osegs], corpus.docs_with_field, corpus.total_term_freq,
                             corpus.docs_with_term)
    seg_lists = [[np.asarray(d, np.uint32) for d, _ in l] for l in corpus.lists]
    rng = np.random.default_rng(12)
    qs, ms, xs = _queries(rng, 8, [[(3, 2)], [(1, 1), (4, 2)], [(6, 3)]], 12)
    qs += [[[8, 9, 0]], [[0], [8, 9, 1]], [[8, 9, 1, 2]], [[8, 9, 1, 2, 3]]]   # fewer than m non-empty lists in segment 1
    ms += [[2], [1, 2], [3], [3]]
    xs += [[], [2], [], [4]]
    check(reader, corpus.osegs, qs, ms, xs, sdb.BM25(), 10, seg_lists=seg_lists)


@pytest.fixture(scope="module", params=NORM_WIDTHS, ids=lambda w: f"norms{w or 0}")
def shapes(request):
    oseg, norms, lists = shape_segment(request.param)
    g = to_gpu(oseg)
    ttf = int(norms.astype(np.uint64).sum()) if norms is not None else oseg.n_docs
    reader = sdb.IndexReader([g], oseg.n_docs, ttf, [len(d) for _, d, _ in lists])
    return dict(oseg=oseg, g=g, reader=reader, lists=lists)


def test_every_encoding_as_group_member(shapes):
    """Each shape term in `2 of 3` with two companions (stream route), and in `3 of 5` next to a required term (legacy)."""
    lists = shapes["lists"]
    L = len(lists)
    seg_lists = [[d for _, d, _ in lists]]
    shape_ids = [t for t, (name, _, _) in enumerate(lists) if not name.endswith("+lead")]
    qs = [[[t, (t + 1) % L, (t + 3) % L]] for t in shape_ids]
    check(shapes["reader"], [shapes["oseg"]], qs, [[2]] * len(qs), [[]] * len(qs), sdb.BM25(), 100, seg_lists=seg_lists)
    qs = [[[(t + 5) % L], [t, t + 1, (t + 2) % L, (t + 4) % L, (t + 6) % L]] for t in shape_ids]
    xs = [[(t + 7) % L] for t in shape_ids]
    check(shapes["reader"], [shapes["oseg"]], qs, [[1, 3]] * len(qs), xs, sdb.BM25(), 100, seg_lists=seg_lists)


@pytest.mark.parametrize("n", [3 * W + 17, 4 * W + 31])
def test_count_window_edges(n):
    edge = [1, W - 1, W, W + 1, 2 * W - 1, 2 * W, 3 * W, n - 1, n]
    rng = np.random.default_rng(n)
    oseg = orc.Segment(n)
    lists = [np.unique(np.array(edge, np.uint32)),
             np.unique(np.concatenate([edge[::2], rng.integers(1, n + 1, 3000)])).astype(np.uint32),
             np.unique(np.concatenate([np.arange(W - 200, W + 200), np.arange(n - 300, n + 1)])).astype(np.uint32),
             np.unique(np.concatenate([np.flatnonzero(rng.random(n) < 0.4) + 1, edge])).astype(np.uint32),
             np.unique(np.concatenate([edge[1::2], rng.integers(1, n + 1, 500)])).astype(np.uint32)]
    for d in lists:
        oseg.add_term(d, np.ones(len(d), np.uint32))
    g = to_gpu(oseg)
    reader = sdb.IndexReader([g], n, n, [len(d) for d in lists])
    qs = [[[0, 1, 2]], [[0, 1, 2, 3]], [[1], [0, 2, 3]], [[0, 2, 4], [1, 3]], [[0, 1, 2, 3, 4]], [[4, 0, 2]]]
    ms = [[2], [3], [1, 2], [2, 1], [4], [2]]
    for xs in ([[]] * len(qs), [[3], [4], [], [], [], [1]]):
        want = [mr.count([lists], q, x, mins=m) for q, x, m in zip(qs, xs, ms)]
        assert sdb.ExecuteCountGroupsBatch(reader, qs, exclude=xs, min_match=ms).tolist() == want
    deleted = np.array([1, W - 1, W, n], np.uint32)
    g.stage_docs_mask(deleted)
    want = [mr.count([lists], q, deleted=[deleted], mins=m) for q, m in zip(qs, ms)]
    assert sdb.ExecuteCountGroupsBatch(reader, qs, min_match=ms).tolist() == want
    g.stage_docs_mask(None)


def test_degenerate_forms(synth):
    """group_min NULL and all-1 give exactly the groups entries' output; m = s gives the AND's."""
    reader, scorer = synth["reader"], sdb.BM25()
    nested = [[[0], [3, 4]], [[1, 2], [5, 6, 7]], [[2, 8, 9]], [[1], [4]]]
    xs = [[], [9], [1], []]
    ands = [[0, 3, 5], [2, 6], [1, 4, 7, 8]]
    for lvl in LEVELS:
        ctx().set_wand(lvl)
        gh, gn, gt = sdb.ExecuteTopKGroupsBatch(reader, nested, scorer, 50, exclude=xs)
        gc = sdb.ExecuteCountGroupsBatch(reader, nested, exclude=xs)
        for mins in (None, [[1] * len(q) for q in nested]):
            mh, mn, mt = sdb.ExecuteTopKGroupsBatch(reader, nested, scorer, 50, exclude=xs, min_match=mins)
            assert np.array_equal(mn, gn) and np.array_equal(mh, gh)
            if lvl == 0:                          # with pruning, totals are lower bounds that vary from run to run
                assert np.array_equal(mt, gt)
            assert np.array_equal(sdb.ExecuteCountGroupsBatch(reader, nested, exclude=xs, min_match=mins), gc)
        eh, en, et = sdb.ExecuteTopKBatch(reader, ands, sdb.AND, scorer, 50)
        as_min = [[q] for q in ands]
        mins = [[len(q)] for q in ands]
        mh, mn, mt = sdb.ExecuteTopKGroupsBatch(reader, as_min, scorer, 50, min_match=mins)
        assert np.array_equal(mn, en)
        if lvl == 0:
            assert np.array_equal(mt, et)
        for q in range(len(ands)):
            assert_hits_equal(mh[q, :mn[q]], eh[q, :en[q]])
        assert np.array_equal(sdb.ExecuteCountGroupsBatch(reader, as_min, min_match=mins), sdb.ExecuteCountBatch(reader, ands, sdb.AND))
        # a mixed batch: every query gives what it gives alone
        mixed = [[[0, 1, 2]], [[3], [4, 5]], [[6, 7, 8, 9, 10]], [[1], [2, 3, 4]]]
        mm = [[2], [1, 1], [5], [1, 2]]
        bh, bn, bt = sdb.ExecuteTopKGroupsBatch(reader, mixed, scorer, 50, min_match=mm)
        bc = sdb.ExecuteCountGroupsBatch(reader, mixed, min_match=mm)
        for q, (groups, m) in enumerate(zip(mixed, mm)):
            h, t = sdb.ExecuteTopKGroups(reader, groups, scorer, 50, min_match=m)
            assert_hits_equal(bh[q, :bn[q]], h)
            if lvl == 0:
                assert bt[q] == t == bc[q]
            assert bc[q] == sdb.ExecuteCountGroups(reader, groups, min_match=m)
    ctx().set_wand(0)


def _raw(reader, fn, ids, group_off, qgo, gmin, nq, k=10):
    arr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    segs = sdb.engine._seg_array(reader.segments)
    if fn == "count":
        out = np.zeros(max(nq, 1), np.uint64)
        return N.lib().sdbg_match_count_batch_groups_min(segs, len(reader.segments), arr(ids), arr(group_off), arr(qgo), arr(gmin),
                                                         nq, None, None, None, arr(out))
    terms = (N.BM25Term * max(len(ids), 1))()
    for i, t in enumerate(ids):
        terms[i] = reader.stats(sdb.BM25(), 0)
        terms[i].term = int(t)
    hits = np.zeros((max(nq, 1), k), sdb.engine.HIT_DTYPE)
    n_out, total = np.zeros(max(nq, 1), np.uint32), np.zeros(max(nq, 1), np.uint64)
    return N.lib().sdbg_bm25_topk_batch_groups_min(segs, len(reader.segments), terms, arr(group_off), arr(qgo), arr(gmin), nq,
                                                   None, None, 1.2, 0.75, None, k, sdb.FLT_MIN, arr(hits), arr(n_out), arr(total))


def test_errors(synth):
    reader = synth["reader"]
    u = lambda *v: np.array(v, np.uint32)
    ids = u(0, 1, 2)
    for fn in ("topk", "count"):
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2), u(1, 2), 1) == 0
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2), None, 1) == 0
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2), u(1, 0), 1) == -1                # m = 0
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2), u(1, 3), 1) == -1                # m > the group's size
        assert _raw(reader, fn, ids, u(0, 1, 3), u(0, 2), u(2, 1), 1) == -1
        assert _raw(reader, fn, ids, u(0, 1, 1, 3), u(0, 3), u(1, 1, 1), 1) == -1          # empty group, as before
        assert _raw(reader, fn, u(0, 1, 0), u(0, 3), u(0, 1), u(2), 1) == -1               # a term twice in a query
        assert _raw(reader, fn, np.arange(17, dtype=np.uint32), u(0, 17), u(0, 1), u(2), 1) == -7   # 17 positive terms
        # a mixed batch whose shape-2 query has an out-of-range term: the valid shape-0 query is not run either
        before = ctx().launches
        assert _raw(reader, fn, u(0, 1, 2, 3, 10_000), u(0, 2, 3, 5), u(0, 1, 3), u(1, 1, 1), 2) == -1
        assert ctx().launches == before, fn
    with pytest.raises(N.SdbgError, match="EINVAL"):
        sdb.ExecuteTopKGroups(reader, [[0, 1, 2]], sdb.BM25(), 10, min_match=[4])
    with pytest.raises(N.SdbgError, match="EINVAL"):
        sdb.ExecuteCountGroups(reader, [[0, 1, 2]], min_match=[0])
    with pytest.raises(ValueError):
        sdb.ExecuteCountGroups(reader, [[0], [1, 2]], min_match=[1])


def test_adapters_with_min_match():
    from serenedb_b200 import build as b
    exe = b.build_adapters()
    n = 200_000
    res = subprocess.run([exe, str(n), "minmatch"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = [json.loads(l) for l in res.stdout.strip().splitlines()]
    assert lines[-1] == {"min_error": -1}                                     # a minimum above the group's size
    lines = lines[:-1]
    assert [(x["nested"], x["filter"]) for x in lines] == [(0, 0), (0, 1), (1, 0), (1, 1)]
    oseg, dc, sum_dl = orc.synth_segment_mt(n, 0, 8, threads=4)
    col = orc.synth_column(2, 1, 1, n).astype(np.int32)
    oseg.add_column(9, col)
    terms = {}
    for t in (1, 2, 5, 6):
        st = orc.bm25_stats(n, sum_dl, int(dc[t]))
        x = orc.BM25Term()
        x.idf, x.norm_const, x.norm_length, x.boost, x.term = st.idf, st.norm_const, st.norm_length, 1.0, t
        terms[t] = x
    lists = [oseg.decode_term(t)[0] for t in range(8)]
    mask = (col >= 250000) & (col <= 749999)
    for out in lines:
        filt = orc.make_pred(9, "BETWEEN", 250000, 749999) if out["filter"] else None
        gids, mins = ([[1], [2, 5, 6]], [1, 2]) if out["nested"] else ([[2, 5, 6]], [2])
        oh, ototal = mr.topk_groups([oseg], [[terms[t] for t in g] for g in gids], [], 100, filt=filt, mins=mins)
        assert [d for d, _ in out["topk"]] == oh["doc"].tolist()
        assert np.array_equal(np.array([s for _, s in out["topk"]], np.float32), oh["score"])
        assert out["total"] <= ototal                                        # the selftest runs with pruning on
        assert np.float32(out["threshold"]) == oh["score"][-1]
        assert out["count"] == ototal == mr.count([lists], gids, mins=mins, masks=[mask if out["filter"] else None])
        assert out["rows_after"] == 0


def test_bench_corpus_batch_pruned_equals_exhaustive():
    """The 10 M-doc benchmark corpus (256 terms), 4096 queries (`2 of (a | b | c)`, `3 of 4`, `a & 2 of (b | c | d)`, `3 of
    6`), top-1000: level 2 == level 0, hits and order; counts == level-0 totals."""
    n = 10_000_000
    nt = 256
    g = sdb.Segment(ctx(), n)
    dc, sum_dl = g.synth_corpus(0, 0, nt, threads=16)
    reader = sdb.IndexReader([g], n, sum_dl, dc)
    rng = np.random.default_rng(20261016)
    qs, ms = [], []
    forms = [([3], [2]), ([4], [3]), ([1, 3], [1, 2]), ([6], [3])]
    for i in range(4096):
        sizes, mins = forms[i % len(forms)]
        ids = [int(t) for t in rng.choice(nt, sum(sizes), replace=False)]
        q, o = [], 0
        for s in sizes:
            q.append(ids[o:o + s])
            o += s
        qs.append(q)
        ms.append(list(mins))
    res = {}
    try:
        for lvl in (0, 2):
            ctx().set_wand(lvl)
            res[lvl] = sdb.ExecuteTopKGroupsBatch(reader, qs, sdb.BM25(), 1000, min_match=ms)
        counts = sdb.ExecuteCountGroupsBatch(reader, qs, min_match=ms)
    finally:
        ctx().set_wand(0)
    (h0, n0, t0), (h2, n2, t2) = res[0], res[2]
    assert np.array_equal(n0, n2) and np.all(t2 <= t0)
    assert np.array_equal(counts, t0) and t0.sum() > 0
    for q in range(len(qs)):
        assert_hits_equal(h2[q, :n2[q]], h0[q, :n0[q]])
