"""The BM25 top-k of group queries across GPUs (sdbg_dist_bm25_topk_batch_groups_min, DESIGN §5), with R ranks simulated
on one GPU: each rank is its own list of segments with an IndexReader that carries the corpus-wide statistics.
TopKGroupsDevice writes rank r's buffer into slice r of one torch buffer and merge_topk_groups_gathered merges all R, as
the dist entry does after its all-gather. The reference is the local ExecuteTopKGroupsBatch over the unsharded corpus,
which the single-GPU suites check: once (rank, ordinal within the rank) is mapped back to (segment, doc), the hits must
be equal with scores bit for bit, n_out equal, and the totals equal with pruning off (a lower bound of the exact total,
at least n_out, with it)."""
import ctypes as C

import numpy as np
import pytest

import serenedb_b200 as sdb
from gpu_util import ctx, metas_of
from serenedb_b200 import _native as N
from serenedb_b200._native import SdbgError
from shape_corpora import Corpus, natural_segments, uniform_segments

pytestmark = pytest.mark.gpu

FILT, FILT2 = 9, 10
MAX_DOC_ID = (1 << 32) - 2
KS = (1, 10, 1000, 8192)


def _stage(c, oseg, rng):
    g = sdb.Segment(c, oseg.n_docs)
    g.stage_postings(oseg.doc_bytes(), metas_of(oseg))
    if oseg.has_norms:
        g.stage_norms(*oseg.norm_bytes())
    g.stage_column(FILT, rng.integers(0, 100, oseg.n_docs).astype(np.int64))
    g.stage_column(FILT2, rng.integers(0, 100, oseg.n_docs).astype(np.int32))
    return g


def _env(c, corpus, ranks, seed):
    rng = np.random.default_rng(seed)
    gsegs = [_stage(c, o, rng) for o in corpus.osegs]
    reader = lambda segs: sdb.IndexReader(segs, corpus.docs_with_field, corpus.total_term_freq, corpus.docs_with_term)
    gbase = np.cumsum([0] + [o.n_docs for o in corpus.osegs])[:-1].astype(np.int64)
    return dict(readers=[reader([gsegs[j] for j in rk]) for rk in ranks], one=reader(gsegs), gsegs=gsegs,
                n_terms=corpus.n_terms, rank_base=np.array([gbase[rk[0]] for rk in ranks], np.int64), gbase=gbase)


def _cut(norms, lists, parts):
    """One corpus (norms, [(docs, freqs)]) cut by doc range into `parts` segments."""
    n = len(norms)
    cuts = [i * n // parts for i in range(parts + 1)]
    segs = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        sub = []
        for d, f in lists:
            m = (d > a) & (d <= b)
            sub.append(((d[m] - a).astype(np.uint32), f[m]))
        segs.append((norms[a:b].copy(), sub))
    return segs


@pytest.fixture(scope="module")
def uniform8():
    """8 doc-range ranks of one segment each."""
    _, parts, _ = uniform_segments(parts=8)
    return _env(ctx(), Corpus(parts), [[j] for j in range(8)], 1)


@pytest.fixture(scope="module")
def uneven():
    """rank 0: two segments; rank 1: one segment with deleted docs; rank 2: a segment where no term has a posting; rank 3:
    a one-doc segment without postings, then a segment with matches."""
    segs = natural_segments()
    rng = np.random.default_rng(3)
    empty = [(np.zeros(0, np.uint32), np.zeros(0, np.uint32))] * len(segs[0][1])
    one = lambda d: [(np.array([d], np.uint32), np.ones(1, np.uint32))]   # a term no query names
    segs.append((rng.integers(5, 50, 2000).astype(np.uint32), empty + one(1000)))
    segs.append((np.array([7], np.uint32), empty + one(1)))
    segs.append(natural_segments(seed=12)[2])
    env = _env(ctx(), Corpus(segs), [[0, 1], [2], [3], [4, 5]], 5)
    env["gsegs"][2].stage_docs_mask(np.unique(rng.integers(1, segs[2][0].size + 1, 5000)).astype(np.uint32))
    return env


@pytest.fixture(params=[0, 1, 2], ids=lambda v: f"wand{v}")
def level(request):
    ctx().set_wand(request.param)
    yield request.param
    ctx().set_wand(0)


def _batch(n_terms, seed, n=24):
    """(queries, exclude, min_match): flat ORs (one group), flat ANDs (single-term groups), nested groups, min-match
    groups, with exclusions on some: one batch of every shape."""
    rng = np.random.default_rng(seed)
    pick = lambda k: [int(t) for t in rng.choice(n_terms, size=k, replace=False)]
    qs, xs, ms = [], [], []
    for i in range(n):
        t = pick(4)
        shape = i % 4
        if shape == 0:
            q, m = [t[:2 + i % 2]], [1]
        elif shape == 1:
            q, m = [[t[0]], [t[1]]], [1, 1]
        elif shape == 2:
            q, m = [[t[0]], t[1:3]], [1, 1]
        else:
            q, m = [t[:3]], [2]
        qs.append(q)
        ms.append(m)
        xs.append([t[3]] if i % 3 == 0 else None)
    return qs, xs, ms


FILTERS = (None, [sdb.pred(FILT, "BETWEEN", 10, 79), sdb.pred(FILT2, "LT", 70)])


def _gather(env, qs, scorer, k, **kw):
    """Every rank's device buffer in one [R, words] torch buffer, as the all-gather leaves it."""
    import torch
    words = sdb.topk_groups_device_bytes(len(qs), k) // 8
    buf = torch.zeros((len(env["readers"]), words), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()      # the library works on its own non-blocking stream
    for r, reader in enumerate(env["readers"]):
        sdb.TopKGroupsDevice(reader, qs, scorer, k, buf[r].data_ptr(), **kw)
    ctx().sync()                  # the device forms do not wait: done before torch touches the buffer again
    return buf


def _merged(env, qs, scorer, k, **kw):
    buf = _gather(env, qs, scorer, k, **kw)
    return sdb.merge_topk_groups_gathered(ctx(), buf.data_ptr(), buf.shape[0], len(qs), k)


def _unsharded(env, qs, k, level, **kw):
    """The reference: the local entry over the unsharded corpus with pruning off (exact totals), then back to `level`."""
    ctx().set_wand(0)
    try:
        return sdb.ExecuteTopKGroupsBatch(env["one"], qs, sdb.BM25(), k, **kw)
    finally:
        ctx().set_wand(level)


def _assert_equal_unsharded(env, got, want, level):
    """Hits and n_out equal; totals equal at pruning level 0, else at most the exact total and at least n_out."""
    hits, n_out, total = got
    whits, wn, wtotal = want
    assert np.array_equal(n_out, wn)
    for q in range(len(n_out)):
        h, w = hits[q, :n_out[q]], whits[q, :wn[q]]
        g_ord = env["rank_base"][h["seg"].astype(np.int64)] + h["doc"].astype(np.int64)
        w_ord = env["gbase"][w["seg"].astype(np.int64)] + w["doc"].astype(np.int64)
        assert np.array_equal(g_ord, w_ord), q
        assert np.array_equal(h["score"].view(np.uint32), w["score"].view(np.uint32)), q
    if level == 0:
        assert np.array_equal(total, wtotal)
    else:
        assert np.all(total <= wtotal) and np.all(total >= n_out)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("corpus_name", ["uniform8", "uneven"])
def test_merge_equals_unsharded(request, corpus_name, k, level):
    env = request.getfixturevalue(corpus_name)
    qs, xs, ms = _batch(env["n_terms"], 7 + k)
    for filt in FILTERS:
        kw = dict(filt=filt, exclude=xs, min_match=ms)
        got = _merged(env, qs, sdb.BM25(), k, **kw)
        _assert_equal_unsharded(env, got, _unsharded(env, qs, k, level, **kw), level)


def test_each_shape_alone(uniform8):
    """A batch of one shape runs whole into the device buffer; a mixed one goes through the per-shape rows."""
    qs, xs, ms = _batch(uniform8["n_terms"], 3)
    for s in range(4):
        kw = dict(exclude=xs[s::4], min_match=ms[s::4])
        got = _merged(uniform8, qs[s::4], sdb.BM25(), 100, **kw)
        _assert_equal_unsharded(uniform8, got, sdb.ExecuteTopKGroupsBatch(uniform8["one"], qs[s::4], sdb.BM25(), 100, **kw), 0)


SCORERS = {"bm25": sdb.BM25(), "bm15": sdb.BM25(b=0.0), "bm1": sdb.BM25(k=0.0), "tfidf": sdb.TFIDF(),
           "tfidf_norm": sdb.TFIDF(normalize=True)}


@pytest.mark.parametrize("name", list(SCORERS))
@pytest.mark.parametrize("corpus_name", ["uniform8", "uneven"])
def test_scorers(request, corpus_name, name):
    env = request.getfixturevalue(corpus_name)
    scorer = SCORERS[name]
    qs, xs, ms = _batch(env["n_terms"], 31)
    for k in (10, 1000):
        for filt in FILTERS:
            kw = dict(filt=filt, exclude=xs, min_match=ms)
            got = _merged(env, qs, scorer, k, **kw)
            _assert_equal_unsharded(env, got, sdb.ExecuteTopKGroupsBatch(env["one"], qs, scorer, k, **kw), 0)
            if name == "bm1":   # every score 0: nothing beats the threshold FLT_MIN, but every match is counted
                assert not got[1].any() and got[2].any()


def test_ties_across_ranks():
    """Equal doc lengths and freqs: a doc holding one of the two terms scores like every other such doc, so the k-th score
    is shared by docs on several ranks and the kept ones must be the lowest (rank, ordinal)."""
    n = 8000
    d0 = np.arange(3, n + 1, 3, dtype=np.uint32)
    d1 = np.arange(5, n + 1, 5, dtype=np.uint32)
    lists = [(d0, np.ones(len(d0), np.uint32)), (d1, np.ones(len(d1), np.uint32))]
    env = _env(ctx(), Corpus(_cut(np.full(n, 10, np.uint32), lists, 8)), [[j] for j in range(8)], 2)
    qs = [[[0, 1]], [[0]], [[1], [0]], [[0, 1]]]
    ms = [[1], [1], [1, 1], [2]]
    for k in (1, 10, 600, 1000, 3000):
        got = _merged(env, qs, sdb.BM25(), k, min_match=ms)
        want = sdb.ExecuteTopKGroupsBatch(env["one"], qs, sdb.BM25(), k, min_match=ms)
        _assert_equal_unsharded(env, got, want, 0)
        if k >= 1000:
            kth = got[0]["score"][0, got[1][0] - 1]
            assert len(set(got[0]["seg"][0, :got[1][0]][got[0]["score"][0, :got[1][0]] == kth].tolist())) > 1


def test_twenty_ranks():
    _, parts, _ = uniform_segments(parts=20)
    env = _env(ctx(), Corpus(parts), [[j] for j in range(20)], 4)
    qs, xs, ms = _batch(env["n_terms"], 41)
    for k in (10, 1000):
        for filt in FILTERS:
            kw = dict(filt=filt, exclude=xs, min_match=ms)
            _assert_equal_unsharded(env, _merged(env, qs, sdb.BM25(), k, **kw),
                                    sdb.ExecuteTopKGroupsBatch(env["one"], qs, sdb.BM25(), k, **kw), 0)


def _single_doc_segment(n_docs):
    """A segment without norms whose only term holds its last doc (sparse: only the postings are stored)."""
    w = sdb.PostingsWriter(n_docs, has_wand=True)
    w.add_term(np.array([n_docs], np.uint32), np.array([2], np.uint32))
    doc, metas = w.finish()
    g = sdb.Segment(ctx(), n_docs)
    g.stage_postings(doc, metas)
    return g


def test_rank_of_the_largest_segment():
    """Rank 0 holds 2^32 - 2 docs and its hit is on the last one; rank 1's doc ties with it and goes after it."""
    big, small = _single_doc_segment(MAX_DOC_ID), _single_doc_segment(5)
    stats = (MAX_DOC_ID + 5, MAX_DOC_ID + 5, [2])
    env = dict(readers=[sdb.IndexReader([g], *stats) for g in (big, small)])
    for k in (1, 10):
        hits, n_out, total = _merged(env, [[[0]]], sdb.BM25(), k)
        assert n_out[0] == min(k, 2) and total[0] == 2
        assert (hits["seg"][0, 0], hits["doc"][0, 0]) == (0, MAX_DOC_ID)
        if k > 1:
            assert (hits["seg"][0, 1], hits["doc"][0, 1]) == (1, 5)
            assert hits["score"][0, 0] == hits["score"][0, 1]
        local, _, _ = sdb.ExecuteTopKGroupsBatch(env["readers"][0], [[[0]]], sdb.BM25(), 1)
        assert local["doc"][0, 0] == MAX_DOC_ID and local["score"][0, 0].view(np.uint32) == hits["score"][0, 0].view(np.uint32)
    big.close()
    small.close()


def test_agrees_with_flat_path(uniform8):
    """Flat queries within 15 ranks and 2^28 docs per rank: the hits of merge_gathered over PreparedBatch.run_device keys."""
    import torch
    rng = np.random.default_rng(8)
    for kind in (sdb.OR, sdb.AND):
        flat = [[int(t) for t in rng.choice(uniform8["n_terms"], 2 + i % 2, replace=False)] for i in range(16)]
        qs = [[q] for q in flat] if kind == sdb.OR else [[[t] for t in q] for q in flat]
        for k in (10, 1000):
            keys = torch.zeros((8, len(flat), k), dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            for r, reader in enumerate(uniform8["readers"]):
                sdb.PreparedBatch(reader, flat, kind, sdb.BM25(), k).run_device(r, keys[r].data_ptr())
            want, wn = sdb.merge_gathered(ctx(), keys.data_ptr(), 8, len(flat), k)
            hits, n_out, _ = _merged(uniform8, qs, sdb.BM25(), k)
            assert np.array_equal(n_out, wn)
            for q in range(len(flat)):
                assert np.array_equal(hits[q, :n_out[q]], want[q, :wn[q]]), (kind, k, q)


def test_world_one_equals_local(uneven):
    """Without sdbg_dist_init the all-gather is a copy: hits of the whole corpus with seg = 0, doc = segment base + doc."""
    qs, xs, ms = _batch(uneven["n_terms"], 17)
    reader = uneven["one"]
    for k in (10, 1000):
        for filt in FILTERS:
            kw = dict(filt=filt, exclude=xs, min_match=ms)
            hits, n_out, total = sdb.ExecuteDistTopKGroupsBatch(reader, qs, sdb.BM25(), k, **kw)
            whits, wn, wtotal = sdb.ExecuteTopKGroupsBatch(reader, qs, sdb.BM25(), k, **kw)
            assert np.array_equal(n_out, wn) and np.array_equal(total, wtotal)
            for q in range(len(qs)):
                h, w = hits[q, :n_out[q]], whits[q, :wn[q]]
                assert np.all(h["seg"] == 0)
                assert np.array_equal(h["doc"].astype(np.int64), uneven["gbase"][w["seg"]] + w["doc"])
                assert np.array_equal(h["score"].view(np.uint32), w["score"].view(np.uint32))


def _expect_rejected(code, fn):
    before = ctx().launches
    with pytest.raises(SdbgError, match="^" + code):
        fn()
    assert ctx().launches == before, "a rejected call queued work"


def test_errors_queue_nothing(uniform8):
    import torch
    reader = uniform8["readers"][0]
    qs = [[[0, 1]], [[2], [3]]]
    buf = torch.zeros((2, sdb.topk_groups_device_bytes(2, 8193) // 8), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    p = buf.data_ptr()
    for k, code in ((0, "EINVAL"), (8193, "EUNSUPPORTED")):
        _expect_rejected(code, lambda: sdb.TopKGroupsDevice(reader, qs, sdb.BM25(), k, p))
        _expect_rejected(code, lambda: sdb.merge_topk_groups_gathered(ctx(), p, 2, 2, k))
        _expect_rejected(code, lambda: sdb.ExecuteDistTopKGroupsBatch(reader, qs, sdb.BM25(), k))
    _expect_rejected("EINVAL", lambda: sdb.merge_topk_groups_gathered(ctx(), p, 0, 2, 10))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.merge_topk_groups_gathered(ctx(), p, 1 << 19, 2, 8192))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.merge_topk_groups_gathered(ctx(), p, (1 << 32) // 10 + 1, 2, 10))
    segs = (C.c_void_p * 1)(reader.segments[0]._h)
    out = np.zeros(10, sdb.engine.HIT_DTYPE)
    n_out, total = np.zeros(1, np.uint32), np.zeros(1, np.uint64)
    _expect_rejected("EINVAL", lambda: N.check(N.lib().sdbg_dist_bm25_topk_batch_groups_min(
        segs, 1, None, None, None, None, 1, None, None, 1.2, 0.75, None, 10, 0.0, out.ctypes.data_as(C.c_void_p),
        n_out.ctypes.data_as(C.c_void_p), total.ctypes.data_as(C.c_void_p)), ctx()._h))


def test_bad_headers_and_rank_failures(uniform8):
    import torch
    env = dict(uniform8, readers=uniform8["readers"][:3], rank_base=uniform8["rank_base"][:3])
    qs = [[[0, 1]], [[2], [3]]]
    for word, value in ((0, 11), (1, 3), (2, 1)):   # k, n_queries, failure word
        buf = _gather(env, qs, sdb.BM25(), 10)
        buf[2, word] = value
        torch.cuda.synchronize()
        _expect_rejected("EINVAL", lambda: sdb.merge_topk_groups_gathered(ctx(), buf.data_ptr(), 3, len(qs), 10))
    one = uniform8["one"]
    first3 = sdb.IndexReader(one.segments[:3], one.docs_with_field, one.total_term_freq, one.docs_with_term)
    buf = _gather(env, qs, sdb.BM25(), 10)
    _assert_equal_unsharded(env, sdb.merge_topk_groups_gathered(ctx(), buf.data_ptr(), 3, len(qs), 10),
                            sdb.ExecuteTopKGroupsBatch(first3, qs, sdb.BM25(), 10), 0)
    with pytest.raises(SdbgError, match="^EINVAL"):   # a term id rank 1 does not hold
        sdb.TopKGroupsDevice(_with_unknown_term(env["readers"][1]), [[[0, 999]], [[2], [3]]], sdb.BM25(), 10, buf[1].data_ptr())
    _expect_rejected("EINVAL", lambda: sdb.merge_topk_groups_gathered(ctx(), buf.data_ptr(), 3, len(qs), 10))


def _with_unknown_term(reader):
    """The reader with statistics for term ids up to 999, which its segments do not hold."""
    dwt = np.zeros(1000, np.uint64)
    dwt[:len(reader.docs_with_term)] = reader.docs_with_term
    return sdb.IndexReader(reader.segments, reader.docs_with_field, reader.total_term_freq, dwt)


# ---------------------------------------------------------------- NCCL at world size 1
@pytest.fixture(scope="module")
def nccl():
    c = sdb.Context(0)
    try:
        c.dist_init(sdb.Context.dist_unique_id(), 0, 1)
    except Exception as e:   # no NCCL library on this box
        c.close()
        pytest.skip("NCCL not available: %s" % e)
    _, parts, _ = uniform_segments(parts=2)
    c.set_wand(0)     # exact totals
    env = _env(c, Corpus(parts), [[0, 1]], 9)
    yield env
    for g in env["gsegs"]:
        g.close()
    c.close()


def test_nccl_world_one_equals_local(nccl):
    reader = nccl["one"]
    qs, xs, ms = _batch(nccl["n_terms"], 19)
    for filt in FILTERS:
        kw = dict(filt=filt, exclude=xs, min_match=ms)
        hits, n_out, total = sdb.ExecuteDistTopKGroupsBatch(reader, qs, sdb.BM25(), 100, **kw)
        whits, wn, wtotal = sdb.ExecuteTopKGroupsBatch(reader, qs, sdb.BM25(), 100, **kw)
        assert np.array_equal(n_out, wn) and np.array_equal(total, wtotal)
        for q in range(len(qs)):
            h, w = hits[q, :n_out[q]], whits[q, :wn[q]]
            assert np.all(h["seg"] == 0)
            assert np.array_equal(h["doc"].astype(np.int64), nccl["gbase"][w["seg"]] + w["doc"])
            assert np.array_equal(h["score"].view(np.uint32), w["score"].view(np.uint32))
    with pytest.raises(SdbgError, match="^EINVAL"):   # a bad term id fails this rank's pass; it still joins the gather
        sdb.ExecuteDistTopKGroupsBatch(_with_unknown_term(reader), [[[0, 999]]], sdb.BM25(), 10)
