"""The match scan (Stream mode, sdbg_match_scan_batch_groups_min / ExecuteMatchScanGroupsBatch): every match of flat,
grouped, min-match and exclusion queries in (segment, doc) order, a LIMIT / OFFSET page per query, optionally scored.

Docs and totals are checked against the NumPy statements (min_match_reference.match_docs) and the count entry, over two
segments of different sizes with deleted docs, with and without filter chains of 2 and 4 predicates. Scores are checked
bit for bit against the oracle's exhaustive evaluation, the top-k entry at pruning level 0 and, for flat queries, the
per-segment streaming scan (StreamScoredDocs), under BM25, BM15, BM1, TFIDF and normalised TFIDF at pruning levels 0, 1
and 2. Then pages, batches, edges (doc ids up to 2^32 - 2, absent terms, empty results), the error codes, the C++
adapter and a sample of the 10 M-doc benchmark corpus."""
import ctypes as C
import json
import subprocess

import numpy as np
import pytest

import bench
import high_doc_reference as hd
import min_match_reference as mr
import orc
import serenedb_b200 as sdb
from gpu_util import ctx, oracle_terms, to_gpu
from serenedb_b200 import _native as N

pytestmark = pytest.mark.gpu

W = 1 << 16                       # docs per window of the count kernel
SIZES = (140_000, 70_000)         # two segments of different sizes
N_TERMS = 24


def _col(stream, row0, n):
    return orc.synth_column(stream, 1, row0 + 1, n).astype(np.int32)


@pytest.fixture(scope="module")
def two():
    """Two segments (doc ids drawn independently), deleted docs in both, int32 columns 8 and 9 for the filters."""
    osegs, gsegs, lists, deleted, cols = [], [], [], [], []
    sum_dl, dwt, row0 = 0, np.zeros(N_TERMS, np.uint64), 0
    rng = np.random.default_rng(5)
    for n in SIZES:
        oseg, dl, ls = orc.synth_segment(n, list(range(N_TERMS)), doc0=row0)
        c8, c9 = _col(5, row0, n), _col(2, row0, n)
        oseg.add_column(8, c8)
        oseg.add_column(9, c9)
        dele = np.unique(rng.integers(1, n + 1, n // 20)).astype(np.uint32)
        oseg.set_docs_mask(dele)
        g = to_gpu(oseg, columns={8: (c8, None), 9: (c9, None)})
        g.stage_docs_mask(dele)
        osegs.append(oseg)
        gsegs.append(g)
        lists.append([d for d, _ in ls])
        deleted.append(dele)
        cols.append({8: c8, 9: c9})
        sum_dl += int(dl.sum())
        dwt += np.array([len(d) for d, _ in ls], np.uint64)
        row0 += n
    reader = sdb.IndexReader(gsegs, sum(SIZES), sum_dl, dwt)
    return dict(osegs=osegs, reader=reader, lists=lists, deleted=deleted, cols=cols)


CHAINS = {
    None: [],
    "chain2": [(9, "BETWEEN", 200000, 799999), (8, "LT", 700000, 0)],
    "chain4": [(9, "BETWEEN", 100000, 899999), (8, "GE", 150000, 0), (9, "NE", 500000, 0), (8, "LE", 850000, 0)],
}


def _mask(vals, op, lo, hi):
    return {"BETWEEN": (vals >= lo) & (vals <= hi), "LT": vals < lo, "GE": vals >= lo, "NE": vals != lo,
            "LE": vals <= lo}[op]


def _filt(chain):
    return [sdb.pred(f, op, lo, hi) for f, op, lo, hi in CHAINS[chain]] or None


def _masks(S, chain):
    out = []
    for cols in S["cols"]:
        m = None
        for f, op, lo, hi in CHAINS[chain]:
            x = _mask(cols[f], op, lo, hi)
            m = x if m is None else m & x
        out.append(m)
    return out


def _want(S, groups, excl, mins, chain=None):
    """(seg, doc) of the NumPy statement, in (segment, doc) order."""
    segs, docs = [], []
    for si, (lists, dele, m) in enumerate(zip(S["lists"], S["deleted"], _masks(S, chain))):
        d = mr.match_docs(lists, groups, excl, dele, m, mins)
        segs.append(np.full(len(d), si, np.uint32))
        docs.append(d)
    return np.concatenate(segs), np.concatenate(docs)


def _scan(reader, qs, scorer=None, xs=None, ms=None, filt=None, limit=None, offset=None):
    if limit is None:
        limit = max(int(sdb.ExecuteCountGroupsBatch(reader, qs, filt=filt, exclude=xs, min_match=ms).max()), 1)
    return sdb.ExecuteMatchScanGroupsBatch(reader, qs, scorer, limit=limit, offset=offset, filt=filt, exclude=xs, min_match=ms)


def _queries():
    """(groups, excluded ids, group minimums): flat OR of 1, 4, 5 and 16 terms, AND of 1..16, `a & (b | c) & !d`,
    `2 of (a | b | c)`, nested min-match with exclusions."""
    q = [([[3]], [], None), ([[0, 5, 9, 14]], [], None), ([[1, 6, 11, 16, 21]], [7], None),
         ([list(range(4, 20))], [], None)]
    q += [([[t] for t in range(n)], [], None) for n in (1, 2, 3, 4, 8, 16)]
    q += [([[16], [10, 12]], [0], None), ([[9, 12, 15]], [], [2]), ([[2], [13, 14, 15, 17]], [4, 5], [1, 3]),
          ([[8, 9, 10, 11], [12, 13]], [1, 2], [2, 1]), ([[18, 16], [20, 22]], [23], None)]
    return q


def _split(q):
    return [g for g, _, _ in q], [x for _, x, _ in q], [m if m is not None else [1] * len(g) for g, _, m in q]


@pytest.mark.parametrize("chain", list(CHAINS), ids=["nofilter", "chain2", "chain4"])
def test_docs_and_totals_every_shape(two, chain):
    qs, xs, ms = _split(_queries())
    filt = _filt(chain)
    counts = sdb.ExecuteCountGroupsBatch(two["reader"], qs, filt=filt, exclude=xs, min_match=ms)
    res = _scan(two["reader"], qs, xs=xs, ms=ms, filt=filt)
    assert counts.sum() > 0
    for q, ((seg, doc, score), total) in enumerate(res):
        ws, wd = _want(two, qs[q], xs[q], ms[q], chain)
        assert total == counts[q] == len(wd), q
        assert np.array_equal(seg, ws) and np.array_equal(doc, wd), q
        assert not score.any()


SCORERS = [sdb.BM25(), sdb.BM25(1.2, 0.0), sdb.BM25(0.0, 0.75), sdb.TFIDF(False), sdb.TFIDF(True)]


def _oracle_scores(S, groups, excl, mins, scorer):
    """{(seg, doc): score} of the oracle's exhaustive evaluation of the query (every match)."""
    oq = [oracle_terms(S["reader"], scorer, g) for g in groups]
    k = max(mr.count(S["lists"], groups, excl, S["deleted"], mins=mins), 1)
    h, _ = mr.topk_groups(S["osegs"], oq, excl, k, k1=scorer.k, b=scorer.b, deleted=S["deleted"], mode=0, mins=mins)
    return {(int(s), int(d)): x for s, d, x in zip(h["seg"], h["doc"], h["score"].view(np.uint32))}


@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("scorer", SCORERS, ids=["bm25", "bm15", "bm1", "tfidf", "tfidf_norm"])
def test_scores_bit_exact(two, scorer, level):
    qs, xs, ms = _split(_queries())
    ref = [_oracle_scores(two, g, x, m, scorer) for g, x, m in zip(qs, xs, ms)]
    try:
        ctx().set_wand(level)
        res = _scan(two["reader"], qs, scorer, xs=xs, ms=ms)
    finally:
        ctx().set_wand(0)
    for q, ((seg, doc, score), total) in enumerate(res):
        ws, wd = _want(two, qs[q], xs[q], ms[q])
        assert total == len(wd) and np.array_equal(seg, ws) and np.array_equal(doc, wd), q
        # BM1 scores every doc 0, which the top-k collectors do not keep: those docs are not in the oracle's hits
        want = [ref[q].get((int(s), int(d)), 0 if scorer.k == 0 else None) for s, d in zip(seg, doc)]
        assert want == score.view(np.uint32).tolist(), q
    # the top-k entry at level 0 with k >= the matches: the same (doc, score) pairs
    small = [q for q in range(len(qs)) if 0 < res[q][1] <= 8192]
    assert small
    k = max(res[q][1] for q in small)
    h, n, t = sdb.ExecuteTopKGroupsBatch(two["reader"], [qs[q] for q in small], scorer, k, exclude=[xs[q] for q in small],
                                         min_match=[ms[q] for q in small])
    for i, q in enumerate(small):
        seg, doc, score = res[q][0]
        got = {(int(s), int(d)): x for s, d, x in zip(seg, doc, score.view(np.uint32))}
        top = {(int(s), int(d)): x for s, d, x in zip(h[i, :n[i]]["seg"], h[i, :n[i]]["doc"], h[i, :n[i]]["score"].view(np.uint32))}
        assert all(got[key] == x for key, x in top.items()), q
        assert len(top) == len(got) or scorer.k == 0, q


@pytest.mark.parametrize("chain", [None, "chain2"], ids=["nofilter", "chain2"])
def test_flat_queries_equal_the_streaming_scan(two, chain):
    """Flat OR of 1..4 terms and AND, with exclusions: segment by segment the same docs and scores as StreamScoredDocs."""
    reader, scorer = two["reader"], sdb.BM25()
    cases = [(sdb.OR, [2]), (sdb.OR, [0, 7]), (sdb.OR, [3, 9, 15]), (sdb.OR, [1, 4, 8, 20]), (sdb.AND, [0, 1, 5]),
             (sdb.AND, [2, 3]), (sdb.AND, list(range(6)))]
    for x in ([], [11]):
        for kind, tis in cases:
            (seg, doc, score), total = sdb.ExecuteMatchScanBatch(reader, [tis], kind, scorer, limit=1 << 18, filt=_filt(chain),
                                                                 exclude=[x])[0]
            assert total == len(doc)
            for si in range(len(SIZES)):
                sd, ss = sdb.StreamScoredDocs(reader, si, tis, kind, scorer, filt=_filt(chain), exclude=x)
                assert np.array_equal(doc[seg == si], sd)
                assert np.array_equal(score[seg == si].view(np.uint32), ss.view(np.uint32))


def _full(S, groups, scorer=None):
    (seg, doc, score), total = _scan(S["reader"], [groups], scorer)[0]
    return seg, doc, score, total


@pytest.mark.parametrize("L", [1, 7, 2048, 100_000])
def test_pages_concatenate(two, L):
    groups = [[16], [10, 12]] if L < 100 else [[0, 5, 9]]
    seg, doc, score, total = _full(two, groups, sdb.BM25())
    assert total > (3 * L if L < 100_000 else L)
    parts = []
    for off in range(0, total + L, L):
        (s, d, x), t = sdb.ExecuteMatchScanGroupsBatch(two["reader"], [groups], sdb.BM25(), limit=L, offset=[off])[0]
        assert t == total and len(d) == max(0, min(L, total - off))
        parts.append((s, d, x))
    assert np.array_equal(np.concatenate([p[0] for p in parts]), seg)
    assert np.array_equal(np.concatenate([p[1] for p in parts]), doc)
    assert np.array_equal(np.concatenate([p[2] for p in parts]).view(np.uint32), score.view(np.uint32))


def test_page_edges_and_per_query_offsets(two):
    """Pages that start and end at a 65 536-doc window edge, at the segment edge and inside a work item; offsets at and
    past the end; different offsets in one batch."""
    groups = [[0, 5, 9]]
    seg, doc, score, total = _full(two, groups, sdb.BM25())
    win = int(np.flatnonzero((seg == 0) & (doc >= W))[0])       # first match of segment 0's second window
    seg_edge = int(np.flatnonzero(seg == 1)[0])                  # first match of segment 1
    edges = [win, seg_edge, total // 3, total - 1]
    L = 5
    offs = [e for x in edges for e in (x, x - L, x - 2)] + [total, total + 10]
    res = sdb.ExecuteMatchScanGroupsBatch(two["reader"], [groups] * len(offs), sdb.BM25(), limit=L, offset=offs)
    for off, ((s, d, x), t) in zip(offs, res):
        assert t == total
        assert np.array_equal(s, seg[off:off + L]) and np.array_equal(d, doc[off:off + L]), off
        assert np.array_equal(x.view(np.uint32), score[off:off + L].view(np.uint32)), off
    assert len(res[-1][0][1]) == 0 and len(res[-2][0][1]) == 0


def test_mixed_batch_equals_shapes_and_single_queries(two):
    q = _queries()
    qs, xs, ms = _split(q)
    offs = [(7 * i) % 50 for i in range(len(qs))]
    for scorer in (None, sdb.BM25()):
        batch = _scan(two["reader"], qs, scorer, xs=xs, ms=ms, limit=3000, offset=offs)
        for i in range(len(qs)):
            alone = _scan(two["reader"], [qs[i]], scorer, xs=[xs[i]], ms=[ms[i]], limit=3000, offset=[offs[i]])[0]
            assert batch[i][1] == alone[1]
            for a, b in zip(batch[i][0], alone[0]):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), i
        # one shape at a time: flat ORs, ANDs, true groups
        for part in ([0, 1, 2, 3], [4, 5, 6, 7, 8, 9], [10, 11, 12, 13, 14]):
            sub = _scan(two["reader"], [qs[i] for i in part], scorer, xs=[xs[i] for i in part], ms=[ms[i] for i in part],
                        limit=3000, offset=[offs[i] for i in part])
            for j, i in enumerate(part):
                assert sub[j][1] == batch[i][1]
                for a, b in zip(sub[j][0], batch[i][0]):
                    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), i
    unscored = _scan(two["reader"], qs, None, xs=xs, ms=ms, limit=3000, offset=offs)
    scored = _scan(two["reader"], qs, sdb.BM25(), xs=xs, ms=ms, limit=3000, offset=offs)
    for (u, tu), (s, ts) in zip(unscored, scored):
        assert tu == ts and np.array_equal(u[0], s[0]) and np.array_equal(u[1], s[1]) and not u[2].any()


def test_absent_terms_and_no_matches():
    """Terms that hold no doc in one segment, and queries without a match."""
    n = 3 * W + 5
    o0, o1 = orc.Segment(n), orc.Segment(2 * W)
    t0 = np.arange(1, n + 1, 3, dtype=np.uint32)
    t1 = np.array([W, W + 1, n], np.uint32)
    t2 = np.array([2, 3], np.uint32)
    for d in (t0, t1, t2):
        o0.add_term(d, np.ones(len(d), np.uint32))
    s1 = [np.array([5, 2 * W], np.uint32), np.zeros(0, np.uint32), np.zeros(0, np.uint32)]   # terms 1 and 2: no doc here
    for d in s1:
        o1.add_term(d, np.ones(len(d), np.uint32))
    reader = sdb.IndexReader([to_gpu(o0), to_gpu(o1)], n + 2 * W, n + 2 * W, [len(t0) + 2, 3, 2])
    qs = [[[1]], [[0], [1]], [[0, 1]], [[1]], [[1], [2]], [[0, 2], [1]]]
    xs = [[], [], [0], [0], [], [0]]
    offs = [0, 0, 0, 1, 0, 0]
    res = sdb.ExecuteMatchScanGroupsBatch(reader, qs, sdb.BM25(), limit=100, exclude=xs, offset=offs)
    lists = [[t0, t1, t2], s1]
    for q, ((seg, doc, _), total) in enumerate(res):
        want = [(si, int(d)) for si in range(2) for d in mr.match_docs(lists[si], qs[q], xs[q])]
        assert total == len(want), q
        assert list(zip(seg.tolist(), doc.tolist())) == want[offs[q]:], q
    assert res[4][1] == 0 and len(res[4][0][1]) == 0          # t1 and t2 share no doc
    assert res[0][1] == 3 and res[1][1] == 1                  # term 1 holds no doc in segment 1


def test_high_doc_ids():
    """A segment of 2^32 - 2 docs whose lists reach the last valid doc id (tests/high_doc_reference.py): every match of
    each landmark list and of its pairs, in doc order, scored as the top-k entry scores it."""
    c = hd.TopCorpus()
    g = to_gpu(c.oracle_segment())
    try:
        reader = sdb.IndexReader([g], hd.TOP, hd.TOP, c.docs_with_term)
        singles = [[[t]] for t in c.shapes]
        counts = sdb.ExecuteCountGroupsBatch(reader, singles)
        res = sdb.ExecuteMatchScanGroupsBatch(reader, singles, None, limit=int(counts.max()))
        for t, ((seg, doc, _), total) in zip(c.shapes, res):
            assert total == len(doc) and np.array_equal(doc, np.unique(np.asarray(c.lists[t][1], np.uint32))), t
        assert max(int(r[0][1][-1]) for r in res if len(r[0][1])) == hd.TOP
        pairs = [[[t, t + 1]] for t in c.shapes if not c.lists[t][0].startswith("spread")]
        qs = [q for q, n in zip(singles + pairs, sdb.ExecuteCountGroupsBatch(reader, singles + pairs)) if 0 < n <= 8192]
        assert qs
        res = sdb.ExecuteMatchScanGroupsBatch(reader, qs, sdb.BM25(), limit=8192)
        h, n, t = sdb.ExecuteTopKGroupsBatch(reader, qs, sdb.BM25(), 8192)
        for i, ((seg, doc, score), total) in enumerate(res):
            assert total == t[i] == len(doc) and np.all(np.diff(doc.astype(np.int64)) > 0)
            order = np.argsort(h[i, :n[i]]["doc"], kind="stable")
            assert np.array_equal(doc, h[i, :n[i]]["doc"][order])
            assert np.array_equal(score.view(np.uint32), h[i, :n[i]]["score"][order].view(np.uint32))
        assert any(int(r[0][1][-1]) > 2 ** 31 for r in res if len(r[0][1]))
    finally:
        g.close()


def _raw(reader, ids, group_off, qgo, nq, limit=10, scored=1, out=True, n_out=True, total=True, excl=None, excl_off=None):
    arr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    terms = (N.BM25Term * max(len(ids), 1))()
    for i, t in enumerate(ids):
        terms[i] = reader.stats(sdb.BM25(), 0)
        terms[i].term = int(t)
    hits = np.zeros((max(nq, 1), max(limit, 1)), sdb.engine.HIT_DTYPE)
    no, tt = np.zeros(max(nq, 1), np.uint32), np.zeros(max(nq, 1), np.uint64)
    return N.lib().sdbg_match_scan_batch_groups_min(
        sdb.engine._seg_array(reader.segments), len(reader.segments), terms, arr(group_off), arr(qgo), None, nq, arr(excl),
        arr(excl_off), 1.2, 0.75, None, None, limit, scored, arr(hits) if out else None, arr(no) if n_out else None,
        arr(tt) if total else None)


def test_errors_before_any_launch(two):
    reader = two["reader"]
    u = lambda *v: np.array(v, np.uint32)
    before = ctx().launches
    assert _raw(reader, u(0, 1), u(0, 1, 2), u(0, 2), 1, limit=0) == -1
    assert _raw(reader, u(0, 1), u(0, 1, 2), u(0, 2), 1, out=False) == -1
    assert _raw(reader, u(0, 1), u(0, 1, 2), u(0, 2), 1, n_out=False) == -1
    assert _raw(reader, u(0, 1), u(0, 1, 2), u(0, 2), 1, total=False) == -1
    assert _raw(reader, u(0, 1), u(0, 1, 2), u(0, 2), 0) == -1                                 # no query
    assert _raw(reader, u(0, 1), u(0, 1, 1, 2), u(0, 3), 1) == -1                              # empty group
    assert _raw(reader, u(0, 0), u(0, 1, 2), u(0, 2), 1) == -1                                 # a term twice
    assert _raw(reader, u(0, 10_000), u(0, 1, 2), u(0, 2), 1) == -1                            # term id out of range
    assert _raw(reader, np.arange(17, dtype=np.uint32), u(0, 17), u(0, 1), 1) == -7            # 17 positive terms
    assert _raw(reader, u(0), u(0, 1), u(0, 1), 1, excl=np.arange(1, 18, dtype=np.uint32), excl_off=u(0, 17)) == -7
    assert _raw(reader, u(0), u(0, 1), u(0, 1), 1, excl=u(1), excl_off=u(1, 0)) == -1         # decreasing excl_off
    nq = 65536                                                                                 # scored: the top-k limit
    ids = np.zeros(nq, np.uint32)
    assert _raw(reader, ids, np.arange(nq + 1, dtype=np.uint32), np.arange(nq + 1, dtype=np.uint32), nq, limit=1) == -7
    assert ctx().launches == before
    assert _raw(reader, ids, np.arange(nq + 1, dtype=np.uint32), np.arange(nq + 1, dtype=np.uint32), nq, limit=1,
                scored=0) == 0                                                                  # unscored: no such limit
    with pytest.raises(ValueError):
        sdb.ExecuteMatchScanGroupsBatch(reader, [[[0]]], None, offset=[1, 2])


def test_adapter_scan_rows():
    from serenedb_b200 import build as b
    exe = b.build_adapters()
    n = 200_000
    res = subprocess.run([exe, str(n), "scan"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    out = [json.loads(l) for l in res.stdout.strip().splitlines()]
    g = sdb.Segment(ctx(), n)
    dc, sum_dl = g.synth_corpus(0, 0, 8, threads=4)
    reader = sdb.IndexReader([g], n, sum_dl, dc)
    for o in out:
        chunks = o["chunks"]
        assert all(0 < c <= 2048 for c in chunks) and o["rows_after"] == 0
        (seg, doc, score), total = sdb.ExecuteMatchScanGroupsBatch(reader, [o["groups"]], sdb.BM25() if o["scored"] else None,
                                                                   limit=1 << 20, min_match=[o["mins"]])[0]
        assert sum(chunks) == total == len(o["docs"])
        assert o["docs"] == doc.tolist() and o["segs"] == seg.tolist()
        assert np.array_equal(np.array(o["scores"], np.float32).view(np.uint32), score.view(np.uint32))


def test_bench_corpus_sample_equals_streaming_scan():
    """32 queries of the benchmark's 10 M-doc corpus: a full drain and LIMIT 1000 OFFSET 5000 against StreamScoredDocs."""
    n = 10_000_000
    g = sdb.Segment(ctx(), n)
    try:
        dc, sum_dl = g.synth_corpus(0, 0, bench.N_TERMS, threads=16)
        reader = sdb.IndexReader([g], n, sum_dl, dc)
        qs = bench.make_queries(4096)
        qs = [qs[i] for i in np.random.default_rng(3).choice(len(qs), 32, replace=False)]
        scorer = sdb.BM25()
        full = sdb.ExecuteMatchScanBatch(reader, qs, sdb.OR, scorer, limit=int(sdb.ExecuteCountBatch(reader, qs, sdb.OR).max()))
        page = sdb.ExecuteMatchScanBatch(reader, qs, sdb.OR, scorer, limit=1000, offset=[5000] * len(qs))
        for q, tis in enumerate(qs):
            sd, ss = sdb.StreamScoredDocs(reader, 0, tis, sdb.OR, scorer)
            (seg, doc, score), total = full[q]
            assert total == len(sd) and np.array_equal(doc, sd) and not seg.any()
            assert np.array_equal(score.view(np.uint32), ss.view(np.uint32))
            (seg, doc, score), total = page[q]
            assert total == len(sd) and np.array_equal(doc, sd[5000:6000])
            assert np.array_equal(score.view(np.uint32), ss[5000:6000].view(np.uint32))
    finally:
        g.close()
