"""Count mode (sdbg_match_count_batch, ExecuteCountBatch) on the GPU: counts equal the NumPy statement of the semantics
(tests/count_reference.py) and the exhaustive top-k's total_matches (pruning level 0). Covers OR of 1..16 terms and AND
of 2..16, the hybrid filter (int32 / int64 / float64 / nullable columns) and deleted docs, exclusions (every block
encoding as the excluded list, self-exclusion, absent ids), every block encoding as a positive list, docs on window
edges, three segments, sparse and skewed queries, every pruning level, the single-term shortcut, the error codes, the
C++ Count scan adapter and a 4096-query batch."""
import ctypes as C
import json
import subprocess

import numpy as np
import pytest

import count_reference as cr
import orc
import serenedb_b200 as sdb
from serenedb_b200 import _native as N
from gpu_util import ctx, metas_of, to_gpu
from shape_corpora import NORM_WIDTHS, Corpus, natural_segments, shape_segment

pytestmark = pytest.mark.gpu

W = 1 << 16   # docs per window of the count kernel


def level0_totals(reader, queries, kind, filt=None, exclude=None):
    ctx().set_wand(0)
    return sdb.ExecuteTopKBatch(reader, queries, kind, sdb.BM25(), 1, filt=filt, exclude=exclude)[2]


def check(reader, seg_lists, queries, kind, filt=None, exclude=None, deleted=None, masks=None, topk=True):
    got = sdb.ExecuteCountBatch(reader, queries, kind, filt=filt, exclude=exclude)
    okind = "AND" if kind == sdb.AND else "OR"
    xs = exclude or [[]] * len(queries)
    want = [cr.count(seg_lists, okind, q, x or [], deleted=deleted, masks=masks) for q, x in zip(queries, xs)]
    assert got.tolist() == want, (queries, exclude)
    if topk:
        assert np.array_equal(got, level0_totals(reader, queries, kind, filt, exclude))
    return got


@pytest.fixture(scope="module")
def synth():
    n = 200_000
    oseg, dl, lists = orc.synth_segment(n, list(range(24)))
    g = to_gpu(oseg)
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d, _ in lists])
    return dict(oseg=oseg, g=g, reader=reader, n=n, lists=[d for d, _ in lists])


def test_or_and_every_term_count(synth):
    rng = np.random.default_rng(1)
    qs_or = [sorted(rng.choice(24, size=t, replace=False).tolist()) for t in range(1, 17)]
    check(synth["reader"], [synth["lists"]], qs_or, sdb.OR)
    qs_and = [sorted(rng.choice(6, size=min(t, 6), replace=False).tolist()) + sorted(rng.choice(np.arange(6, 24), size=max(0, t - 6), replace=False).tolist())
              for t in range(2, 17)]
    got = check(synth["reader"], [synth["lists"]], qs_and, sdb.AND)
    assert got[0] > 0


def test_filter_and_deleted_docs():
    n = 150_000
    oseg, dl, lists = orc.synth_segment(n, list(range(10)))
    lists = [d for d, _ in lists]
    rng = np.random.default_rng(8)
    cols = {1: (orc.synth_column(2, 1, 1, n).astype(np.int32), None), 2: (orc.synth_column(3, 1, 1, n).astype(np.int64), None),
            3: (orc.synth_column(4, 2, 1, n), None), 4: (rng.integers(0, 1000, n).astype(np.int64), rng.random(n) < 0.6)}
    g = to_gpu(oseg, columns={f: (v, cr.validity_words(m) if m is not None else None) for f, (v, m) in cols.items()})
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d in lists])
    deleted = np.unique(rng.integers(1, n + 1, 9000)).astype(np.uint32)
    qs = [[0, 3], [1], [2, 5, 7, 9], [0, 1], [4]]
    preds = [(1, "BETWEEN", 200000, 799999), (2, "LT", 500000, 0), (3, "GE", 0.25, 0), (4, "GT", 300, 0), (4, "IS_NULL", 0, 0),
             (4, "IS_NOT_NULL", 0, 0)]
    for with_deleted in (False, True):
        g.stage_docs_mask(deleted if with_deleted else None)
        dele = [deleted] if with_deleted else None
        for kind in (sdb.OR, sdb.AND):
            check(reader, [lists], qs, kind, deleted=dele)
            for f, op, lo, hi in preds:
                m = cr.pred_mask(cols[f][0], cols[f][1], op, lo, hi)
                check(reader, [lists], qs, kind, filt=sdb.pred(f, op, lo, hi), deleted=dele, masks=[m])
    g.stage_docs_mask(None)


def test_exclusions(synth):
    reader, lists = synth["reader"], [synth["lists"]]
    rng = np.random.default_rng(5)
    qs, xs = [], []
    for ne in range(1, 17):
        q = sorted(rng.choice(8, size=2, replace=False).tolist())
        qs.append(q)
        xs.append(rng.choice([t for t in range(24) if t not in q], size=ne, replace=False).tolist())
    for kind in (sdb.OR, sdb.AND):
        check(reader, lists, qs, kind, exclude=xs)
    check(reader, lists, [[0, 3], [1]], sdb.OR, exclude=[[999], [5, 10_000]])          # ids the segment lacks
    got = check(reader, lists, [[0, 3], [2, 5, 7]], sdb.AND, exclude=[[3], [7]])         # self-exclusion empties an AND
    assert got.tolist() == [0, 0]
    got = check(reader, lists, [[0, 3], [2, 5, 7]], sdb.OR, exclude=[[3], [2, 5]])
    assert got[0] == len(np.setdiff1d(lists[0][0], lists[0][3]))


@pytest.fixture(scope="module", params=NORM_WIDTHS, ids=lambda w: f"norms{w or 0}")
def shapes(request):
    oseg, norms, lists = shape_segment(request.param)
    g = to_gpu(oseg)
    ttf = int(norms.astype(np.uint64).sum()) if norms is not None else oseg.n_docs
    reader = sdb.IndexReader([g], oseg.n_docs, ttf, [len(d) for _, d, _ in lists])
    return dict(oseg=oseg, g=g, reader=reader, lists=[d for _, d, _ in lists], names=[nm for nm, _, _ in lists])


def test_every_encoding(shapes):
    """Each shape term alone and with its companion, OR and AND; each shape term excluded from its companion. The
    segment without norms spans 2^30 docs: windows that hold no posting are skipped."""
    lists, names = shapes["lists"], shapes["names"]
    shape_ids = [t for t, nm in enumerate(names) if not nm.endswith("+lead")]
    singles = [[t] for t in shape_ids]
    pairs = [[t, t + 1] for t in shape_ids]
    check(shapes["reader"], [lists], singles, sdb.OR, topk=False)
    check(shapes["reader"], [lists], pairs, sdb.OR)
    check(shapes["reader"], [lists], pairs, sdb.AND)
    check(shapes["reader"], [lists], [[t + 1] for t in shape_ids], sdb.OR, exclude=[[t] for t in shape_ids])
    check(shapes["reader"], [lists], [[t + 1, (t + 3) % len(lists)] for t in shape_ids], sdb.AND, exclude=[[t] for t in shape_ids])


@pytest.mark.parametrize("n", [3 * W + 17, 4 * W, 4 * W + 31, 5 * W + 63])
def test_window_edges(n):
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
    qs = [[0], [0, 1], [0, 2], [1, 2, 3], [0, 3], [2, 3]]
    for kind in (sdb.OR, sdb.AND):
        check(reader, [lists], qs, kind)
        check(reader, [lists], qs, kind, exclude=[[3], [2], [1], [0], [1], [0]])
    deleted = np.array([1, W, n], np.uint32)
    g.stage_docs_mask(deleted)
    check(reader, [lists], qs, sdb.OR, deleted=[deleted])
    g.stage_docs_mask(None)


def test_three_segments():
    corpus = Corpus(natural_segments())
    reader = sdb.IndexReader([to_gpu(o) for o in corpus.osegs], corpus.docs_with_field, corpus.total_term_freq,
                             corpus.docs_with_term)
    seg_lists = [[np.asarray(d, np.uint32) for d, _ in l] for l in corpus.lists]
    rng = np.random.default_rng(12)
    qs = [sorted(rng.choice(corpus.n_terms, size=int(rng.integers(1, 5)), replace=False).tolist()) for _ in range(20)]
    xs = [[int(rng.integers(0, corpus.n_terms))] for _ in qs]
    for kind in (sdb.OR, sdb.AND):
        check(reader, seg_lists, qs, kind)
        check(reader, seg_lists, qs, kind, exclude=[[t for t in x if t not in q] for q, x in zip(qs, xs)])


def test_sparse_and_skewed():
    n = 2_000_000
    rng = np.random.default_rng(3)
    oseg = orc.Segment(n)
    lists = [np.sort(rng.choice(np.arange(1, n + 1), 5, replace=False)).astype(np.uint32),
             np.sort(rng.choice(np.arange(1, n + 1), 7, replace=False)).astype(np.uint32),
             (np.flatnonzero(rng.random(n) < 0.5) + 1).astype(np.uint32)]
    lists[0] = np.union1d(lists[0], lists[1][:2]).astype(np.uint32)
    for d in lists:
        oseg.add_term(d, np.ones(len(d), np.uint32))
    g = to_gpu(oseg)
    reader = sdb.IndexReader([g], n, n, [len(d) for d in lists])
    check(reader, [lists], [[0, 1]], sdb.OR)
    check(reader, [lists], [[0, 1], [0, 2], [1, 2]], sdb.AND)
    check(reader, [lists], [[0, 2]], sdb.OR, exclude=[[1]])


def test_pruning_level_does_not_matter(synth):
    qs = [[0, 3], [1, 4, 9], [2], [5, 6, 7, 8]]
    res = []
    for lvl in (0, 1, 2):
        ctx().set_wand(lvl)
        res.append([sdb.ExecuteCountBatch(synth["reader"], qs, k) for k in (sdb.OR, sdb.AND)])
    ctx().set_wand(0)
    for r in res[1:]:
        assert all(np.array_equal(a, b) for a, b in zip(r, res[0]))
    check(synth["reader"], [synth["lists"]], qs, sdb.OR)


def test_single_term_shortcut(synth):
    reader = synth["reader"]
    before = ctx().launches
    got = sdb.ExecuteCountBatch(reader, [[t] for t in range(24)], sdb.OR)
    assert ctx().launches == before
    assert got.tolist() == [len(d) for d in synth["lists"]]
    assert sdb.ExecuteCount(reader, [7], sdb.AND) == len(synth["lists"][7])
    assert ctx().launches == before
    assert sdb.ExecuteCount(reader, [7], sdb.OR, exclude=[999]) == len(synth["lists"][7])   # absent id: still no launch
    assert ctx().launches == before
    assert sdb.ExecuteCount(reader, [7], sdb.OR, exclude=[3]) == len(np.setdiff1d(synth["lists"][7], synth["lists"][3]))
    assert ctx().launches > before


def _raw(reader, terms, off, nq, excl=None, xoff=None, filt=None, counts=True):
    arr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    out = np.zeros(max(nq, 1), np.uint64)
    return N.lib().sdbg_match_count_batch(sdb.engine._seg_array(reader.segments), len(reader.segments), sdb.OR, arr(terms), arr(off),
                                          nq, arr(excl), arr(xoff), C.byref(filt) if filt is not None else None,
                                          arr(out) if counts else None)


def test_errors(synth):
    reader = synth["reader"]
    t = np.array([0, 1], np.uint32)
    off = np.array([0, 2], np.uint32)
    assert _raw(reader, t, off, 0) == -1
    assert _raw(reader, None, off, 1) == -1
    assert _raw(reader, t, None, 1) == -1
    assert _raw(reader, t, off, 1, counts=False) == -1
    assert _raw(reader, t, np.array([0, 0], np.uint32), 1) == -7                       # no positive term
    assert _raw(reader, np.arange(17, dtype=np.uint32), np.array([0, 17], np.uint32), 1) == -7
    assert _raw(reader, t, off, 1, np.arange(2, 19, dtype=np.uint32), np.array([0, 17], np.uint32)) == -7
    assert _raw(reader, t, np.array([0, 1, 2], np.uint32), 2, np.array([3, 4], np.uint32), np.array([0, 2, 1], np.uint32)) == -1
    assert _raw(reader, t, off, 1, None, np.array([0, 1], np.uint32)) == -1
    assert _raw(reader, np.array([0, 10_000], np.uint32), off, 1) == -1
    assert _raw(reader, t, off, 1, filt=sdb.pred(77, "LT", 5)) == -5
    with pytest.raises(N.SdbgError, match="term id out of range"):
        sdb.ExecuteCount(reader, [0, 10_000], sdb.OR)
    empty = sdb.Segment(ctx(), 100)
    assert _raw(sdb.IndexReader([empty], 100, 100, [0]), t, off, 1) == -1              # no postings staged
    other = sdb.Context(0)
    seg2 = sdb.Segment(other, synth["n"])
    seg2.stage_postings(synth["oseg"].doc_bytes(), metas_of(synth["oseg"]))
    mixed = sdb.IndexReader([synth["g"], seg2], synth["n"], 1, [0])
    assert _raw(mixed, t, off, 1) == -1                                                # segments of two contexts
    seg2.close()
    other.close()


def test_adapter_count_scan(synth):
    from serenedb_b200 import build as b
    exe = b.build_adapters()
    n = 200_000
    res = subprocess.run([exe, str(n), "count"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = [json.loads(l) for l in res.stdout.strip().splitlines()]
    assert len(lines) == 8
    oseg, dc, _ = orc.synth_segment_mt(n, 0, 8, threads=4)
    lists = [oseg.decode_term(t)[0] for t in range(8)]
    col = orc.synth_column(2, 1, 1, n).astype(np.int32)
    mask = cr.pred_mask(col, None, "BETWEEN", 250000, 749999)
    for out in lines:
        kind = "AND" if out["kind"] == sdb.AND else "OR"
        want = cr.count([lists], kind, [2, 5], [3] if out["excl"] else [], masks=[mask if out["filter"] else None])
        assert out["rows"] == 1 and out["rows_after"] == 0 and out["count"] == want, out


def test_batch_4096_at_scale():
    n = 2_000_000
    nt = 64
    g = sdb.Segment(ctx(), n)
    dc, sum_dl = g.synth_corpus(0, 0, nt)
    reader = sdb.IndexReader([g], n, sum_dl, dc)
    rng = np.random.default_rng(2026)
    qs = [sorted(rng.choice(nt, int(rng.integers(1, 5)), replace=False).tolist()) for _ in range(4096)]
    for kind in (sdb.OR, sdb.AND):
        got = sdb.ExecuteCountBatch(reader, qs, kind)
        assert np.array_equal(got, level0_totals(reader, qs, kind))
