"""Sorted scan (sdbg_match_topk_by_column_batch, ExecuteTopKByColumnBatch) on the GPU: docs, segments, values, NULL
flags and order equal the NumPy statement of the semantics (tests/sort_reference.py) exactly, and n_out equals
min(k, count). Covers OR of 1..16 terms and AND of 2..16 with exclusions, the hybrid filter (including filter column ==
sort column), deleted docs, every block encoding, window edges, three segments, int64 raw / bit-packed, int32, float64
with special values and nullable sort columns, both directions and NULL placements, k = 1 / k > matches / k = 4096,
an all-ties column, every pruning level, zonemap skipping on a clustered column, the error codes and a 4096-query batch
over the 10 M-doc benchmark corpus checked against StreamScoredDocs + gather."""
import ctypes as C
import json
import subprocess

import numpy as np
import pytest

import count_reference as cr
import orc
import sort_reference as sr
import serenedb_b200 as sdb
from serenedb_b200 import _native as N
from gpu_util import ctx, to_gpu
from shape_corpora import NORM_WIDTHS, Corpus, natural_segments, shape_segment

pytestmark = pytest.mark.gpu

W = 1 << 16
ORDERS = [(d, nf) for d in (False, True) for nf in (False, True)]


def check(reader, seg_lists, columns, queries, kind, field, k, desc=False, nf=False, filt=None, exclude=None,
          deleted=None, masks=None):
    got = sdb.ExecuteTopKByColumnBatch(reader, queries, kind, field, k, desc, nf, filt=filt, exclude=exclude)
    okind = "AND" if kind == sdb.AND else "OR"
    xs = exclude or [[]] * len(queries)
    counts = sdb.ExecuteCountBatch(reader, queries, kind, filt=filt, exclude=exclude)
    for q, (terms, x) in enumerate(zip(queries, xs)):
        want = sr.sorted_hits(seg_lists, okind, terms, columns, desc, nf, k=k, excl=x or [], deleted=deleted, masks=masks)
        n = int(got["n_out"][q])
        assert n == min(k, int(counts[q])) == len(want["docs"]), (q, terms, n, counts[q])
        assert np.array_equal(got["docs"][q], want["docs"]), (q, terms, desc, nf)
        assert np.array_equal(got["segs"][q], want["segs"])
        assert np.array_equal(got["nulls"][q], want["nulls"])
        assert got["values"][q].dtype == want["values"].dtype
        assert np.array_equal(got["values"][q].view(np.uint8), want["values"].view(np.uint8))
    return got


@pytest.fixture(scope="module")
def synth():
    n = 200_000
    oseg, dl, lists = orc.synth_segment(n, list(range(24)))
    rng = np.random.default_rng(7)
    fvals = rng.normal(size=n)
    fvals[rng.integers(0, n, 300)] = np.nan
    fvals[rng.integers(0, n, 50)] = -np.nan
    fvals[rng.integers(0, n, 50)] = np.inf
    fvals[rng.integers(0, n, 50)] = -np.inf
    fvals[rng.integers(0, n, 100)] = 0.0
    fvals[rng.integers(0, n, 100)] = -0.0
    i64 = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, endpoint=True)
    i64[rng.integers(0, n, 40)] = np.iinfo(np.int64).min
    i64[rng.integers(0, n, 40)] = np.iinfo(np.int64).max
    cols = {1: (i64, None),                                                         # int64, full range: held raw
            2: (rng.integers(-1000, 1000, n).astype(np.int32), None),
            3: (fvals, None),
            4: (rng.integers(0, 50, n).astype(np.int64), rng.random(n) < 0.7),     # nullable
            5: (np.full(n - 5000, 42, np.int64), None),                             # constant; last 5000 docs NULL
            6: (rng.integers(0, 300, n).astype(np.int64), None)}                    # narrow: bit-packed
    g = to_gpu(oseg, columns={f: (v, cr.validity_words(m) if m is not None else None) for f, (v, m) in cols.items()})
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d, _ in lists])
    return dict(g=g, reader=reader, n=n, lists=[d for d, _ in lists], cols=cols)


def cols_of(synth, f):
    return [synth["cols"][f]]


def test_or_and_every_term_count_and_type(synth):
    reader, lists = synth["reader"], [synth["lists"]]
    rng = np.random.default_rng(1)
    qs_or = [sorted(rng.choice(24, size=t, replace=False).tolist()) for t in range(1, 17)]
    qs_and = [sorted(rng.choice(6, size=min(t, 6), replace=False).tolist()) +
              sorted(rng.choice(np.arange(6, 24), size=max(0, t - 6), replace=False).tolist()) for t in range(2, 17)]
    assert synth["g"].column_packed(6, synth["n"]) is not None and synth["g"].column_packed(1, synth["n"]) is None
    for f in (1, 2, 3, 4, 5, 6):
        for desc, nf in ORDERS:
            check(reader, lists, cols_of(synth, f), qs_or, sdb.OR, f, 100, desc, nf)
        check(reader, lists, cols_of(synth, f), qs_and, sdb.AND, f, 100, f % 2 == 0, f % 3 == 0)


def test_k_edges(synth):
    reader, lists = synth["reader"], [synth["lists"]]
    qs = [[0], [3, 7], [1, 2, 3, 4]]
    for k in (1, 4096):
        for f in (1, 3, 4):
            check(reader, lists, cols_of(synth, f), qs, sdb.OR, f, k, True, False)
    m = cr.pred_mask(synth["cols"][2][0], None, "BETWEEN", 0, 9)
    got = check(reader, lists, cols_of(synth, 4), [[0, 1]], sdb.OR, 4, 4096, False, True, filt=sdb.pred(2, "BETWEEN", 0, 9),
                masks=[m])                                                               # k > matches
    assert 0 < got["n_out"][0] < 4096
    check(reader, lists, cols_of(synth, 5), qs, sdb.OR, 5, 700, True, True)                # all ties: doc order
    check(reader, lists, cols_of(synth, 5), qs, sdb.OR, 5, 4096, False, False)


def test_exclusions(synth):
    reader, lists = synth["reader"], [synth["lists"]]
    rng = np.random.default_rng(5)
    qs, xs = [], []
    for ne in range(1, 17):
        q = sorted(rng.choice(8, size=2, replace=False).tolist())
        qs.append(q)
        xs.append(rng.choice([t for t in range(24) if t not in q], size=ne, replace=False).tolist())
    for kind in (sdb.OR, sdb.AND):
        check(reader, lists, cols_of(synth, 2), qs, kind, 2, 50, True, False, exclude=xs)
    check(reader, lists, cols_of(synth, 2), [[0, 3], [1]], sdb.OR, 2, 50, exclude=[[999], [5, 10_000]])   # absent ids
    got = check(reader, lists, cols_of(synth, 2), [[0, 3], [2, 5, 7]], sdb.AND, 2, 50, exclude=[[3], [7]])  # self-exclusion
    assert got["n_out"].tolist() == [0, 0]


def test_filter_and_deleted_docs(synth):
    reader, lists, g, n = synth["reader"], [synth["lists"]], synth["g"], synth["n"]
    rng = np.random.default_rng(8)
    deleted = np.unique(rng.integers(1, n + 1, 9000)).astype(np.uint32)
    qs = [[0, 3], [1], [2, 5, 7, 9], [0, 1]]
    preds = [(2, "BETWEEN", -500, 499), (1, "LT", 0, 0), (3, "GE", 0.25, 0), (4, "GT", 20, 0), (4, "IS_NULL", 0, 0),
             (4, "IS_NOT_NULL", 0, 0)]
    for with_deleted in (False, True):
        g.stage_docs_mask(deleted if with_deleted else None)
        dele = [deleted] if with_deleted else None
        for kind in (sdb.OR, sdb.AND):
            check(reader, lists, cols_of(synth, 6), qs, kind, 6, 64, True, False, deleted=dele)
            for f, op, lo, hi in preds:
                m = cr.pred_mask(synth["cols"][f][0], synth["cols"][f][1], op, lo, hi)
                for sf in sorted({f, 3}):                                             # filter column == sort column too
                    check(reader, lists, cols_of(synth, sf), qs, kind, sf, 64, sf == 3, True,
                          filt=sdb.pred(f, op, lo, hi), deleted=dele, masks=[m])
    g.stage_docs_mask(None)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_pruning_levels_identical(synth, level):
    reader, lists = synth["reader"], [synth["lists"]]
    qs = [[0, 3], [1, 4, 9], [2], [5, 6, 7, 8], [10, 11]]
    try:
        ctx().set_wand(level)
        for f in (1, 3, 6):
            for desc, nf in ORDERS:
                check(reader, lists, cols_of(synth, f), qs, sdb.OR, f, 300, desc, nf)
            check(reader, lists, cols_of(synth, f), qs[:2], sdb.AND, f, 300, True, False)
    finally:
        ctx().set_wand(0)


@pytest.fixture(scope="module", params=NORM_WIDTHS, ids=lambda w: f"norms{w or 0}")
def shapes(request):
    oseg, norms, lists = shape_segment(request.param)
    n = oseg.n_docs
    rows = min(n, 3_000_000)   # the 2^30-doc shape: docs past the column's rows sort as NULL
    vals = (np.arange(rows, dtype=np.int64) * 7919) % 100_003
    g = to_gpu(oseg, columns={1: (vals, None)})
    ttf = int(norms.astype(np.uint64).sum()) if norms is not None else n
    reader = sdb.IndexReader([g], n, ttf, [len(d) for _, d, _ in lists])
    return dict(reader=reader, lists=[d for _, d, _ in lists], names=[nm for nm, _, _ in lists], cols=[(vals, None)])


def test_every_encoding(shapes):
    lists, names = shapes["lists"], shapes["names"]
    shape_ids = [t for t, nm in enumerate(names) if not nm.endswith("+lead")]
    pairs = [[t, t + 1] for t in shape_ids]
    for kind in (sdb.OR, sdb.AND):
        check(shapes["reader"], [lists], shapes["cols"], pairs, kind, 1, 200, kind == sdb.OR, False)
    check(shapes["reader"], [lists], shapes["cols"], [[t + 1] for t in shape_ids], sdb.OR, 1, 200, False, True,
          exclude=[[t] for t in shape_ids])


@pytest.mark.parametrize("n", [3 * W + 17, 4 * W + 31])
def test_window_edges(n):
    edge = [1, W - 1, W, W + 1, 2 * W - 1, 2 * W, 2 * W + 1, 3 * W, n - 1, n]
    rng = np.random.default_rng(n)
    oseg = orc.Segment(n)
    lists = [np.unique(np.array(edge, np.uint32)),
             np.unique(np.concatenate([edge[::2], rng.integers(1, n + 1, 3000)])).astype(np.uint32)]
    for d in lists:
        oseg.add_term(d, np.ones(len(d), np.uint32))
    vals = np.zeros(n, np.int64)
    vals[np.array(edge) - 1] = 1000 + np.arange(len(edge))   # the edge docs hold the largest values
    g = to_gpu(oseg, columns={1: (vals, None)})
    reader = sdb.IndexReader([g], n, n, [len(d) for d in lists])
    try:
        for level in (0, 2):
            ctx().set_wand(level)
            for desc, nf in ORDERS:
                check(reader, [lists], [(vals, None)], [[0], [0, 1], [1]], sdb.OR, 1, 5, desc, nf)
    finally:
        ctx().set_wand(0)


def test_three_segments():
    corpus = Corpus(natural_segments())
    rng = np.random.default_rng(12)
    cols = []
    segs = []
    for o in corpus.osegs:
        v = rng.integers(0, 20, o.n_docs).astype(np.int32)   # many ties across segments
        m = rng.random(o.n_docs) < 0.9
        cols.append((v, m))
        segs.append(to_gpu(o, columns={1: (v, cr.validity_words(m))}))
    reader = sdb.IndexReader(segs, corpus.docs_with_field, corpus.total_term_freq, corpus.docs_with_term)
    seg_lists = [[np.asarray(d, np.uint32) for d, _ in l] for l in corpus.lists]
    qs = [sorted(rng.choice(corpus.n_terms, size=int(rng.integers(1, 5)), replace=False).tolist()) for _ in range(20)]
    for kind in (sdb.OR, sdb.AND):
        for desc, nf in ORDERS:
            check(reader, seg_lists, cols, qs, kind, 1, 40, desc, nf)


@pytest.mark.parametrize("level", [1, 2])
def test_three_segments_clustered_with_zonemaps(level):
    """Three NOT NULL segments of one clustered column (ts continues across segments, so the last segment holds the
    newest rows): the seed window is chosen across segments, the threshold is shared by the segments' items, and
    windows are skipped in the segments that cannot compete. Exclusions, a filter and deleted docs included."""
    sizes = (300_000, 450_000, 250_000)
    gsegs, seg_lists, cols, dels, masks = [], [], [], [], []
    row0 = 0
    for i, n in enumerate(sizes):
        oseg, _, lists = orc.synth_segment(n, list(range(6)), doc0=row0)
        ts = ((np.arange(n) + row0) // 100).astype(np.int64)
        row0 += n
        rng = np.random.default_rng(40 + i)
        f2 = rng.integers(0, 100, n).astype(np.int32)
        dele = np.unique(rng.integers(1, n + 1, 2000)).astype(np.uint32)
        g = to_gpu(oseg, columns={1: (ts, None), 2: (f2, None)})
        g.stage_docs_mask(dele)
        gsegs.append(g); seg_lists.append([d for d, _ in lists]); cols.append((ts, None)); dels.append(dele)
        masks.append(cr.pred_mask(f2, None, "LT", 70))
    reader = sdb.IndexReader(gsegs, sum(sizes), sum(sizes), [1] * 6)
    qs = [[0, 1], [2], [1, 3, 4], [0, 5]]
    xs = [[2], [], [0], [4]]
    try:
        for desc in (True, False):
            ctx().set_wand(level)
            check(reader, seg_lists, cols, qs, sdb.OR, 1, 200, desc, False, exclude=xs, deleted=dels)
            judged, skipped = _scan_stats()
            assert judged > 0 and skipped > 0, (desc, judged, skipped)
            check(reader, seg_lists, cols, qs, sdb.AND, 1, 200, desc, True, deleted=dels)
            check(reader, seg_lists, cols, qs, sdb.OR, 1, 200, desc, False, filt=sdb.pred(2, "LT", 70), exclude=xs,
                  deleted=dels, masks=masks)
    finally:
        ctx().set_wand(0)


def _scan_stats():
    t, s = C.c_uint64(), C.c_uint64()
    N.check(N.lib().sdbg_scan_stats(ctx()._h, C.byref(t), C.byref(s)))
    return t.value, s.value


@pytest.mark.parametrize("kind_f", ["int", "float"])
def test_zonemap_skips_on_clustered_column(kind_f):
    """ts = row / 100 (DESC: newest first; ASC: oldest first): with pruning the seed window sets the threshold and the
    other windows are skipped; hits equal level 0. The float column holds a NaN with the sign bit in a middle window,
    which sorts above everything: under DESC that window bounds the best key, so it is the seed, and the windows before
    it are skipped. A bound that read the NaN as the zone's smallest value would seed the last window and skip the NaN."""
    n = 2_000_000
    oseg, dl, lists = orc.synth_segment(n, list(range(4)))
    lists = [d for d, _ in lists]
    ts = (np.arange(n) // 100).astype(np.int64)
    fts = ts.astype(np.float64)
    nan_doc = int(lists[0][len(lists[0]) // 2])
    fts[nan_doc - 1] = np.array([0xFFF8000000000000], np.uint64).view(np.float64)[0]
    vals = ts if kind_f == "int" else fts
    g = to_gpu(oseg, columns={1: (vals, None)})
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d in lists])
    qs = [[0, 1], [2], [1, 3]]
    try:
        for desc in (True, False):
            ctx().set_wand(0)
            base = check(reader, [lists], [(vals, None)], qs, sdb.OR, 1, 100, desc, False)
            assert _scan_stats() == (0, 0)
            ctx().set_wand(2)
            got = check(reader, [lists], [(vals, None)], qs, sdb.OR, 1, 100, desc, False)
            judged, skipped = _scan_stats()
            assert judged > 0 and skipped > 0, (desc, judged, skipped)
            for key in ("docs", "segs", "nulls"):
                assert all(np.array_equal(a, b) for a, b in zip(got[key], base[key]))
            if kind_f == "float" and desc:
                assert got["docs"][0][0] == nan_doc and np.isnan(got["values"][0][0])
    finally:
        ctx().set_wand(0)


def test_adapter_sorted_scan():
    """GpuSortedScan through adapter_selftest: `t2 | t5` [minus t3] ORDER BY the int32 column, LIMIT 4096, every
    direction and NULL placement, without and with the filter: the rows equal the reference, in chunks of at most
    STANDARD_VECTOR_SIZE, then cardinality 0."""
    from serenedb_b200 import build as b
    exe = b.build_adapters()
    n = 200_000
    res = subprocess.run([exe, str(n), "sorted"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = [json.loads(l) for l in res.stdout.strip().splitlines()]
    assert len(lines) == 16
    oseg, _, _ = orc.synth_segment_mt(n, 0, 8, threads=4)
    lists = [oseg.decode_term(t)[0] for t in range(8)]
    col = orc.synth_column(2, 1, 1, n).astype(np.int32)
    mask = cr.pred_mask(col, None, "BETWEEN", 250000, 749999)
    for out in lines:
        want = sr.sorted_hits([lists], "OR", [2, 5], [(col, None)], bool(out["desc"]), bool(out["nulls_first"]), k=4096,
                              excl=[3] if out["excl"] else [], masks=[mask if out["filter"] else None])
        assert out["docs"] == want["docs"].tolist(), {k: out[k] for k in ("filter", "excl", "desc", "nulls_first")}
        assert out["segs"] == want["segs"].tolist()
        assert out["values"] == want["values"].astype(np.int64).tolist()
        assert out["valid"] == (~want["nulls"]).astype(int).tolist()
        assert out["max_chunk"] <= 2048 and out["chunks"] == -(-len(want["docs"]) // 2048) and out["rows_after"] == 0


def _raw(reader, terms, off, nq, field=1, k=10, out=True, n_out=True, excl=None, xoff=None, filt=None):
    arr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    hits = np.zeros(max(nq, 1) * max(k, 1), sdb.engine.SORT_HIT_DTYPE)
    no = np.zeros(max(nq, 1), np.uint32)
    return N.lib().sdbg_match_topk_by_column_batch(sdb.engine._seg_array(reader.segments), len(reader.segments), sdb.OR,
                                                   arr(terms), arr(off), nq, arr(excl), arr(xoff),
                                                   C.byref(filt) if filt is not None else None, field, 0, 0, k,
                                                   arr(hits) if out else None, arr(no) if n_out else None)


def test_errors(synth):
    reader = synth["reader"]
    t = np.array([0, 1], np.uint32)
    off = np.array([0, 2], np.uint32)
    assert _raw(reader, t, off, 1) == 0
    assert _raw(reader, t, off, 0) == -1
    assert _raw(reader, None, off, 1) == -1
    assert _raw(reader, t, off, 1, k=0) == -1
    assert _raw(reader, t, off, 1, out=False) == -1
    assert _raw(reader, t, off, 1, n_out=False) == -1
    assert _raw(reader, t, off, 1, k=4097) == -7
    assert _raw(reader, t, off, 1, field=77) == -5
    assert _raw(reader, t, np.array([0, 0], np.uint32), 1) == -7
    assert _raw(reader, np.arange(17, dtype=np.uint32), np.array([0, 17], np.uint32), 1) == -7
    assert _raw(reader, t, off, 1, excl=np.arange(2, 19, dtype=np.uint32), xoff=np.array([0, 17], np.uint32)) == -7
    assert _raw(reader, t, off, 1, xoff=np.array([0, 1], np.uint32)) == -1
    assert _raw(reader, np.array([0, 10_000], np.uint32), off, 1) == -1
    assert _raw(reader, t, off, 1, filt=sdb.pred(77, "LT", 5)) == -5
    n = 1000
    o2 = orc.Segment(n)
    o2.add_term(np.arange(1, n + 1, dtype=np.uint32), np.ones(n, np.uint32))
    g_a = to_gpu(o2, columns={1: (np.arange(n, dtype=np.int64), None)})
    g_b = to_gpu(o2, columns={1: (np.arange(n, dtype=np.float64), None)})
    mixed = sdb.IndexReader([g_a, g_b], 2 * n, 2 * n, [2 * n])
    one = np.array([0], np.uint32)
    assert _raw(mixed, one, np.array([0, 1], np.uint32), 1) == -1                      # type differs across segments
    with pytest.raises(N.SdbgError, match="sort column"):
        sdb.ExecuteTopKByColumn(mixed, [0], sdb.OR, 1, 5)


def test_batch_4096_at_bench_scale():
    """bench.py's corpus: 10 M docs, 64 terms, 4096 two-term ORs, top-1000 by a uniform column; 64 sampled queries
    checked against StreamScoredDocs + gather + a host sort."""
    n, nt = 10_000_000, 64
    g = sdb.Segment(ctx(), n)
    dc, sum_dl = g.synth_corpus(0, 0, nt)
    g.synth_column(1, 11, 1, 1, n)
    reader = sdb.IndexReader([g], n, sum_dl, dc)
    rng = np.random.default_rng(2026)
    qs = [sorted(rng.choice(nt, 2, replace=False).tolist()) for _ in range(4096)]
    k = 1000
    counts = sdb.ExecuteCountBatch(reader, qs, sdb.OR)
    for level in (0, 2):
        ctx().set_wand(level)
        got = sdb.ExecuteTopKByColumnBatch(reader, qs, sdb.OR, 1, k)
        assert np.array_equal(got["n_out"], np.minimum(counts, k))
        for q in range(0, 4096, 64):
            docs, _ = sdb.StreamScoredDocs(reader, 0, qs[q], sdb.OR, sdb.BM25())
            vals, valid = g.gather(1, docs, np.int64)
            assert valid.all()
            o = np.lexsort((docs, vals))[:k]
            assert np.array_equal(got["docs"][q], docs[o]), q
            assert np.array_equal(got["values"][q], vals[o]), q
    ctx().set_wand(0)
