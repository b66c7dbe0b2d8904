"""Facet counts (sdbg_match_facet_counts_batch, ExecuteFacetCountsBatch) on the GPU: per-key counts and NULL counts equal
the NumPy statement of the semantics (tests/facet_reference.py) exactly, and sum(counts) + nulls equals ExecuteCountBatch
for every query. Covers OR of 1..16 terms and AND of 2..16 with exclusions, the hybrid filter (including filter column ==
key column), deleted docs, every block encoding, window edges, three segments (a query without a match in one, a key
column shorter than its segment in another), int64 bit-packed / raw nullable / borrowed and int32 keys, key_span 1 and
32768, negative key_min and key_min = INT64_MAX - span + 1, a single-key column, an all-NULL column, the single-term
shortcut case, every pruning level, the error codes, the cookbook's products_facets, the adapter and a 4096-query batch
over the 10 M-doc benchmark corpus checked against StreamScoredDocs + gather + bincount."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import count_reference as cr
import facet_reference as fr
import orc
import serenedb_b200 as sdb
from serenedb_b200 import _native as N
from gpu_util import ctx, to_gpu
from shape_corpora import NORM_WIDTHS, Corpus, natural_segments, shape_segment

pytestmark = pytest.mark.gpu

W = 1 << 16
I64_MAX = np.iinfo(np.int64).max
HERE = os.path.dirname(os.path.abspath(__file__))


def check(reader, seg_lists, columns, queries, kind, field, key_min, key_span, filt=None, exclude=None, deleted=None,
          masks=None):
    got = sdb.ExecuteFacetCountsBatch(reader, queries, kind, field, key_min, key_span, filt=filt, exclude=exclude)
    okind = "AND" if kind == sdb.AND else "OR"
    xs = exclude or [[]] * len(queries)
    counts = sdb.ExecuteCountBatch(reader, queries, kind, filt=filt, exclude=exclude)
    assert got["counts"].shape == (len(queries), key_span) and got["key_min"] == key_min
    for q, (terms, x) in enumerate(zip(queries, xs)):
        want, nulls = fr.facet_counts(seg_lists, okind, terms, columns, key_min, key_span, excl=x or [], deleted=deleted,
                                      masks=masks)
        assert np.array_equal(got["counts"][q], want), (q, terms, field)
        assert int(got["nulls"][q]) == nulls, (q, terms, field)
        assert int(got["counts"][q].sum()) + int(got["nulls"][q]) == int(counts[q]), (q, terms)
    return got


@pytest.fixture(scope="module")
def synth():
    import torch
    n = 200_000
    oseg, dl, lists = orc.synth_segment(n, list(range(24)))
    rng = np.random.default_rng(17)
    borrowed = rng.integers(-3000, 3000, n).astype(np.int64)
    cols = {1: (rng.integers(-1000, 1001, n).astype(np.int64), None),                 # narrow: bit-packed
            2: (rng.integers(-500, 500, n).astype(np.int32), None),
            3: (rng.normal(size=n), None),                                             # float64: unsupported
            4: (rng.integers(-20, 30, n).astype(np.int64), rng.random(n) < 0.7),       # nullable raw
            5: (np.full(n - 5000, 42, np.int64), None),                                # one key; last 5000 docs NULL
            6: (np.zeros(n, np.int64), np.zeros(n, bool)),                             # all NULL
            7: (I64_MAX - rng.integers(0, 100, n).astype(np.int64), None),             # at the top of int64
            8: (rng.integers(0, 32768, n).astype(np.int64), None)}                     # 32768 keys
    g = to_gpu(oseg, columns={f: (v, cr.validity_words(m) if m is not None else None) for f, (v, m) in cols.items()})
    t = torch.from_numpy(borrowed).cuda()
    g.stage_column_device(9, t.data_ptr(), np.int64, n)
    cols[9] = (borrowed, None)
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d, _ in lists])
    return dict(g=g, reader=reader, n=n, lists=[d for d, _ in lists], cols=cols, keep=t)


# (field, key_min, key_span) of each key column, the range taken wider than the values where that tests something
RANGES = {1: (-1000, 2001), 2: (-500, 1000), 4: (-25, 60), 5: (42, 1), 6: (0, 1), 7: (I64_MAX - 99, 100),
          8: (0, 32768), 9: (-3000, 6000)}


def test_or_and_every_term_count_and_type(synth):
    reader, lists = synth["reader"], [synth["lists"]]
    rng = np.random.default_rng(1)
    qs_or = [sorted(rng.choice(24, size=t, replace=False).tolist()) for t in range(1, 17)]
    qs_and = [sorted(rng.choice(6, size=min(t, 6), replace=False).tolist()) +
              sorted(rng.choice(np.arange(6, 24), size=max(0, t - 6), replace=False).tolist()) for t in range(2, 17)]
    assert synth["g"].column_packed(1, synth["n"]) is not None and synth["g"].column_packed(4, synth["n"]) is None
    for f, (lo, span) in RANGES.items():
        col = [synth["cols"][f]]
        check(reader, lists, col, qs_or, sdb.OR, f, lo, span)
        check(reader, lists, col, qs_and, sdb.AND, f, lo, span)


def test_default_range_and_dict(synth):
    reader, lists = synth["reader"], [synth["lists"]]
    got = sdb.ExecuteFacetCountsBatch(reader, [[0, 3]], sdb.OR, 4)
    assert got["key_min"] == -20 and got["counts"].shape == (1, 50)
    assert sdb.ExecuteFacetCounts(reader, [0, 3], sdb.OR, 4) == fr.facet_dict(lists, "OR", [0, 3], [synth["cols"][4]])
    assert sdb.ExecuteFacetCounts(reader, [1], sdb.OR, 6) == {None: len(synth["lists"][1])}       # all NULL
    assert sdb.ExecuteFacetCounts(reader, [2], sdb.AND, 5) == fr.facet_dict(lists, "AND", [2], [synth["cols"][5]])
    with pytest.raises(ValueError):
        sdb.ExecuteFacetCountsBatch(reader, [[0]], sdb.OR, 3)            # float64 key
    with pytest.raises(ValueError):
        sdb.ExecuteFacetCountsBatch(reader, [[0]], sdb.OR, 77)           # not staged


def test_single_term_without_filter(synth):
    """The count answers these from docs_count without a launch; the facet pass must scan them."""
    reader, lists = synth["reader"], [synth["lists"]]
    qs = [[t] for t in range(24)]
    for f in (1, 2, 4, 5):
        lo, span = RANGES[f]
        check(reader, lists, [synth["cols"][f]], qs, sdb.OR, f, lo, span)
        check(reader, lists, [synth["cols"][f]], qs, sdb.AND, f, lo, span)


def test_exclusions(synth):
    reader, lists = synth["reader"], [synth["lists"]]
    rng = np.random.default_rng(5)
    qs, xs = [], []
    for ne in range(1, 17):
        q = sorted(rng.choice(8, size=2, replace=False).tolist())
        qs.append(q)
        xs.append(rng.choice([t for t in range(24) if t not in q], size=ne, replace=False).tolist())
    for kind in (sdb.OR, sdb.AND):
        check(reader, lists, [synth["cols"][2]], qs, kind, 2, -500, 1000, exclude=xs)
    check(reader, lists, [synth["cols"][2]], [[0, 3], [1]], sdb.OR, 2, -500, 1000, exclude=[[999], [5, 10_000]])
    got = check(reader, lists, [synth["cols"][2]], [[0, 3], [2, 5, 7]], sdb.AND, 2, -500, 1000, exclude=[[3], [7]])
    assert got["counts"].sum() == 0 and got["nulls"].sum() == 0


def test_filter_and_deleted_docs(synth):
    reader, lists, g, n = synth["reader"], [synth["lists"]], synth["g"], synth["n"]
    rng = np.random.default_rng(8)
    deleted = np.unique(rng.integers(1, n + 1, 9000)).astype(np.uint32)
    qs = [[0, 3], [1], [2, 5, 7, 9], [0, 1]]
    preds = [(2, "BETWEEN", -100, 99), (1, "LT", 0, 0), (3, "GE", 0.25, 0), (4, "GT", 5, 0), (4, "IS_NULL", 0, 0),
             (4, "IS_NOT_NULL", 0, 0)]
    try:
        for with_deleted in (False, True):
            g.stage_docs_mask(deleted if with_deleted else None)
            dele = [deleted] if with_deleted else None
            for kind in (sdb.OR, sdb.AND):
                check(reader, lists, [synth["cols"][1]], qs, kind, 1, -1000, 2001, deleted=dele)
                for f, op, lo, hi in preds:
                    m = cr.pred_mask(synth["cols"][f][0], synth["cols"][f][1], op, lo, hi)
                    for kf in sorted({f, 4} - {3}):                                    # filter column == key column too
                        klo, kspan = RANGES[kf]
                        check(reader, lists, [synth["cols"][kf]], qs, kind, kf, klo, kspan, filt=sdb.pred(f, op, lo, hi),
                              deleted=dele, masks=[m])
    finally:
        g.stage_docs_mask(None)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_pruning_levels_identical(synth, level):
    reader = synth["reader"]
    qs = [[0, 3], [1, 4, 9], [2], [5, 6, 7, 8], [10, 11]]
    try:
        ctx().set_wand(0)
        base = [sdb.ExecuteFacetCountsBatch(reader, qs, kind, 1, -1000, 2001) for kind in (sdb.OR, sdb.AND)]
        ctx().set_wand(level)
        got = [sdb.ExecuteFacetCountsBatch(reader, qs, kind, 1, -1000, 2001) for kind in (sdb.OR, sdb.AND)]
    finally:
        ctx().set_wand(0)
    for b, r in zip(base, got):
        assert np.array_equal(b["counts"], r["counts"]) and np.array_equal(b["nulls"], r["nulls"])
    check(reader, [synth["lists"]], [synth["cols"][1]], qs, sdb.OR, 1, -1000, 2001)


@pytest.fixture(scope="module", params=NORM_WIDTHS, ids=lambda w: f"norms{w or 0}")
def shapes(request):
    oseg, norms, lists = shape_segment(request.param)
    n = oseg.n_docs
    rows = min(n, 3_000_000)   # the 2^30-doc shape: docs past the column's rows have a NULL key
    vals = (np.arange(rows, dtype=np.int64) * 7919) % 1009 - 500
    g = to_gpu(oseg, columns={1: (vals, None)})
    ttf = int(norms.astype(np.uint64).sum()) if norms is not None else n
    reader = sdb.IndexReader([g], n, ttf, [len(d) for _, d, _ in lists])
    return dict(reader=reader, lists=[d for _, d, _ in lists], names=[nm for nm, _, _ in lists], cols=[(vals, None)])


def test_every_encoding(shapes):
    lists, names = shapes["lists"], shapes["names"]
    shape_ids = [t for t, nm in enumerate(names) if not nm.endswith("+lead")]
    pairs = [[t, t + 1] for t in shape_ids]
    for kind in (sdb.OR, sdb.AND):
        check(shapes["reader"], [lists], shapes["cols"], pairs, kind, 1, -500, 1009)
    check(shapes["reader"], [lists], shapes["cols"], [[t + 1] for t in shape_ids], sdb.OR, 1, -500, 1009,
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
    vals[np.array(edge) - 1] = 1 + np.arange(len(edge))   # each edge doc its own key
    g = to_gpu(oseg, columns={1: (vals, None)})
    reader = sdb.IndexReader([g], n, n, [len(d) for d in lists])
    got = check(reader, [lists], [(vals, None)], [[0], [0, 1], [1]], sdb.OR, 1, 0, 11)
    assert got["counts"][0].tolist() == [0] + [1] * 10


def test_three_segments():
    segs = natural_segments()
    norms1, lists1 = segs[1]
    d6 = lists1[6][0]
    keep = ~np.isin(lists1[9][0], d6)                        # terms 6 and 9 never meet in segment 1
    lists1[9] = (lists1[9][0][keep], lists1[9][1][keep])
    corpus = Corpus(segs)
    rng = np.random.default_rng(12)
    cols, gsegs = [], []
    for i, o in enumerate(corpus.osegs):
        rows = o.n_docs - 777 if i == 2 else o.n_docs        # segment 2: the last 777 docs have a NULL key
        v = rng.integers(-7, 13, rows).astype(np.int32)
        m = rng.random(rows) < 0.9
        cols.append((v, m))
        gsegs.append(to_gpu(o, columns={1: (v, cr.validity_words(m))}))
    reader = sdb.IndexReader(gsegs, corpus.docs_with_field, corpus.total_term_freq, corpus.docs_with_term)
    seg_lists = [[np.asarray(d, np.uint32) for d, _ in l] for l in corpus.lists]
    assert len(cr.match_docs(seg_lists[1], "AND", [6, 9])) == 0
    qs = [sorted(rng.choice(corpus.n_terms, size=int(rng.integers(1, 5)), replace=False).tolist()) for _ in range(20)]
    qs += [[6, 9], [0, 9]]
    for kind in (sdb.OR, sdb.AND):
        check(reader, seg_lists, cols, qs, kind, 1, -7, 20)
    check(reader, seg_lists, cols, qs, sdb.OR, 1, -7, 20, exclude=[[3]] * len(qs))


def _raw(reader, terms, off, nq, field=1, key_min=-1000, key_span=2001, counts=True, nulls=True, excl=None, xoff=None,
         filt=None):
    arr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    c = np.zeros(max(nq, 1) * max(key_span, 1), np.uint64)
    nn = np.zeros(max(nq, 1), np.uint64)
    return N.lib().sdbg_match_facet_counts_batch(sdb.engine._seg_array(reader.segments), len(reader.segments), sdb.OR,
                                                 arr(terms), arr(off), nq, arr(excl), arr(xoff),
                                                 C.byref(filt) if filt is not None else None, field, key_min, key_span,
                                                 arr(c) if counts else None, arr(nn) if nulls else None)


def test_errors(synth):
    reader = synth["reader"]
    t = np.array([0, 1], np.uint32)
    off = np.array([0, 2], np.uint32)
    assert _raw(reader, t, off, 1) == 0
    assert _raw(reader, t, off, 0) == -1
    assert _raw(reader, None, off, 1) == -1
    assert _raw(reader, t, off, 1, counts=False) == -1
    assert _raw(reader, t, off, 1, nulls=False) == -1
    assert _raw(reader, t, off, 1, key_span=0) == -1
    assert _raw(reader, t, off, 1, field=7, key_min=I64_MAX - 98, key_span=100) == -1     # overflows int64
    assert _raw(reader, t, off, 1, key_span=32769) == -7
    assert _raw(reader, t, off, 1, field=77) == -5
    assert _raw(reader, t, off, 1, field=3) == -7                                         # float64
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
    g_b = to_gpu(o2, columns={1: (np.arange(n, dtype=np.int32), None)})
    mixed = sdb.IndexReader([g_a, g_b], 2 * n, 2 * n, [2 * n])
    one = np.array([0], np.uint32)
    before = ctx().launches
    assert _raw(mixed, one, np.array([0, 1], np.uint32), 1, key_min=0, key_span=n) == -1   # type differs across segments
    assert ctx().launches == before
    # after the scan: keys outside the range
    assert _raw(reader, t, off, 1, key_min=-999, key_span=2000) == -1
    assert _raw(reader, t, off, 1, key_min=-1000, key_span=2000) == -1
    with pytest.raises(N.SdbgError, match="outside"):
        sdb.ExecuteFacetCountsBatch(reader, [[0, 1]], sdb.OR, 1, 0, 1000)


def test_errors_queue_nothing(synth):
    reader = synth["reader"]
    t = np.array([0, 1], np.uint32)
    off = np.array([0, 2], np.uint32)
    before = ctx().launches
    for kw in (dict(counts=False), dict(key_span=0), dict(field=7, key_min=I64_MAX - 98, key_span=100),
               dict(key_span=32769), dict(field=77), dict(field=3), dict(filt=sdb.pred(77, "LT", 5))):
        assert _raw(reader, t, off, 1, **kw) != 0, kw
    assert _raw(reader, np.array([0, 10_000], np.uint32), off, 1) != 0
    assert ctx().launches == before


def test_products_facets():
    """The reference's faceted-search cookbook: 8 products, a term every product holds, facet counts per category, brand
    and price band."""
    with open(os.path.join(HERE, "golden", "groupby_goldens.json")) as f:
        g = json.load(f)["products_facets"]
    o = orc.Segment(8)
    o.add_term(np.arange(1, 9, dtype=np.uint32), np.ones(8, np.uint32))
    fields = {"category": 1, "brand": 2, "band": 3}
    gs = to_gpu(o, columns={fields[f]: (np.asarray(g["rows"][f], np.int64), None) for f in fields})
    reader = sdb.IndexReader([gs], 8, 8, [8])
    for f, fid in fields.items():
        got = sdb.ExecuteFacetCounts(reader, [0], sdb.OR, fid)
        names = g[f + "_names"]
        assert {names[k]: v for k, v in got.items()} == g["expect_" + f]


def test_adapter_facet_scan():
    """GpuFacetScan through adapter_selftest: `t2 | t5`, `t2 & t5` and `(t2 | t5) & !t3` GROUP BY the 2001-key column,
    without and with the filter: the groups equal the reference, in key order, then cardinality 0; a column whose range
    spans more than 32768 values throws SDBG_EUNSUPPORTED."""
    from serenedb_b200 import build as b
    exe = b.build_adapters()
    n = 200_000
    res = subprocess.run([exe, str(n), "facet"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = [json.loads(l) for l in res.stdout.strip().splitlines()]
    assert len(lines) == 9 and lines[-1] == {"wide_error": -7}
    oseg, _, _ = orc.synth_segment_mt(n, 0, 8, threads=4)
    lists = [oseg.decode_term(t)[0] for t in range(8)]
    key = orc.synth_column(15, 3, 1, n)
    fcol = orc.synth_column(2, 1, 1, n)   # column 9: kind 6 is kind 1 stored as int32
    mask = cr.pred_mask(fcol, None, "BETWEEN", 250000, 749999)
    for out in lines[:-1]:
        kind = "AND" if out["kind"] == sdb.AND else "OR"
        want = fr.facet_dict([lists], kind, [2, 5], [(key, None)], excl=[3] if out["excl"] else [],
                             masks=[mask if out["filter"] else None])
        assert None not in want
        assert out["keys"] == sorted(want) and out["counts"] == [want[k] for k in sorted(want)]
        assert out["valid"] == [1] * len(want)
        assert out["chunks"] == 1 and out["max_chunk"] <= 2048 and out["rows_after"] == 0


def test_batch_4096_at_bench_scale():
    """bench.py's corpus: 10 M docs, its terms and 4096 two-term ORs (bench.make_queries), faceted on the bit-packed
    2001-key column v = h % 2001 - 1000; the invariant for every query, and 64 sampled queries against
    StreamScoredDocs + gather + bincount."""
    import bench
    n = 10_000_000
    g = sdb.Segment(ctx(), n)
    dc, sum_dl = g.synth_corpus(0, 0, bench.N_TERMS)
    g.synth_column(1, 13, 3, 1, n)
    assert g.column_packed(1, n) is not None
    reader = sdb.IndexReader([g], n, sum_dl, dc)
    qs = bench.make_queries(4096)
    counts = sdb.ExecuteCountBatch(reader, qs, sdb.OR)
    got = sdb.ExecuteFacetCountsBatch(reader, qs, sdb.OR, 1, -1000, 2001)
    assert np.array_equal(got["counts"].sum(axis=1), counts) and not got["nulls"].any()
    for q in range(0, 4096, 64):
        docs, _ = sdb.StreamScoredDocs(reader, 0, qs[q], sdb.OR, sdb.BM25())
        vals, valid = g.gather(1, docs, np.int64)
        assert valid.all()
        assert np.array_equal(got["counts"][q], np.bincount(vals + 1000, minlength=2001).astype(np.uint64)), q
