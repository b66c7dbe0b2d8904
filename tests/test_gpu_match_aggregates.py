"""Aggregates over a full-text query's matches (sdbg_match_aggregate_batch(_groups_min), ExecuteMatchAggregates*) on the
GPU against the Python statement of the semantics (tests/agg_reference.py): counts, integer sums, MIN and MAX exactly,
float64 sums within count_value * 2^-52 * sum(|v|) of the exact sum, with IEEE NaN / infinity rules. count also equals the
facet entries' counts (grouped) or the count entries' (ungrouped).

Covers OR and AND of 1..16 terms; int64 raw, bit-packed and nullable, int32 and float64 value columns (NaN, +-inf, -0.0),
the value column equal to the key column; the ungrouped form; exclusions, the filter and deleted docs; pruning levels
0 / 1 / 2; every block encoding, window edges and three segments; doc ids up to 2^32 - 2; sums of INT64_MAX / INT64_MIN
over many work items and segments; OR-group and min-match queries including a mixed-shape batch; every error code with
nothing queued; a 4096-query batch at benchmark scale; and the adapter (GpuMatchAggScan)."""
import ctypes as C
import json
import math
import subprocess

import numpy as np
import pytest

import agg_reference as ar
import count_reference as cr
import high_doc_reference as hd
import orc
import serenedb_b200 as sdb
from gpu_util import ctx, to_gpu
from serenedb_b200 import _native as N
from shape_corpora import NORM_WIDTHS, Corpus, natural_segments, shape_segment

pytestmark = pytest.mark.gpu

W = 1 << 16
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
FIELDS = ("count", "count_value", "sum", "min", "max")


def assert_cell(got, idx, want, is_float, what):
    """One GPU cell (the result dict's fields at idx) against a reference cell."""
    assert int(got["count"][idx]) == want["count"], (what, "count")
    assert int(got["count_value"][idx]) == want["count_value"], (what, "count_value")
    if not is_float:
        assert (got["sum"][idx], int(got["min"][idx]), int(got["max"][idx])) == (want["sum"], want["min"], want["max"]), what
        return
    s, mn, mx = float(got["sum"][idx]), float(got["min"][idx]), float(got["max"][idx])
    if math.isnan(want["sum"]) or math.isinf(want["sum"]):
        assert (math.isnan(s) and math.isnan(want["sum"])) or s == want["sum"], (what, s, want["sum"])
    else:
        assert abs(s - want["sum"]) <= want["count_value"] * 2.0 ** -52 * want["abs"], (what, s, want["sum"])
    for g, w in ((mn, want["min"]), (mx, want["max"])):
        if math.isnan(w):
            assert np.float64(g).view(np.uint64) == 0x7FF8000000000000, (what, g)
        else:
            assert g == w and math.copysign(1.0, g) == math.copysign(1.0, w), (what, g, w)


def check(reader, seg_lists, key_cols, val_cols, queries, kind, key_field, value_field, key_min=0, key_span=1, filt=None,
          exclude=None, deleted=None, masks=None, groups=False, mins=None):
    """Runs one batch and compares every query's cells with the reference; returns the result."""
    is_float = np.asarray(val_cols[0][0]).dtype == np.float64
    xs = exclude or [[]] * len(queries)
    if groups:
        got = sdb.ExecuteMatchAggregatesGroupsBatch(reader, queries, value_field, key_field, key_min, key_span, filt=filt,
                                                    exclude=exclude, min_match=mins)
    else:
        got = sdb.ExecuteMatchAggregatesBatch(reader, queries, kind, value_field, key_field, key_min, key_span, filt=filt,
                                              exclude=exclude)
    if key_field is None:
        counts = (sdb.ExecuteCountGroupsBatch(reader, queries, filt=filt, exclude=exclude, min_match=mins) if groups else
                  sdb.ExecuteCountBatch(reader, queries, kind, filt=filt, exclude=exclude))
        assert np.array_equal(got["count"][:, 0], counts) and not got["null"]["count"].any()
    else:
        fc = (sdb.ExecuteFacetCountsGroupsBatch(reader, queries, key_field, key_min, key_span, filt=filt, exclude=exclude,
                                                min_match=mins) if groups else
              sdb.ExecuteFacetCountsBatch(reader, queries, kind, key_field, key_min, key_span, filt=filt, exclude=exclude))
        assert np.array_equal(got["count"], fc["counts"]) and np.array_equal(got["null"]["count"], fc["nulls"])
    okind = "AND" if kind == sdb.AND else "OR"
    for q, (terms, x) in enumerate(zip(queries, xs)):
        if groups:
            cells, null = ar.aggregate_groups(seg_lists, terms, key_cols, val_cols, key_min, key_span, excl=x or [],
                                              deleted=deleted, masks=masks, mins=mins[q] if mins else None)
        else:
            cells, null = ar.aggregate(seg_lists, okind, terms, key_cols, val_cols, key_min, key_span, excl=x or [],
                                       deleted=deleted, masks=masks)
        for b, want in enumerate(cells):
            assert_cell(got, (q, b), want, is_float, (q, terms, b))
        assert_cell(got["null"], q, null, is_float, (q, terms, "NULL"))
    return got


@pytest.fixture(scope="module")
def synth():
    n = 200_000
    oseg, dl, lists = orc.synth_segment(n, list(range(24)))
    rng = np.random.default_rng(23)
    f = rng.normal(size=n) * 1e3
    f[rng.integers(0, n, 300)] = -0.0
    f[rng.integers(0, n, 300)] = 0.0
    specials = rng.normal(size=n)
    specials[rng.integers(0, n, 5)] = np.nan
    specials[rng.integers(0, n, 5)] = np.inf
    specials[rng.integers(0, n, 5)] = -np.inf
    specials[rng.integers(0, n, 50)] = -0.0
    cols = {1: (rng.integers(-1000, 1001, n).astype(np.int64), None),                      # bit-packed
            2: (rng.integers(-500, 500, n).astype(np.int32), None),
            3: (f, None),
            4: (rng.integers(-20, 30, n).astype(np.int64), rng.random(n) < 0.7),            # nullable raw
            5: (rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64), None),                   # raw, full range
            6: (np.zeros(n, np.int64), np.zeros(n, bool)),                                  # all NULL
            7: (specials, rng.random(n) < 0.9),                                             # float64 NaN / inf, nullable
            8: (rng.integers(0, 16, n - 3000).astype(np.int64), None),                      # 16 keys; last 3000 docs NULL
            9: (rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int32), rng.random(n) < 0.8)}  # int32 nullable, full range
    g = to_gpu(oseg, columns={fl: (v, cr.validity_words(m) if m is not None else None) for fl, (v, m) in cols.items()})
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d, _ in lists])
    return dict(g=g, reader=reader, n=n, lists=[d for d, _ in lists], cols=cols)


KEYS = {1: (-1000, 2001), 8: (0, 16), 4: (-25, 60), 2: (-500, 1000)}
VALUES = (1, 2, 3, 4, 5, 7, 9)


def _queries(seed):
    rng = np.random.default_rng(seed)
    qs_or = [sorted(rng.choice(24, size=t, replace=False).tolist()) for t in range(1, 17)]
    qs_and = [sorted(rng.choice(6, size=min(t, 6), replace=False).tolist()) +
              sorted(rng.choice(np.arange(6, 24), size=max(0, t - 6), replace=False).tolist()) for t in range(2, 17)]
    return qs_or, qs_and


def test_every_value_type_ungrouped(synth):
    reader, lists, cols = synth["reader"], [synth["lists"]], synth["cols"]
    qs_or, qs_and = _queries(1)
    assert synth["g"].column_packed(1, synth["n"]) is not None and synth["g"].column_packed(5, synth["n"]) is None
    for v in VALUES + (6,):
        check(reader, lists, None, [cols[v]], qs_or, sdb.OR, None, v)
        check(reader, lists, None, [cols[v]], qs_and, sdb.AND, None, v)


def test_every_value_type_grouped(synth):
    reader, lists, cols = synth["reader"], [synth["lists"]], synth["cols"]
    qs_or, qs_and = _queries(2)
    for k, (lo, span) in KEYS.items():
        for v in VALUES:
            check(reader, lists, [cols[k]], [cols[v]], qs_or[::3], sdb.OR, k, v, lo, span)
            check(reader, lists, [cols[k]], [cols[v]], qs_and[::3], sdb.AND, k, v, lo, span)
    for k in (1, 4, 8):   # value column == key column
        lo, span = KEYS[k]
        check(reader, lists, [cols[k]], [cols[k]], qs_or, sdb.OR, k, k, lo, span)


def test_dict_forms(synth):
    reader, lists, cols = synth["reader"], [synth["lists"]], synth["cols"]
    one = sdb.ExecuteMatchAggregates(reader, [0, 3], sdb.OR, 5)
    (want,), _ = ar.aggregate(lists, "OR", [0, 3], None, [cols[5]])
    assert {f: one[f] for f in FIELDS} == want and one["avg"] == want["sum"] / want["count_value"]
    by_key = sdb.ExecuteMatchAggregates(reader, [0, 3], sdb.OR, 2, key_field=8)
    cells, null = ar.aggregate(lists, "OR", [0, 3], [cols[8]], [cols[2]], 0, 16)
    assert sorted(k for k in by_key if k is not None) == [k for k in range(16) if cells[k]["count"]]
    assert by_key[None]["count"] == null["count"] > 0
    for k, c in enumerate(cells):
        if c["count"]:
            assert {f: by_key[k][f] for f in FIELDS} == c
    empty = sdb.ExecuteMatchAggregates(reader, [1], sdb.OR, 6)
    assert empty["count"] > 0 and empty["count_value"] == 0 and math.isnan(empty["avg"])
    with pytest.raises(ValueError):
        sdb.ExecuteMatchAggregatesBatch(reader, [[0]], sdb.OR, 77)


def test_exclusions_filter_deleted(synth):
    reader, lists, g, n, cols = synth["reader"], [synth["lists"]], synth["g"], synth["n"], synth["cols"]
    rng = np.random.default_rng(5)
    qs, xs = [], []
    for ne in range(1, 17):
        q = sorted(rng.choice(8, size=2, replace=False).tolist())
        qs.append(q)
        xs.append(rng.choice([t for t in range(24) if t not in q], size=ne, replace=False).tolist())
    for kind in (sdb.OR, sdb.AND):
        check(reader, lists, [cols[8]], [cols[3]], qs, kind, 8, 3, 0, 16, exclude=xs)
        check(reader, lists, None, [cols[5]], qs, kind, None, 5, exclude=xs)
    deleted = np.unique(rng.integers(1, n + 1, 9000)).astype(np.uint32)
    qs = [[0, 3], [1], [2, 5, 7, 9], [0, 1]]
    preds = [(2, "BETWEEN", -100, 99), (3, "GE", 0.25, 0), (4, "IS_NULL", 0, 0), (4, "GT", 5, 0)]
    try:
        for with_deleted in (False, True):
            g.stage_docs_mask(deleted if with_deleted else None)
            dele = [deleted] if with_deleted else None
            for kind in (sdb.OR, sdb.AND):
                check(reader, lists, None, [cols[1]], qs, kind, None, 1, deleted=dele)
                for fl, op, lo, hi in preds:
                    m = cr.pred_mask(cols[fl][0], cols[fl][1], op, lo, hi)
                    filt = sdb.pred(fl, op, lo, hi)
                    check(reader, lists, [cols[4]], [cols[fl]], qs, kind, 4, fl, -25, 60, filt=filt, deleted=dele, masks=[m])
                    check(reader, lists, None, [cols[7]], qs, kind, None, 7, filt=filt, deleted=dele, masks=[m])
    finally:
        g.stage_docs_mask(None)


@pytest.mark.parametrize("level", [1, 2])
def test_pruning_levels_identical(synth, level):
    reader = synth["reader"]
    qs = [[0, 3], [1, 4, 9], [2], [5, 6, 7, 8], [10, 11]]
    runs = []
    try:
        for lv in (0, level):
            ctx().set_wand(lv)
            runs.append([sdb.ExecuteMatchAggregatesBatch(reader, qs, kind, v, 1, -1000, 2001) for kind in (sdb.OR, sdb.AND)
                         for v in (5, 3)])
    finally:
        ctx().set_wand(0)
    for a, b in zip(*runs):
        for f in FIELDS:
            assert np.array_equal(a[f], b[f]) or (a[f].dtype == np.float64 and np.allclose(a[f], b[f], rtol=1e-12,
                                                                                              equal_nan=True)), f
            assert np.array_equal(a["null"][f], b["null"][f]), f


def test_extreme_sums_over_items_and_segments():
    """Three segments of INT64_MAX / INT64_MIN values, one list over every doc: thousands of work items each flush a
    128-bit partial whose low word carries; the total is exact."""
    sizes = [1_500_000, 700_001, 3 * W + 5]
    segs, seg_lists, cols = [], [], []
    for i, n in enumerate(sizes):
        o = orc.Segment(n)
        d = np.arange(1, n + 1, dtype=np.uint32)
        o.add_term(d, np.ones(n, np.uint32))
        o.add_term(d[::3], np.ones(len(d[::3]), np.uint32))
        v = np.where(np.arange(n) % 7 == 3, I64_MIN, I64_MAX).astype(np.int64) if i != 1 else np.full(n, I64_MAX, np.int64)
        segs.append(to_gpu(o, columns={1: (v, None)}))
        seg_lists.append([d, d[::3]])
        cols.append((v, None))
    reader = sdb.IndexReader(segs, sum(sizes), sum(sizes), [sum(sizes), sum(len(range(0, n, 3)) for n in sizes)])
    got = check(reader, seg_lists, None, cols, [[0], [1], [0, 1]], sdb.OR, None, 1)
    assert got["sum"][0, 0] == sum(int(c[0].astype(object).sum()) for c in cols)
    check(reader, seg_lists, None, cols, [[0, 1]], sdb.AND, None, 1)


@pytest.fixture(scope="module", params=NORM_WIDTHS, ids=lambda w: f"norms{w or 0}")
def shapes(request):
    oseg, norms, lists = shape_segment(request.param)
    n = oseg.n_docs
    rows = min(n, 3_000_000)   # the 2^30-doc shape: docs past the column's rows have a NULL key and value
    keys = (np.arange(rows, dtype=np.int64) * 7919) % 1009 - 500
    vals = (np.arange(rows, dtype=np.int64) * 104729) % 100003 - 50000
    g = to_gpu(oseg, columns={1: (keys, None), 2: (vals, None)})
    ttf = int(norms.astype(np.uint64).sum()) if norms is not None else n
    reader = sdb.IndexReader([g], n, ttf, [len(d) for _, d, _ in lists])
    return dict(reader=reader, lists=[d for _, d, _ in lists], names=[nm for nm, _, _ in lists], keys=[(keys, None)],
                vals=[(vals, None)])


def test_every_encoding(shapes):
    lists, names, S = shapes["lists"], shapes["names"], shapes
    shape_ids = [t for t, nm in enumerate(names) if not nm.endswith("+lead")]
    pairs = [[t, t + 1] for t in shape_ids]
    for kind in (sdb.OR, sdb.AND):
        check(S["reader"], [lists], S["keys"], S["vals"], pairs, kind, 1, 2, -500, 1009)
        check(S["reader"], [lists], None, S["vals"], pairs, kind, None, 2)
    check(S["reader"], [lists], None, S["vals"], [[t + 1] for t in shape_ids], sdb.OR, None, 2,
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
    keys = np.zeros(n, np.int64)
    keys[np.array(edge) - 1] = 1 + np.arange(len(edge))
    vals = rng.normal(size=n)
    g = to_gpu(oseg, columns={1: (keys, None), 2: (vals, None)})
    reader = sdb.IndexReader([g], n, n, [len(d) for d in lists])
    got = check(reader, [lists], [(keys, None)], [(vals, None)], [[0], [0, 1], [1]], sdb.OR, 1, 2, 0, 11)
    assert got["count"][0].tolist() == [0] + [1] * 10
    assert got["max"][0, 1:].tolist() == vals[np.array(edge) - 1].tolist()


def test_three_segments():
    segs = natural_segments()
    corpus = Corpus(segs)
    rng = np.random.default_rng(12)
    kcols, vcols, gsegs = [], [], []
    for i, o in enumerate(corpus.osegs):
        rows = o.n_docs - 777 if i == 2 else o.n_docs        # segment 2: the last 777 docs have a NULL key and value
        k = rng.integers(-7, 13, rows).astype(np.int32)
        km = rng.random(rows) < 0.9
        v = rng.integers(I64_MIN, I64_MAX, rows, dtype=np.int64)
        vm = rng.random(rows) < 0.85
        kcols.append((k, km))
        vcols.append((v, vm))
        gsegs.append(to_gpu(o, columns={1: (k, cr.validity_words(km)), 2: (v, cr.validity_words(vm))}))
    reader = sdb.IndexReader(gsegs, corpus.docs_with_field, corpus.total_term_freq, corpus.docs_with_term)
    seg_lists = [[np.asarray(d, np.uint32) for d, _ in l] for l in corpus.lists]
    qs = [sorted(rng.choice(corpus.n_terms, size=int(rng.integers(1, 5)), replace=False).tolist()) for _ in range(20)]
    for kind in (sdb.OR, sdb.AND):
        check(reader, seg_lists, kcols, vcols, qs, kind, 1, 2, -7, 20)
        check(reader, seg_lists, None, vcols, qs, kind, None, 2)
    check(reader, seg_lists, kcols, vcols, qs, sdb.OR, 1, 2, -7, 20, exclude=[[3]] * len(qs))


def test_groups_and_min_match(synth):
    """A mixed-shape batch: one-group queries, all-single-term groups, true OR groups and min-match groups, with
    exclusions; the degenerate shapes equal the flat entry's results."""
    reader, lists, cols = synth["reader"], [synth["lists"]], synth["cols"]
    qs = [[[0, 3]], [[1], [4]], [[2], [5, 7]], [[0, 1, 2]], [[6, 8], [9, 10, 11]], [[1, 2, 3, 4]], [[12], [13, 14, 15]]]
    mins = [[1], [1, 1], [1, 1], [2], [1, 2], [3], [1, 2]]
    xs = [[20], None, [21], None, [22, 23], None, [5]]
    for k, v in ((8, 5), (4, 3), (1, 7), (None, 9), (None, 3)):
        lo, span = KEYS.get(k, (0, 1))
        kc = [cols[k]] if k is not None else None
        check(reader, lists, kc, [cols[v]], qs, None, k, v, lo, span, exclude=xs, groups=True, mins=mins)
    flat = sdb.ExecuteMatchAggregatesBatch(reader, [[0, 3], [1, 4]], sdb.OR, 5, 8, 0, 16)
    grp = sdb.ExecuteMatchAggregatesGroupsBatch(reader, [[[0, 3]], [[1, 4]]], 5, 8, 0, 16)
    assert all(np.array_equal(flat[f], grp[f]) for f in FIELDS)
    flat = sdb.ExecuteMatchAggregatesBatch(reader, [[1, 4]], sdb.AND, 3)
    grp = sdb.ExecuteMatchAggregatesGroupsBatch(reader, [[[1], [4]]], 3)
    assert all(np.array_equal(flat[f], grp[f]) for f in FIELDS if f != "sum")
    assert np.allclose(flat["sum"], grp["sum"], rtol=1e-12)   # float64: the order of the additions is unspecified


# ---------------------------------------------------------------- doc ids up to 2^32 - 2
@pytest.fixture(scope="module")
def top():
    c = hd.TopCorpus()
    g = to_gpu(c.oracle_segment())
    g.synth_column(hd.FULL_FIELD, hd.FULL_STREAM, hd.FULL_KIND, 0, hd.TOP)
    g.stage_column(hd.SHORT_FIELD, hd.short_column())
    reader = sdb.IndexReader([g], hd.TOP, hd.TOP, c.docs_with_term)
    yield dict(c=c, g=g, reader=reader)
    g.close()


def test_high_doc_ids(top):
    """Over the matches at the landmarks, with and without deleted docs: the full int32 column's values ungrouped, and
    grouped by themselves under a filter that keeps 4096 keys; the short column's values (NULL for every doc past 2^20)
    ungrouped."""
    c = top["c"]
    lists = [d for _, d, _ in c.lists]
    qs = [[t] for t in c.shapes] + [[t, t + 1] for t in c.shapes if not c.lists[t][0].startswith("spread")]
    try:
        for deleted in (False, True):
            top["g"].stage_docs_mask(c.deleted if deleted else None)
            lo, span = 400000, 4096
            pf = sdb.pred(hd.FULL_FIELD, "BETWEEN", lo, lo + span - 1)
            got = sdb.ExecuteMatchAggregatesBatch(top["reader"], qs, sdb.OR, hd.FULL_FIELD)
            by = sdb.ExecuteMatchAggregatesBatch(top["reader"], qs, sdb.OR, hd.FULL_FIELD, hd.FULL_FIELD, lo, span, filt=pf)
            sh = sdb.ExecuteMatchAggregatesBatch(top["reader"], qs, sdb.OR, hd.SHORT_FIELD)
            full, short = c.small_columns(hd.FULL_FIELD), c.small_columns(hd.SHORT_FIELD)
            for q, p in enumerate(qs):
                docs = cr.match_docs(lists, "OR", p, (), c.deleted if deleted else None).astype(np.uint32)
                (want,), _ = ar.cells_of_docs([c.small(docs)], None, [full], 0, 1)
                assert_cell(got, (q, 0), want, False, p)
                (want,), _ = ar.cells_of_docs([c.small(docs)], None, [short], 0, 1)
                assert_cell(sh, (q, 0), want, False, p)
                v = hd.full_values(docs)
                fd = docs[(v >= lo) & (v < lo + span)]
                cells, null = ar.cells_of_docs([c.small(fd)], [full], [full], lo, span)
                for b in range(span):
                    assert_cell(by, (q, b), cells[b], False, (p, b))
                assert null["count"] == 0 and int(by["null"]["count"][q]) == 0
    finally:
        top["g"].stage_docs_mask(None)


# ---------------------------------------------------------------- errors
def _raw(reader, terms, off, nq, key_field=1, key_min=-1000, key_span=2001, value_field=5, out=True, nulls=True, excl=None,
         xoff=None, filt=None):
    arr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    o = np.zeros(max(nq, 1) * max(key_span, 1), sdb.engine.MATCH_AGG_DTYPE)
    nn = np.zeros(max(nq, 1), sdb.engine.MATCH_AGG_DTYPE)
    return N.lib().sdbg_match_aggregate_batch(sdb.engine._seg_array(reader.segments), len(reader.segments), sdb.OR,
                                              arr(terms), arr(off), nq, arr(excl), arr(xoff),
                                              C.byref(filt) if filt is not None else None, key_field, key_min, key_span,
                                              value_field, arr(o) if out else None, arr(nn) if nulls else None)


def _raw_groups(reader, key_field=1, key_min=-1000, key_span=2001, value_field=5):
    arr = lambda a: a.ctypes.data_as(C.c_void_p)
    t = np.array([0, 1, 2], np.uint32)
    go = np.array([0, 1, 3], np.uint32)
    qgo = np.array([0, 2], np.uint32)
    o = np.zeros(max(key_span, 1), sdb.engine.MATCH_AGG_DTYPE)
    nn = np.zeros(1, sdb.engine.MATCH_AGG_DTYPE)
    return N.lib().sdbg_match_aggregate_batch_groups_min(sdb.engine._seg_array(reader.segments), len(reader.segments), arr(t),
                                                         arr(go), arr(qgo), None, 1, None, None, None, key_field, key_min,
                                                         key_span, value_field, arr(o), arr(nn))


def test_errors_queue_nothing(synth):
    reader = synth["reader"]
    t = np.array([0, 1], np.uint32)
    off = np.array([0, 2], np.uint32)
    assert _raw(reader, t, off, 1) == 0
    assert _raw(reader, t, off, 1, key_field=N.UINT64_MAX, key_min=0, key_span=1) == 0
    assert _raw_groups(reader) == 0
    cases = [(dict(out=False), -1), (dict(nulls=False), -1), (dict(key_span=0), -1), (dict(key_span=4097), -7),
             (dict(key_span=4096), 0), (dict(key_field=77), -5), (dict(key_field=3, key_min=0, key_span=10), -7),
             (dict(value_field=77), -5), (dict(key_field=N.UINT64_MAX, key_min=0, key_span=2), -1),
             (dict(key_field=N.UINT64_MAX, key_min=1, key_span=1), -1),
             (dict(key_min=I64_MAX - 98, key_span=100), -1), (dict(filt=sdb.pred(77, "LT", 5)), -5),
             (dict(excl=np.arange(2, 19, dtype=np.uint32), xoff=np.array([0, 17], np.uint32)), -7)]
    for kw, code in cases:
        if code:
            before = ctx().launches
            assert _raw(reader, t, off, 1, **kw) == code, kw
            assert ctx().launches == before, kw
        else:
            assert _raw(reader, t, off, 1, **kw) == 0, kw
    before = ctx().launches
    assert _raw(reader, None, off, 1) == -1 and _raw(reader, t, off, 0) == -1
    assert _raw(reader, np.array([0, 10_000], np.uint32), off, 1) == -1
    assert _raw_groups(reader, key_span=4097) == -7 and _raw_groups(reader, value_field=77) == -5
    assert _raw_groups(reader, key_field=N.UINT64_MAX, key_min=0, key_span=3) == -1
    assert ctx().launches == before
    n = 1000
    o2 = orc.Segment(n)
    o2.add_term(np.arange(1, n + 1, dtype=np.uint32), np.ones(n, np.uint32))
    g_a = to_gpu(o2, columns={1: (np.arange(n, dtype=np.int64), None), 2: (np.arange(n, dtype=np.int64), None)})
    g_b = to_gpu(o2, columns={1: (np.arange(n, dtype=np.int64), None), 2: (np.arange(n, dtype=np.float64), None)})
    mixed = sdb.IndexReader([g_a, g_b], 2 * n, 2 * n, [2 * n])
    one = np.array([0], np.uint32)
    before = ctx().launches
    assert _raw(mixed, one, np.array([0, 1], np.uint32), 1, key_min=0, key_span=n, value_field=2) == -1
    assert ctx().launches == before
    # after the scan: keys outside the range
    assert _raw(reader, t, off, 1, key_min=-999, key_span=2000) == -1
    with pytest.raises(N.SdbgError, match="outside"):
        sdb.ExecuteMatchAggregatesBatch(reader, [[0, 1]], sdb.OR, 5, 1, 0, 1000)


def test_adapter_match_agg_scan():
    """GpuMatchAggScan through adapter_selftest, flat and grouped queries: the int32 column 9 grouped by the 2001-key
    column 15 (rows in key order) and the float64 column 16 ungrouped (one row), without and with the filter; a key range
    wider than 4096 values throws SDBG_EUNSUPPORTED."""
    from serenedb_b200 import build as b
    exe = b.build_adapters()
    n = 200_000
    oseg, _, _ = orc.synth_segment_mt(n, 0, 8, threads=4)
    lists = [oseg.decode_term(t)[0] for t in range(8)]
    key = orc.synth_column(15, 3, 1, n)
    val = orc.synth_column(2, 1, 1, n)   # column 9: kind 6 is kind 1 stored as int32
    fval = orc.synth_column(16, 4, 1, n)
    mask = cr.pred_mask(orc.synth_column(2, 1, 1, n), None, "BETWEEN", 250000, 749999)
    for mode in ([], ["groups"]):
        res = subprocess.run([exe, str(n), "aggregate"] + mode, capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stdout + res.stderr
        lines = [json.loads(line.replace("nan", "NaN")) for line in res.stdout.strip().splitlines()]
        assert len(lines) == 9 and lines[-1] == {"wide_error": -7}
        for out in lines[:-1]:
            x = [3] if out["excl"] else []
            m = [mask if out["filter"] else None]
            if mode:
                grp, mins = ([[2], [5, 6]], None) if out["kind"] == 0 else ([[2, 5, 6]], [2])
                cells, null = ar.aggregate_groups([lists], grp, [(key, None)], [(val, None)], -1000, 2001, excl=x, masks=m, mins=mins)
                (whole,), _ = ar.aggregate_groups([lists], grp, None, [(fval, None)], excl=x, masks=m, mins=mins)
            else:
                kind = "AND" if out["kind"] == sdb.AND else "OR"
                cells, null = ar.aggregate([lists], kind, [2, 5], [(key, None)], [(val, None)], -1000, 2001, excl=x, masks=m)
                (whole,), _ = ar.aggregate([lists], kind, [2, 5], None, [(fval, None)], excl=x, masks=m)
            assert null["count"] == 0
            gr = out["grouped"]
            want = [(k - 1000, c) for k, c in enumerate(cells) if c["count"]]
            assert gr["keys"] == [k for k, _ in want] and gr["valid"] == [1] * len(want)
            assert gr["chunks"] == (1 if want else 0) and gr["rows_after"] == 0
            for i, (_, c) in enumerate(want):
                s = (gr["sum_hi"][i] << 64) | (gr["sum_lo"][i] & 0xFFFFFFFFFFFFFFFF)
                assert (gr["count"][i], gr["count_value"][i], s, gr["min"][i], gr["max"][i]) == \
                    (c["count"], c["count_value"], c["sum"], c["min"], c["max"])
                assert gr["avg"][i] == pytest.approx(c["sum"] / c["count_value"], rel=1e-12)
            un = out["ungrouped"]
            assert un["chunks"] == 1 and un["count"] == [whole["count"]] and un["count_value"] == [whole["count_value"]]
            got = {"count": [un["count"][0]], "count_value": [un["count_value"][0]], "sum": [un["sum_f64"][0]],
                   "min": [np.int64(un["min"][0]).view(np.float64)], "max": [np.int64(un["max"][0]).view(np.float64)]}
            assert_cell(got, 0, whole, True, out)


def test_batch_4096_at_bench_scale():
    """bench.py's corpus: 10 M docs, its 4096 two-term ORs (bench.make_queries); SUM / MIN / MAX of the bit-packed
    2001-key column, ungrouped and grouped by a 16-key column; counts against the count and facet entries for every
    query, 32 sampled queries against StreamScoredDocs + gather."""
    import bench
    n = 10_000_000
    g = sdb.Segment(ctx(), n)
    dc, sum_dl = g.synth_corpus(0, 0, bench.N_TERMS)
    g.synth_column(1, 13, 3, 1, n)
    g.synth_column(2, 14, 4, 1, n)
    keys16 = (np.arange(n, dtype=np.int64) * 2654435761) % 16
    g.stage_column(3, keys16)
    assert g.column_packed(1, n) is not None
    reader = sdb.IndexReader([g], n, sum_dl, dc)
    qs = bench.make_queries(4096)
    counts = sdb.ExecuteCountBatch(reader, qs, sdb.OR)
    whole = sdb.ExecuteMatchAggregatesBatch(reader, qs, sdb.OR, 1)
    fwhole = sdb.ExecuteMatchAggregatesBatch(reader, qs, sdb.OR, 2)
    by = sdb.ExecuteMatchAggregatesBatch(reader, qs, sdb.OR, 1, 3, 0, 16)
    assert np.array_equal(whole["count"][:, 0], counts) and np.array_equal(by["count"].sum(axis=1), counts)
    assert np.array_equal(by["count"], sdb.ExecuteFacetCountsBatch(reader, qs, sdb.OR, 3, 0, 16)["counts"])
    for q in range(0, 4096, 128):
        docs, _ = sdb.StreamScoredDocs(reader, 0, qs[q], sdb.OR, sdb.BM25())
        v, _ = g.gather(1, docs, np.int64)
        f, _ = g.gather(2, docs, np.float64)
        k = keys16[docs.astype(np.int64) - 1]
        (want,), _ = ar.cells_of_docs([np.arange(1, len(docs) + 1)], None, [(v, None)], 0, 1)
        assert_cell(whole, (q, 0), want, False, q)
        (want,), _ = ar.cells_of_docs([np.arange(1, len(docs) + 1)], None, [(f, None)], 0, 1)
        assert_cell(fwhole, (q, 0), want, True, q)
        cells, _ = ar.cells_of_docs([np.arange(1, len(docs) + 1)], [(k, None)], [(v, None)], 0, 16)
        for b in range(16):
            assert_cell(by, (q, b), cells[b], False, (q, b))
