"""Sorted scan and facet counts of OR-group and min-match queries (sdbg_match_topk_by_column_batch_groups_min /
sdbg_match_facet_counts_batch_groups_min, ExecuteTopKByColumnGroupsBatch / ExecuteFacetCountsGroupsBatch) on the GPU:
equal to tests/groups_column_reference.py, n_out == min(k, count) and
sum(counts) + nulls == count against ExecuteCountGroupsBatch. Covers nested m = 1 groups and m >= 2 groups alone and in
an AND, exclusions, the hybrid filter (also on the sort / key column), deleted docs, every sort and key column type,
pruning levels, three segments with a group short of non-empty lists in one, zonemap skipping with seed windows, every
block encoding, window edges, mixed-shape batches, the shared-memory extremes, the error codes, the adapters and a
4096-query batch over the 10 M-doc benchmark corpus."""
import ctypes as C
import json
import subprocess

import numpy as np
import pytest

import count_reference as cr
import groups_column_reference as gr
import orc
import serenedb_b200 as sdb
from serenedb_b200 import _native as N
from gpu_util import ctx, to_gpu
from shape_corpora import NORM_WIDTHS, Corpus, natural_segments, shape_segment

pytestmark = pytest.mark.gpu

W = 1 << 16
ORDERS = [(d, nf) for d in (False, True) for nf in (False, True)]
# nested m = 1 groups, m >= 2 groups alone and inside an AND
QS = [[[0], [1, 2]], [[3, 4], [5, 6, 7]], [[8, 9, 10]], [[11], [12, 13, 14]], [[1, 5, 9]], [[2, 3, 4, 8]],
      [[0, 6], [7], [15, 16]], [[17, 18, 19, 20], [21, 22]]]
MS = [[1, 1], [1, 1], [2], [1, 2], [2], [3], [1, 1, 1], [2, 1]]
XS = [[], [20], [], [21, 22], [], [0], [], [3]]


def check_sort(reader, seg_lists, columns, queries, mins, field, k, desc=False, nf=False, filt=None, exclude=None,
               deleted=None, masks=None):
    got = sdb.ExecuteTopKByColumnGroupsBatch(reader, queries, field, k, desc, nf, filt=filt, exclude=exclude,
                                             min_match=mins)
    counts = sdb.ExecuteCountGroupsBatch(reader, queries, filt=filt, exclude=exclude, min_match=mins)
    xs = exclude or [[]] * len(queries)
    ms = mins or [None] * len(queries)
    for q, groups in enumerate(queries):
        want = gr.sorted_hits(seg_lists, groups, columns, desc, nf, k=k, excl=xs[q] or [], deleted=deleted, masks=masks,
                              mins=ms[q])
        n = int(got["n_out"][q])
        assert n == min(k, int(counts[q])) == len(want["docs"]), (q, groups, n, counts[q])
        assert np.array_equal(got["docs"][q], want["docs"]), (q, groups, desc, nf)
        assert np.array_equal(got["segs"][q], want["segs"])
        assert np.array_equal(got["nulls"][q], want["nulls"])
        assert got["values"][q].dtype == want["values"].dtype
        assert np.array_equal(got["values"][q].view(np.uint8), want["values"].view(np.uint8))
    return got


def check_facet(reader, seg_lists, columns, queries, mins, field, key_min=None, key_span=None, filt=None, exclude=None,
                deleted=None, masks=None):
    got = sdb.ExecuteFacetCountsGroupsBatch(reader, queries, field, key_min, key_span, filt=filt, exclude=exclude,
                                            min_match=mins)
    counts = sdb.ExecuteCountGroupsBatch(reader, queries, filt=filt, exclude=exclude, min_match=mins)
    xs = exclude or [[]] * len(queries)
    ms = mins or [None] * len(queries)
    span = got["counts"].shape[1]
    for q, groups in enumerate(queries):
        wc, wn = gr.facet_counts(seg_lists, groups, columns, got["key_min"], span, excl=xs[q] or [], deleted=deleted,
                                 masks=masks, mins=ms[q])
        assert np.array_equal(got["counts"][q], wc), (q, groups)
        assert int(got["nulls"][q]) == wn
        assert int(got["counts"][q].sum()) + wn == int(counts[q])
    return got


@pytest.fixture(scope="module")
def synth():
    n = 200_000
    oseg, dl, lists = orc.synth_segment(n, list(range(24)))
    rng = np.random.default_rng(7)
    fvals = rng.normal(size=n)
    fvals[rng.integers(0, n, 300)] = np.nan
    fvals[rng.integers(0, n, 50)] = -np.inf
    fvals[rng.integers(0, n, 100)] = -0.0
    i64 = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, endpoint=True)
    cols = {1: (i64, None),                                                         # int64, full range: held raw
            2: (rng.integers(-1000, 1000, n).astype(np.int32), None),
            3: (fvals, None),
            4: (rng.integers(0, 50, n).astype(np.int64), rng.random(n) < 0.7),     # nullable
            5: (np.full(n - 5000, 42, np.int64), None),                             # constant; last 5000 docs NULL
            6: (rng.integers(0, 300, n).astype(np.int64), None)}                    # narrow: bit-packed
    g = to_gpu(oseg, columns={f: (v, cr.validity_words(m) if m is not None else None) for f, (v, m) in cols.items()})
    reader = sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d, _ in lists])
    return dict(g=g, reader=reader, n=n, lists=[d for d, _ in lists], cols=cols)


def test_every_sort_column_and_key(synth):
    reader, lists, cols = synth["reader"], [synth["lists"]], synth["cols"]
    assert synth["g"].column_packed(6, synth["n"]) is not None and synth["g"].column_packed(1, synth["n"]) is None
    for f in (1, 2, 3, 4, 5, 6):
        for desc, nf in ORDERS:
            check_sort(reader, lists, [cols[f]], QS, MS, f, 100, desc, nf, exclude=XS)
    for f in (2, 4, 5, 6):
        check_facet(reader, lists, [cols[f]], QS, MS, f, exclude=XS)
    check_facet(reader, lists, [cols[6]], QS, None, 6)                                   # min_match NULL: all 1


def test_filter_and_deleted_docs(synth):
    reader, lists, g, n, cols = synth["reader"], [synth["lists"]], synth["g"], synth["n"], synth["cols"]
    rng = np.random.default_rng(8)
    deleted = np.unique(rng.integers(1, n + 1, 9000)).astype(np.uint32)
    preds = [(2, "BETWEEN", -500, 499), (3, "GE", 0.25, 0), (4, "GT", 20, 0), (4, "IS_NULL", 0, 0)]
    try:
        for with_deleted in (False, True):
            g.stage_docs_mask(deleted if with_deleted else None)
            dele = [deleted] if with_deleted else None
            check_sort(reader, lists, [cols[6]], QS, MS, 6, 64, True, False, exclude=XS, deleted=dele)
            check_facet(reader, lists, [cols[6]], QS, MS, 6, exclude=XS, deleted=dele)
            for f, op, lo, hi in preds:
                m = cr.pred_mask(cols[f][0], cols[f][1], op, lo, hi)
                kw = dict(filt=sdb.pred(f, op, lo, hi), exclude=XS, deleted=dele, masks=[m])
                for sf in sorted({f, 3}):                                             # filter column == sort column too
                    check_sort(reader, lists, [cols[sf]], QS, MS, sf, 64, sf == 3, True, **kw)
                if f != 3:                                                            # filter column == key column
                    check_facet(reader, lists, [cols[f]], QS, MS, f, **kw)
    finally:
        g.stage_docs_mask(None)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_pruning_levels_identical(synth, level):
    reader, lists, cols = synth["reader"], [synth["lists"]], synth["cols"]
    try:
        ctx().set_wand(level)
        for f in (1, 3, 6):
            for desc, nf in ORDERS:
                check_sort(reader, lists, [cols[f]], QS, MS, f, 300, desc, nf, exclude=XS)
        check_facet(reader, lists, [cols[2]], QS, MS, 2, exclude=XS)
    finally:
        ctx().set_wand(0)


def test_three_segments_with_a_group_short_in_one():
    segs = natural_segments()
    norms, lists = segs[1]
    lists[8] = (np.zeros(0, np.uint32), np.zeros(0, np.uint32))          # terms 8 and 9 hold no doc in segment 1
    lists[9] = (np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    corpus = Corpus(segs)
    rng = np.random.default_rng(12)
    cols, gsegs = [], []
    for o in corpus.osegs:
        v = rng.integers(0, 20, o.n_docs).astype(np.int32)   # many ties across segments
        m = rng.random(o.n_docs) < 0.9
        cols.append((v, m))
        gsegs.append(to_gpu(o, columns={1: (v, cr.validity_words(m))}))
    reader = sdb.IndexReader(gsegs, corpus.docs_with_field, corpus.total_term_freq, corpus.docs_with_term)
    seg_lists = [[np.asarray(d, np.uint32) for d, _ in l] for l in corpus.lists]
    qs = [[[0, 1, 2]], [[3], [4, 5, 6, 7]], [[8, 9, 0]], [[0], [8, 9, 1]], [[8, 9, 1, 2]], [[1], [2, 3]]]
    ms = [[2], [1, 2], [2], [1, 2], [3], [1, 1]]
    xs = [[], [2], [], [4], [], [5]]
    for desc, nf in ORDERS:
        check_sort(reader, seg_lists, cols, qs, ms, 1, 40, desc, nf, exclude=xs)
    check_facet(reader, seg_lists, cols, qs, ms, 1, exclude=xs)


def _scan_stats():
    t, s = C.c_uint64(), C.c_uint64()
    N.check(N.lib().sdbg_scan_stats(ctx()._h, C.byref(t), C.byref(s)))
    return t.value, s.value


@pytest.fixture(scope="module")
def clustered():
    """ts = row / 100 over 1 M docs (DESC: newest first)."""
    n = 1_000_000
    oseg, dl, lists = orc.synth_segment(n, list(range(8)))
    lists = [d for d, _ in lists]
    ts = (np.arange(n) // 100).astype(np.int64)
    g = to_gpu(oseg, columns={1: (ts, None)})
    return dict(reader=sdb.IndexReader([g], n, int(dl.sum()), [len(d) for d in lists]), lists=[lists], cols=[(ts, None)])


@pytest.mark.parametrize("level", [1, 2])
def test_clustered_column_skips_windows_with_seeds(clustered, level):
    qs = [[[0], [1, 2]], [[3, 4, 5]], [[1], [2, 6, 7]], [[0, 3], [4, 5]]]
    ms = [[1, 1], [2], [1, 2], [1, 1]]
    try:
        for desc in (True, False):
            ctx().set_wand(0)
            base = check_sort(clustered["reader"], clustered["lists"], clustered["cols"], qs, ms, 1, 100, desc)
            ctx().set_wand(level)
            got = check_sort(clustered["reader"], clustered["lists"], clustered["cols"], qs, ms, 1, 100, desc)
            judged, skipped = _scan_stats()
            assert judged > 0 and skipped > 0, (desc, judged, skipped)
            assert all(np.array_equal(a, b) for a, b in zip(got["docs"], base["docs"]))
    finally:
        ctx().set_wand(0)


def test_mixed_shape_batch(clustered):
    """Shapes 0 (one group), 1 (single-term groups, also from m = s) and 2 in one call: results in the caller's order,
    each equal to the flat entry's for shapes 0 / 1, and scan stats equal to the sum over the shapes run one at a time."""
    reader, lists, cols = clustered["reader"], clustered["lists"], clustered["cols"]
    qs = [[[0], [1, 2]], [[3, 4]], [[5], [6]], [[1, 2, 3]], [[0, 1, 2]], [[7]], [[4], [5, 6]]]
    ms = [[1, 1], [1], [1, 1], [3], [2], [1], [1, 1]]
    shape = [2, 0, 1, 1, 2, 0, 2]
    xs = [[], [5], [], [0], [], [], [7]]
    try:
        ctx().set_wand(2)
        got = check_sort(reader, lists, cols, qs, ms, 1, 50, True, exclude=xs)
        stats = _scan_stats()
        check_facet(reader, lists, cols, qs, ms, 1, exclude=xs)
        total = np.zeros(2, np.uint64)
        for sh in (0, 1, 2):
            sub = [q for q in range(len(qs)) if shape[q] == sh]
            part = sdb.ExecuteTopKByColumnGroupsBatch(reader, [qs[q] for q in sub], 1, 50, True,
                                                      exclude=[xs[q] for q in sub], min_match=[ms[q] for q in sub])
            total += np.array(_scan_stats(), np.uint64)
            for j, q in enumerate(sub):
                assert np.array_equal(part["docs"][j], got["docs"][q])
        assert stats == tuple(int(v) for v in total) and stats[1] > 0, (stats, total)
        flat = sdb.ExecuteTopKByColumnBatch(reader, [[3, 4], [7]], sdb.OR, 1, 50, True, exclude=[[5], []])
        assert np.array_equal(flat["docs"][0], got["docs"][1]) and np.array_equal(flat["docs"][1], got["docs"][5])
        flat = sdb.ExecuteTopKByColumnBatch(reader, [[5, 6], [1, 2, 3]], sdb.AND, 1, 50, True, exclude=[[], [0]])
        assert np.array_equal(flat["docs"][0], got["docs"][2]) and np.array_equal(flat["docs"][1], got["docs"][3])
        fa = sdb.ExecuteFacetCountsBatch(reader, [[5, 6]], sdb.AND, 1)
        fg = sdb.ExecuteFacetCountsGroupsBatch(reader, [[[5], [6]]], 1)
        assert fa["key_min"] == fg["key_min"] and np.array_equal(fa["counts"], fg["counts"])
    finally:
        ctx().set_wand(0)


@pytest.fixture(scope="module", params=NORM_WIDTHS, ids=lambda w: f"norms{w or 0}")
def shapes(request):
    oseg, norms, lists = shape_segment(request.param)
    n = oseg.n_docs
    rows = min(n, 3_000_000)   # the 2^30-doc shape: docs past the column's rows are NULL
    vals = (np.arange(rows, dtype=np.int64) * 7919) % 100_003
    keys = (np.arange(rows, dtype=np.int64) * 31) % 4001 - 2000
    g = to_gpu(oseg, columns={1: (vals, None), 2: (keys, None)})
    ttf = int(norms.astype(np.uint64).sum()) if norms is not None else n
    reader = sdb.IndexReader([g], n, ttf, [len(d) for _, d, _ in lists])
    return dict(reader=reader, lists=[d for _, d, _ in lists], names=[nm for nm, _, _ in lists], vals=vals, keys=keys)


def test_every_encoding_as_group_member(shapes):
    lists, L = shapes["lists"], len(shapes["lists"])
    shape_ids = [t for t, nm in enumerate(shapes["names"]) if not nm.endswith("+lead")]
    qs = [[[t, (t + 1) % L, (t + 3) % L]] for t in shape_ids] + [[[(t + 5) % L], [t, (t + 2) % L]] for t in shape_ids]
    ms = [[2]] * len(shape_ids) + [[1, 1]] * len(shape_ids)
    xs = [[]] * len(shape_ids) + [[(t + 7) % L] for t in shape_ids]
    check_sort(shapes["reader"], [lists], [(shapes["vals"], None)], qs, ms, 1, 200, True, False, exclude=xs)
    check_facet(shapes["reader"], [lists], [(shapes["keys"], None)], qs, ms, 2, -2000, 4001, exclude=xs)


def test_window_edges():
    n = 3 * W + 17
    edge = [1, W - 1, W, W + 1, 2 * W - 1, 2 * W, 3 * W, n - 1, n]
    rng = np.random.default_rng(n)
    oseg = orc.Segment(n)
    lists = [np.unique(np.array(edge, np.uint32)),
             np.unique(np.concatenate([edge[::2], rng.integers(1, n + 1, 3000)])).astype(np.uint32),
             np.unique(np.concatenate([np.arange(W - 200, W + 200), np.arange(n - 300, n + 1)])).astype(np.uint32),
             np.unique(np.concatenate([np.flatnonzero(rng.random(n) < 0.4) + 1, edge])).astype(np.uint32)]
    for d in lists:
        oseg.add_term(d, np.ones(len(d), np.uint32))
    vals = np.zeros(n, np.int64)
    vals[np.array(edge) - 1] = 1000 + np.arange(len(edge))   # the edge docs hold the largest values
    g = to_gpu(oseg, columns={1: (vals, None)})
    reader = sdb.IndexReader([g], n, n, [len(d) for d in lists])
    qs = [[[0, 1, 2]], [[1], [0, 2, 3]], [[0, 2], [1, 3]], [[3, 0, 2]]]
    ms = [[2], [1, 2], [1, 1], [2]]
    try:
        for level in (0, 2):
            ctx().set_wand(level)
            for desc, nf in ORDERS:
                check_sort(reader, [lists], [(vals, None)], qs, ms, 1, 5, desc, nf)
            check_facet(reader, [lists], [(vals, None)], qs, ms, 1, 0, 1009)
    finally:
        ctx().set_wand(0)


def test_shared_memory_extremes():
    """`15 of 16` (4 counter planes) with k = 4096 (8192 keys: 128 KB) and with key_span = 32768 (128 KB)."""
    n = 100_000
    docs = np.arange(1, n + 1, dtype=np.uint32)
    oseg = orc.Segment(n)
    lists = [docs[docs % 17 != t] for t in range(16)]                    # a doc misses at most one of the 16 terms
    for d in lists:
        oseg.add_term(d, np.ones(len(d), np.uint32))
    rng = np.random.default_rng(15)
    vals = rng.integers(0, 1 << 40, n).astype(np.int64)
    keys = rng.integers(0, 32768, n).astype(np.int64)
    keys[:2] = (0, 32767)
    g = to_gpu(oseg, columns={1: (vals, None), 2: (keys, None)})
    reader = sdb.IndexReader([g], n, n, [len(d) for d in lists])
    qs = [[list(range(16))], [[0], list(range(1, 16))]]
    ms = [[15], [1, 14]]
    for level in (0, 2):
        ctx().set_wand(level)
        try:
            got = check_sort(reader, [lists], [(vals, None)], qs, ms, 1, 4096, level == 2)
            assert np.all(got["n_out"] == 4096)
        finally:
            ctx().set_wand(0)
    got = check_facet(reader, [lists], [(keys, None)], qs, ms, 2, 0, 32768)
    assert got["counts"].shape == (2, 32768) and got["counts"][0].sum() > 0


def _raw(reader, fn, ids, group_off, qgo, gmin, nq, field=1, k=10, key_min=0, key_span=2000, out=True, excl=None,
         xoff=None, filt=None):
    arr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    segs = sdb.engine._seg_array(reader.segments)
    fp = C.byref(filt) if filt is not None else None
    if fn == "sort":
        hits = np.zeros(max(nq, 1) * max(k, 1), sdb.engine.SORT_HIT_DTYPE)
        no = np.zeros(max(nq, 1), np.uint32)
        return N.lib().sdbg_match_topk_by_column_batch_groups_min(segs, len(reader.segments), arr(ids), arr(group_off), arr(qgo),
                                                                  arr(gmin), nq, arr(excl), arr(xoff), fp, field, 0, 0, k,
                                                                  arr(hits) if out else None, arr(no))
    counts = np.zeros((max(nq, 1), max(min(key_span, 40000), 1)), np.uint64)
    nulls = np.zeros(max(nq, 1), np.uint64)
    return N.lib().sdbg_match_facet_counts_batch_groups_min(segs, len(reader.segments), arr(ids), arr(group_off), arr(qgo),
                                                            arr(gmin), nq, arr(excl), arr(xoff), fp, field, key_min, key_span,
                                                            arr(counts) if out else None, arr(nulls))


def test_errors_queue_nothing(synth):
    reader = synth["reader"]
    u = lambda *v: np.array(v, np.uint32)
    ids, go, qgo = u(0, 1, 2), u(0, 1, 3), u(0, 2)
    for fn, field in (("sort", 1), ("facet", 2)):
        assert _raw(reader, fn, ids, go, qgo, u(1, 2), 1, field=field, key_min=-1000) == 0
        before = ctx().launches
        bad = [dict(gmin=u(1, 0)), dict(gmin=u(1, 3)), dict(go=u(0, 1, 1, 3), qgo=u(0, 3), gmin=u(1, 1, 1)),
               dict(ids=u(0, 1, 0)), dict(ids=np.arange(17, dtype=np.uint32), go=u(0, 1, 17)),
               dict(go=np.arange(18, dtype=np.uint32), qgo=u(0, 17), ids=np.arange(17, dtype=np.uint32), gmin=None),
               dict(ids=u(0, 1, 10_000)), dict(field=77), dict(filt=sdb.pred(77, "LT", 5)), dict(nq=0), dict(out=False),
               dict(excl=np.arange(3, 20, dtype=np.uint32), xoff=u(0, 17)), dict(xoff=u(0, 1))]
        bad += [dict(k=0), dict(k=4097)] if fn == "sort" else [dict(key_span=0), dict(key_span=32769), dict(field=3)]
        codes = {}
        for kw in bad:
            args = dict(ids=ids, go=go, qgo=qgo, gmin=u(1, 2), nq=1, field=field)
            args.update(kw)
            rc = _raw(reader, fn, args.pop("ids"), args.pop("go"), args.pop("qgo"), args.pop("gmin"), args.pop("nq"), **args)
            codes[str(sorted(kw))[:60]] = rc
            assert rc != 0, (fn, kw)
        assert ctx().launches == before, fn
        # a mixed batch whose shape-2 query is malformed: the valid shape-0 query is not run either
        assert _raw(reader, fn, u(0, 1, 2, 3, 10_000), u(0, 2, 3, 5), u(0, 1, 3), u(1, 1, 1), 2, field=field,
                    key_min=-1000) == -1
        assert ctx().launches == before, fn
    r = lambda fn, **kw: _raw(reader, fn, kw.pop("ids", ids), kw.pop("go", go), qgo, kw.pop("gmin", u(1, 2)), 1, **kw)
    assert r("sort", k=4097) == -7 and r("sort", k=0) == -1 and r("sort", field=77) == -5 and r("sort", out=False) == -1
    assert r("facet", field=3) == -7 and r("facet", field=2, key_span=32769) == -7 and r("facet", field=77) == -5
    assert r("facet", field=2, key_span=0) == -1 and r("facet", field=2, key_min=2**63 - 10, key_span=100) == -1
    assert r("sort", gmin=u(1, 3)) == -1 and r("sort", ids=np.arange(17, dtype=np.uint32), go=u(0, 1, 17)) == -7
    assert r("facet", field=2, key_min=-999, key_span=2000) == -1                        # found after the scan
    with pytest.raises(N.SdbgError, match="outside"):
        sdb.ExecuteFacetCountsGroupsBatch(reader, [[[0], [1, 2]]], 2, 0, 1000)


def _run_selftest(mode):
    from serenedb_b200 import build as b
    exe = b.build_adapters()
    res = subprocess.run([exe, "200000", mode, "groups"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    return [json.loads(l) for l in res.stdout.strip().splitlines()]


def _selftest_corpus():
    n = 200_000
    oseg, _, _ = orc.synth_segment_mt(n, 0, 8, threads=4)
    lists = [oseg.decode_term(t)[0] for t in range(8)]
    fcol = orc.synth_column(2, 1, 1, n)   # column 9: kind 6 is kind 1 stored as int32
    return lists, fcol.astype(np.int32), cr.pred_mask(fcol, None, "BETWEEN", 250000, 749999)


GROUP_QUERIES = [([[2], [5, 6]], [1, 1]), ([[2, 5, 6]], [2])]


def test_adapter_sorted_scan_with_groups():
    lines = _run_selftest("sorted")
    assert len(lines) == 32
    lists, col, mask = _selftest_corpus()
    for out in lines:
        groups, mins = GROUP_QUERIES[out["query"]]
        want = gr.sorted_hits([lists], groups, [(col, None)], bool(out["desc"]), bool(out["nulls_first"]), k=4096,
                              excl=[3] if out["excl"] else [], masks=[mask if out["filter"] else None],
                              mins=mins)
        assert out["docs"] == want["docs"].tolist()
        assert out["values"] == want["values"].astype(np.int64).tolist()
        assert out["valid"] == (~want["nulls"]).astype(int).tolist()
        assert out["max_chunk"] <= 2048 and out["chunks"] == -(-len(want["docs"]) // 2048) and out["rows_after"] == 0


def test_adapter_facet_scan_with_groups():
    lines = _run_selftest("facet")
    assert len(lines) == 9 and lines[-1] == {"wide_error": -7}
    lists, _, mask = _selftest_corpus()
    key = orc.synth_column(15, 3, 1, 200_000)
    for out in lines[:-1]:
        groups, mins = GROUP_QUERIES[out["kind"]]
        want = gr.facet_dict([lists], groups, [(key, None)], excl=[3] if out["excl"] else [],
                             masks=[mask if out["filter"] else None], mins=mins)
        assert sum(want.values()) > 0
        assert out["keys"] == sorted(want) and out["counts"] == [want[k] for k in sorted(want)]
        assert out["rows_after"] == 0


def test_batch_4096_at_bench_scale():
    """bench.py's corpus: 10 M docs, 4096 `2 of (a | b | c)` queries, sorted at k = 1000 by a uniform column (levels 0
    and 2) and faceted on the 2001-key column: the invariants for every query, 64 sampled queries against the doc lists
    from StreamScoredDocs + gather."""
    import bench
    n = 10_000_000
    g = sdb.Segment(ctx(), n)
    dc, sum_dl = g.synth_corpus(0, 0, bench.N_TERMS)
    g.synth_column(1, 11, 1, 1, n)
    g.synth_column(2, 13, 3, 1, n)
    reader = sdb.IndexReader([g], n, sum_dl, dc)
    rng = np.random.default_rng(2027)
    qs = [[sorted(rng.choice(bench.N_TERMS, 3, replace=False).tolist())] for _ in range(4096)]
    ms = [[2]] * 4096
    k = 1000
    counts = sdb.ExecuteCountGroupsBatch(reader, qs, min_match=ms)
    assert counts.sum() > 0
    fac = sdb.ExecuteFacetCountsGroupsBatch(reader, qs, 2, -1000, 2001, min_match=ms)
    assert np.array_equal(fac["counts"].sum(axis=1) + fac["nulls"], counts)
    try:
        for level in (0, 2):
            ctx().set_wand(level)
            got = sdb.ExecuteTopKByColumnGroupsBatch(reader, qs, 1, k, min_match=ms)
            assert np.array_equal(got["n_out"], np.minimum(counts, k))
            for q in range(0, 4096, 64):
                term_docs = [sdb.StreamScoredDocs(reader, 0, [t], sdb.OR, sdb.BM25())[0] for t in qs[q][0]]
                docs, hits = np.unique(np.concatenate(term_docs), return_counts=True)
                docs = docs[hits >= 2]
                vals, valid = g.gather(1, docs, np.int64)
                assert valid.all()
                o = np.lexsort((docs, vals))[:k]
                assert np.array_equal(got["docs"][q], docs[o]), q
                assert np.array_equal(got["values"][q], vals[o]), q
                if level == 0:
                    keys, _ = g.gather(2, docs, np.int64)
                    assert np.array_equal(fac["counts"][q], np.bincount(keys + 1000, minlength=2001).astype(np.uint64)), q
    finally:
        ctx().set_wand(0)
