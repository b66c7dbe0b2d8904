"""Every full-text path at the top of the doc-id domain: doc ids at and above 2^31, up to the last valid id 2^32 - 2, in
one segment of exactly 2^32 - 2 docs (tests/high_doc_reference.py). Sparse lists sit at the landmarks (2^31 +- 1, the
last windows' and zones' boundaries, the last partial window, 2^32 - 2) in every block encoding that reaches them. An
int32 column over every row (16 GB, generated in HBM) gives the filters, sort keys and facet keys; a short column whose
rows end at 2^20 makes every high doc NULL; the deleted-docs mask (a 512 MB bitmap) holds every landmark.

Top-k and the streaming scan are compared bit for bit with the oracle on the remapped small segment; count, facet counts
and the sorted scan with the NumPy references. Batch sizes 1, 64 and 1100 take the planner's chain count g from its
largest value to 1. The per-call doc limits are checked last."""
import ctypes as C

import numpy as np
import pytest

import count_reference as cr
import facet_reference as fr
import high_doc_reference as hd
import orc
import serenedb_b200 as sdb
import sort_reference as sr
from gpu_util import assert_hits_equal, ctx, oracle_terms, to_gpu
from serenedb_b200 import _native as N
from serenedb_b200._native import SdbgError

pytestmark = pytest.mark.gpu

KS = (1, 10, 1000, 8192)
FILT_LO, FILT_HI = 200000, 699999           # half of the full column's values
KEY_MIN, KEY_SPAN = 400000, 32768


@pytest.fixture(scope="module")
def top():
    c = hd.TopCorpus()
    g = to_gpu(c.oracle_segment())
    g.synth_column(hd.FULL_FIELD, hd.FULL_STREAM, hd.FULL_KIND, 0, hd.TOP)
    g.stage_column(hd.SHORT_FIELD, hd.short_column())
    reader = sdb.IndexReader([g], hd.TOP, hd.TOP, c.docs_with_term)
    # one more doc: a call over both segments holds 2^32 - 1 docs
    o1 = orc.Segment(1, has_wand=True)
    for _ in c.lists:
        o1.add_term(np.array([1], np.uint32), np.array([1], np.uint32))
    one = to_gpu(o1)
    one.stage_column(hd.FULL_FIELD, np.array([5], np.int32))
    S = dict(c=c, g=g, one=one, reader=reader, small={False: c.small_segment(), True: c.small_segment(with_mask=True)},
             cache={})
    yield S
    ctx().set_wand(0)
    g.close()
    one.close()


def _kind(kind):
    return sdb.AND if kind == "AND" else sdb.OR


def _all_hits(S, kind, tis, scorer, deleted=False, filt=False):
    """Every hit of a flat query, best first, at the high doc ids, from the oracle on the small segment."""
    key = (kind, tuple(tis), scorer.k, scorer.b, deleted, filt)
    if key not in S["cache"]:
        c = S["c"]
        n = len(c.U)
        of = orc.make_pred(hd.FULL_FIELD, "BETWEEN", FILT_LO, FILT_HI) if filt else None
        oh, total, _ = orc.bm25_topk([S["small"][deleted]], kind, oracle_terms(S["reader"], scorer, tis), n, k1=scorer.k,
                                     b=scorer.b, filt=of, mode=1)
        S["cache"][key] = (hd.map_hits(c, oh), total)
    return S["cache"][key]


def _queries(S, seed=7):
    """(kind, term ids): each shape alone, ANDed and ORed with its companion, and random 2..16-term queries."""
    c = S["c"]
    rng = np.random.default_rng(seed)
    q = [("OR", [t]) for t in c.shapes]
    q += [("AND", [t, t + 1]) for t in c.shapes if not c.lists[t][0].startswith("spread")]
    q += [("OR", [t, t + 1]) for t in c.shapes if not c.lists[t][0].startswith("spread")]
    q += [("AND", [c.names["spread_a"], c.names["spread_b"]]), ("OR", [c.names["spread_a"], c.names["spread_b"]])]
    n_terms = len(c.lists)
    for _ in range(12):
        nt = int(rng.integers(2, 17))
        tis = sorted(int(x) for x in rng.choice(n_terms, size=nt, replace=False))
        q.append(("OR", tis))
        q.append(("AND", [c.names["spread_a"], c.names["spread_b"]] + [t for t in tis[:3] if t not in
                                                                       (c.names["spread_a"], c.names["spread_b"])]))
    return q


def _batch(queries, nq):
    """nq queries cycling through `queries`."""
    return [queries[i % len(queries)] for i in range(nq)]


def _check_topk(hits, n_out, total, ref, k, exact_total):
    oh, ototal = ref
    assert_hits_equal(hits[:n_out], oh[:k])
    assert total == ototal if exact_total else total <= ototal


def _run_topk(S, queries, nq, k, scorer, wand, filt=False, deleted=False):
    pf = sdb.pred(hd.FULL_FIELD, "BETWEEN", FILT_LO, FILT_HI) if filt else None
    for kind in ("OR", "AND"):
        qs = [tis for kd, tis in queries if kd == kind]
        if not qs:
            continue
        batch = _batch(qs, nq)
        if nq == 1:
            res = []
            for tis in qs:
                h, n, t = sdb.ExecuteTopKBatch(S["reader"], [tis], _kind(kind), scorer, k, filt=pf)
                res.append((tis, h[0], n[0], t[0]))
        else:
            h, n, t = sdb.ExecuteTopKBatch(S["reader"], batch, _kind(kind), scorer, k, filt=pf)
            res = [(tis, h[i], n[i], t[i]) for i, tis in enumerate(batch)]
        for tis, h, n, t in res:
            ref = _all_hits(S, kind, tis, scorer, deleted, filt)
            _check_topk(h, int(n), int(t), ref, k, wand == 0 or kind == "AND")


@pytest.mark.parametrize("kernel", ["stream", "legacy"])
@pytest.mark.parametrize("wand", [0, 1, 2])
@pytest.mark.parametrize("nq", [1, 64, 1100])
def test_topk(top, nq, wand, kernel, monkeypatch):
    if kernel == "legacy":
        monkeypatch.setenv("SDBG_STREAM", "0")
    ctx().set_wand(wand)
    qs = _queries(top)
    for k in KS:
        if nq == 1100 and k == 8192 and wand == 1:
            continue      # 1100 x 8192 hits per call: levels 0 and 2 cover the largest k at this batch size
        _run_topk(top, qs, nq, k, sdb.BM25(), wand)


@pytest.mark.parametrize("scorer", [sdb.BM25(b=0.0), sdb.BM25(k=0.0), sdb.TFIDF(False), sdb.TFIDF(True)],
                         ids=["bm15", "bm1", "tfidf", "tfidf_norm"])
@pytest.mark.parametrize("nq", [1, 64])
def test_topk_other_scorers(top, nq, scorer):
    """BM15, BM1 and TFIDF run the legacy window kernel."""
    ctx().set_wand(0)
    for k in (10, 1000):
        _run_topk(top, _queries(top)[::2], nq, k, scorer, 0)


@pytest.mark.parametrize("mode", ["filter", "deleted", "both"])
def test_topk_filter_and_deleted_docs(top, mode):
    filt, deleted = mode != "deleted", mode != "filter"
    if deleted:
        top["g"].stage_docs_mask(top["c"].deleted)
    try:
        for wand in (0, 2):
            ctx().set_wand(wand)
            for nq in (1, 64):
                for k in (10, 1000):
                    _run_topk(top, _queries(top), nq, k, sdb.BM25(), wand, filt=filt, deleted=deleted)
    finally:
        top["g"].stage_docs_mask(None)


# ---------------------------------------------------------------- exclusions, groups, min-match
def _matches(S, kind, pos, excl=(), groups=None, mins=None, deleted=False, filt=False):
    """High doc ids the query matches: count_reference's set logic on the lists, then the column predicate evaluated at
    the matched rows only."""
    c = S["c"]
    lists = [d for _, d, _ in c.lists]
    dele = c.deleted if deleted else None
    if groups is None:
        docs = cr.match_docs(lists, kind, pos, excl, dele)
    else:
        docs = None
        for gi, grp in enumerate(groups):
            m = mins[gi] if mins is not None else 1
            every = np.concatenate([lists[t] for t in grp])
            u, cnt = np.unique(every, return_counts=True)
            ok = u[cnt >= m]
            docs = ok if docs is None else np.intersect1d(docs, ok)
        docs = cr.match_docs([docs] + [lists[t] for t in excl], "OR", [0], list(range(1, len(excl) + 1)), dele)
    if filt:
        v = hd.full_values(docs)
        docs = docs[(v >= FILT_LO) & (v <= FILT_HI)]
    return docs.astype(np.uint32)


def _restrict(ref, docs):
    """The oracle's hits of a wider query restricted to `docs`, order kept."""
    oh, _ = ref
    keep = oh[np.isin(oh["doc"], docs)]
    return keep, len(docs)


def _group_queries(S):
    c = S["c"]
    a, b = c.names["spread_a"], c.names["spread_b"]
    L, T = c.names["landmarks"], c.names["bitset_top"]
    return [([[a], [b, L]], None), ([[a, b, L]], [2]), ([[a, b, L, T, T + 1]], [2]), ([[a, L], [b, T, T + 1]], [1, 1]),
            ([[L, a], [b, T]], [2, 1]), ([[a, b, L, c.names["dsvb_high"], c.names["raw_block"]]], [3])]


@pytest.mark.parametrize("wand", [0, 2])
@pytest.mark.parametrize("nq", [1, 64])
def test_exclusions_groups_min_match(top, nq, wand):
    ctx().set_wand(wand)
    c = top["c"]
    scorer = sdb.BM25()
    a, b, L = c.names["spread_a"], c.names["spread_b"], c.names["landmarks"]
    excl_q = [("OR", [a], [L]), ("OR", [a, b], [L, c.names["bitset_top"]]), ("AND", [a, b], [L]),
              ("OR", [L, c.names["single_top"]], [c.names["same32_pair"]]), ("OR", [a, b, L], [c.names["raw_tail_high"]])]
    for k in (10, 1000, 8192):
        for kind in ("OR", "AND"):
            qs = [(p, x) for kd, p, x in excl_q if kd == kind]
            batch = _batch(qs, nq) if nq > 1 else qs
            h, n, t = sdb.ExecuteTopKBatch(top["reader"], [p for p, _ in batch], _kind(kind), scorer, k,
                                           exclude=[x for _, x in batch])
            for i, (p, x) in enumerate(batch):
                ref = _restrict(_all_hits(top, kind, p, scorer), _matches(top, kind, p, excl=x))
                _check_topk(h[i], int(n[i]), int(t[i]), ref, k, wand == 0 or kind == "AND")
        gq = _group_queries(top)
        batch = _batch(gq, nq) if nq > 1 else gq
        h, n, t = sdb.ExecuteTopKGroupsBatch(top["reader"], [g for g, _ in batch], scorer, k,
                                             min_match=[m if m is not None else [1] * len(g) for g, m in batch],
                                             exclude=[[c.names["raw_tail_high"]] if i % 2 else None for i in range(len(batch))])
        for i, (grp, m) in enumerate(batch):
            x = [c.names["raw_tail_high"]] if i % 2 else []
            flat = sorted({t for gg in grp for t in gg})
            ref = _restrict(_all_hits(top, "OR", flat, scorer), _matches(top, "OR", flat, excl=x, groups=grp, mins=m))
            _check_topk(h[i], int(n[i]), int(t[i]), ref, k, wand == 0)


# ---------------------------------------------------------------- count, facets, sorted scan
def _count_queries(S):
    c = S["c"]
    return [("OR", [t]) for t in c.shapes] + [("AND", [t, t + 1]) for t in c.shapes if not c.lists[t][0].startswith("spread")] + \
        [("OR", [c.names["spread_a"], c.names["spread_b"], c.names["landmarks"]]),
         ("AND", [c.names["spread_a"], c.names["spread_b"]]), ("AND", [c.names["spread_a"], c.names["landmarks"]])]


@pytest.mark.parametrize("mode", ["plain", "filter", "deleted", "both"])
def test_count(top, mode):
    filt, deleted = mode in ("filter", "both"), mode in ("deleted", "both")
    pf = sdb.pred(hd.FULL_FIELD, "BETWEEN", FILT_LO, FILT_HI) if filt else None
    if deleted:
        top["g"].stage_docs_mask(top["c"].deleted)
    try:
        for kind in ("OR", "AND"):
            qs = [p for kd, p in _count_queries(top) if kd == kind]
            for nq in (1, 64):
                batch = _batch(qs, nq) if nq > 1 else qs
                got = sdb.ExecuteCountBatch(top["reader"], batch, _kind(kind), filt=pf)
                for i, p in enumerate(batch):
                    assert got[i] == len(_matches(top, kind, p, deleted=deleted, filt=filt)), (kind, p)
        gq = _group_queries(top)
        got = sdb.ExecuteCountGroupsBatch(top["reader"], [g for g, _ in gq], filt=pf,
                                          min_match=[m if m is not None else [1] * len(g) for g, m in gq])
        for i, (grp, m) in enumerate(gq):
            flat = sorted({t for gg in grp for t in gg})
            assert got[i] == len(_matches(top, "OR", flat, groups=grp, mins=m, deleted=deleted, filt=filt)), grp
    finally:
        top["g"].stage_docs_mask(None)


def _facet_ref(S, docs, field, key_min, key_span):
    c = S["c"]
    return fr.facet_counts([[c.small(docs)]], "OR", [0], [c.small_columns(field)], key_min, key_span)


@pytest.mark.parametrize("deleted", [False, True], ids=["all", "deleted"])
def test_facet_counts(top, deleted):
    """Keys of the full-length column under a BETWEEN filter on the same column (every passing key has a bin), and the
    short column's keys, NULL for every doc past its rows."""
    pf = sdb.pred(hd.FULL_FIELD, "BETWEEN", KEY_MIN, KEY_MIN + KEY_SPAN - 1)
    if deleted:
        top["g"].stage_docs_mask(top["c"].deleted)
    try:
        for kind in ("OR", "AND"):
            qs = [p for kd, p in _count_queries(top) if kd == kind]
            r = sdb.ExecuteFacetCountsBatch(top["reader"], qs, _kind(kind), hd.FULL_FIELD, KEY_MIN, KEY_SPAN, filt=pf)
            rs = sdb.ExecuteFacetCountsBatch(top["reader"], qs, _kind(kind), hd.SHORT_FIELD, 0, 5000)
            for i, p in enumerate(qs):
                docs = _matches(top, kind, p, deleted=deleted)
                v = hd.full_values(docs)
                fd = docs[(v >= KEY_MIN) & (v < KEY_MIN + KEY_SPAN)]
                counts, nulls = _facet_ref(top, fd, hd.FULL_FIELD, KEY_MIN, KEY_SPAN)
                assert np.array_equal(r["counts"][i], counts) and r["nulls"][i] == nulls == 0, p
                counts, nulls = _facet_ref(top, docs, hd.SHORT_FIELD, 0, 5000)
                assert np.array_equal(rs["counts"][i], counts) and rs["nulls"][i] == nulls, p
        gq = _group_queries(top)
        mins = [m if m is not None else [1] * len(g) for g, m in gq]
        r = sdb.ExecuteFacetCountsGroupsBatch(top["reader"], [g for g, _ in gq], hd.SHORT_FIELD, 0, 5000, min_match=mins)
        for i, (grp, m) in enumerate(gq):
            flat = sorted({t for gg in grp for t in gg})
            counts, nulls = _facet_ref(top, _matches(top, "OR", flat, groups=grp, mins=m, deleted=deleted), hd.SHORT_FIELD, 0, 5000)
            assert np.array_equal(r["counts"][i], counts) and r["nulls"][i] == nulls, grp
    finally:
        top["g"].stage_docs_mask(None)


def _check_sorted(S, got, docs, field, desc, nulls_first, k):
    c = S["c"]
    ref = sr.sorted_hits([[c.small(docs)]], "OR", [0], [c.small_columns(field)], desc, nulls_first, k)
    assert np.array_equal(got["docs"], c.big(ref["docs"]))
    assert np.array_equal(got["nulls"], ref["nulls"])
    assert np.array_equal(got["values"][~ref["nulls"]], ref["values"][~ref["nulls"]])


@pytest.mark.parametrize("wand", [0, 2])
@pytest.mark.parametrize("field", [hd.FULL_FIELD, hd.SHORT_FIELD], ids=["full", "short"])
def test_sorted_scan(top, field, wand):
    """ORDER BY a column LIMIT k over exactly 2^32 - 2 docs, both directions and NULL placements; deleted docs and a
    filter on the second half. The full column is NOT NULL, so level 2 prunes windows by its zonemap."""
    ctx().set_wand(wand)
    pf = sdb.pred(hd.FULL_FIELD, "BETWEEN", FILT_LO, FILT_HI)
    for deleted in (False, True):
        if deleted:
            top["g"].stage_docs_mask(top["c"].deleted)
        try:
            for k in (1, 100, 4096):
                for desc in (False, True):
                    for nf in (False, True):
                        for kind in ("OR", "AND"):
                            qs = [p for kd, p in _count_queries(top) if kd == kind]
                            for filt in (False, True):
                                r = sdb.ExecuteTopKByColumnBatch(top["reader"], qs, _kind(kind), field, k, desc, nf,
                                                                 filt=pf if filt else None)
                                for i, p in enumerate(qs):
                                    got = {key: r[key][i] for key in ("docs", "values", "nulls")}
                                    _check_sorted(top, got, _matches(top, kind, p, deleted=deleted, filt=filt), field, desc, nf, k)
                        gq = _group_queries(top)
                        mins = [m if m is not None else [1] * len(g) for g, m in gq]
                        r = sdb.ExecuteTopKByColumnGroupsBatch(top["reader"], [g for g, _ in gq], field, k, desc, nf,
                                                               min_match=mins)
                        for i, (grp, m) in enumerate(gq):
                            flat = sorted({t for gg in grp for t in gg})
                            got = {key: r[key][i] for key in ("docs", "values", "nulls")}
                            _check_sorted(top, got, _matches(top, "OR", flat, groups=grp, mins=m, deleted=deleted), field,
                                          desc, nf, k)
        finally:
            top["g"].stage_docs_mask(None)
    if field == hd.SHORT_FIELD and wand == 2:
        # NULLS LAST with ~1000 non-NULL matches: once k of them are in, every window past the column's rows (up to
        # 2^32 - 2) holds only NULL keys and is skipped by the zonemap, without being decoded
        a = top["c"].names["spread_a"]
        got = sdb.ExecuteTopKByColumn(top["reader"], [a], sdb.OR, field, 100)
        judged, skipped = ctx().scan_stats()
        assert 0 < skipped < judged
        _check_sorted(top, got, _matches(top, "OR", [a]), field, False, False, 100)


# ---------------------------------------------------------------- streaming scan
def _ranges():
    out = [(1, None), (1, hd.EOF), (hd.TOP, hd.EOF), (1, hd.TOP), (2 ** 31, 2 ** 31 + 1)]
    for x in hd.LANDMARKS:
        out += [(x, hd.EOF), (1, x), (x - 1, x + 1)]
    return out


def test_stream_scored_docs(top):
    """Every match with its score, ascending by doc, over the whole segment (doc_max = 2^32 - 1, what EmitScoredDocs asks
    for) and over ranges that start or end at each landmark."""
    c = top["c"]
    scorer = sdb.BM25()
    a, b, L = c.names["spread_a"], c.names["spread_b"], c.names["landmarks"]
    qs = [("OR", [L], None), ("OR", [a, b], None), ("OR", [a, b, L, c.names["bitset_top"]], None), ("AND", [a, b], None),
          ("AND", [a, L], None), ("OR", [c.names["single_top"], c.names["same32_top"]], None),
          ("OR", [a, L], [b]), ("AND", [a, b], [L]), ("OR", [c.names["dsvb_high"], c.names["raw_block"]], [L])]
    for kind, p, x in qs:
        oh, _ = _all_hits(top, kind, p, scorer)
        if x:
            oh, _ = _restrict((oh, 0), _matches(top, kind, p, excl=x))
        oh = oh[np.argsort(oh["doc"], kind="stable")]
        for lo, hi in _ranges():
            docs, scores = sdb.StreamScoredDocs(top["reader"], 0, p, _kind(kind), scorer, doc_min=lo, doc_max=hi, exclude=x)
            end = hd.EOF if hi is None else hi
            want = oh[(oh["doc"] >= lo) & (oh["doc"] < end)]
            assert np.array_equal(docs, want["doc"]), (kind, p, x, lo, hi)
            assert np.array_equal(scores.view(np.uint32), want["score"].view(np.uint32)), (kind, p, x, lo, hi)


# ---------------------------------------------------------------- limits
def test_doc_count_limits(top):
    """Top-k and sorted calls take exactly 2^32 - 2 docs (the tests above); 2^32 - 1 is refused before anything is
    queued. Count and facet counts take any set of valid segments. A segment of 2^32 - 1 docs cannot be created."""
    c = top["c"]
    L = c.names["landmarks"]
    r2 = sdb.IndexReader([top["g"], top["one"]], hd.TOP + 1, hd.TOP + 1, [n + 1 for n in c.docs_with_term])
    before = ctx().launches
    with pytest.raises(SdbgError, match="EUNSUPPORTED"):
        sdb.ExecuteTopKBatch(r2, [[L]], sdb.OR, sdb.BM25(), 10)
    with pytest.raises(SdbgError, match="EUNSUPPORTED"):
        sdb.ExecuteTopKGroupsBatch(r2, [[[L]]], sdb.BM25(), 10)
    with pytest.raises(SdbgError, match="EUNSUPPORTED"):
        sdb.ExecuteTopKByColumnBatch(r2, [[L]], sdb.OR, hd.FULL_FIELD, 10)
    with pytest.raises(SdbgError, match="EUNSUPPORTED"):
        sdb.ExecuteTopKByColumnGroupsBatch(r2, [[[L]]], hd.FULL_FIELD, 10)
    assert ctx().launches == before
    n_l = len(c.lists[L][1])
    assert sdb.ExecuteCountBatch(r2, [[L]], sdb.OR)[0] == n_l + 1
    assert sdb.ExecuteCountGroupsBatch(r2, [[[L]]])[0] == n_l + 1
    f = sdb.ExecuteFacetCountsBatch(r2, [[L]], sdb.OR, hd.FULL_FIELD, 0, 16,
                                    filt=sdb.pred(hd.FULL_FIELD, "BETWEEN", 0, 15))
    v = hd.full_values(c.lists[L][1])
    want = np.bincount(v[v < 16], minlength=16).astype(np.uint64)
    want[5] += 1                                              # the one-doc segment's key
    assert np.array_equal(f["counts"][0], want)
    h = C.c_void_p()
    assert N.ERR[N.lib().sdbg_segment_create(ctx()._h, hd.EOF, C.byref(h))] == "EINVAL" and not h.value
    assert N.lib().sdbg_segment_create(ctx()._h, hd.TOP, C.byref(h)) == 0
    N.lib().sdbg_segment_destroy(h)
    with pytest.raises(ValueError):
        sdb.Segment(ctx(), 2 ** 32 + 5)
