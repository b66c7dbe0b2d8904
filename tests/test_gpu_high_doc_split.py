"""The full-text paths over two segments whose doc counts sum to exactly 2^32 - 2 (high_doc_reference.SplitCorpus): A holds
2^31 + 2^20 docs with a 1-byte norm column (2 GB, norm rows past 2^31), B the rest, so B's keys carry ordinal_base =
2^31 + 2^20 and reach ordinal 2^32 - 2. Landmarks sit at 2^31 +- 1 and at the ends of both segments. The int32 column runs
over every row of both segments (B's rows continue A's).

Top-k, exclusions, OR groups and min-match are compared bit for bit with the oracle on the two remapped small segments
(norms of the mapped docs included; ties by (segment, doc) are kept by the remap); count and the sorted scan with the
NumPy references."""
import numpy as np
import pytest

import count_reference as cr
import high_doc_reference as hd
import orc
import serenedb_b200 as sdb
import sort_reference as sr
from gpu_util import assert_hits_equal, ctx, metas_of, oracle_terms, to_gpu

pytestmark = pytest.mark.gpu

KS = (1, 10, 1000, 8192)
FILT_LO, FILT_HI = 200000, 699999


@pytest.fixture(scope="module")
def split():
    s = hd.SplitCorpus()
    a, b = s.segs
    oa = a.oracle_segment()                  # no block-max data: the writer needs no norms
    ga = sdb.Segment(ctx(), a.n_docs)
    ga.stage_postings(oa.doc_bytes(), metas_of(oa), has_wand=False)
    ga.stage_norms(hd.split_norm_bytes(), 1)
    del oa
    gb = to_gpu(b.oracle_segment())
    ga.synth_column(hd.FULL_FIELD, hd.FULL_STREAM, hd.FULL_KIND, 0, a.n_docs)
    gb.synth_column(hd.FULL_FIELD, hd.FULL_STREAM, hd.FULL_KIND, a.n_docs, b.n_docs)
    reader = sdb.IndexReader([ga, gb], hd.TOP, s.total_term_freq, s.docs_with_term)
    S = dict(s=s, g=[ga, gb], reader=reader, cache={},
             small={d: [c.small_segment(with_mask=d) for c in s.segs] for d in (False, True)})
    yield S
    ctx().set_wand(0)
    ga.close()
    gb.close()


def _kind(kind):
    return sdb.AND if kind == "AND" else sdb.OR


def _mask(S, on):
    for g, c in zip(S["g"], S["s"].segs):
        g.stage_docs_mask(c.deleted if on else None)


def _all_hits(S, kind, tis, scorer, deleted=False, filt=False):
    """Every hit of a flat query over both segments, best first, at the high doc ids (oracle on the small segments)."""
    key = (kind, tuple(tis), scorer.k, scorer.b, deleted, filt)
    if key not in S["cache"]:
        segs = S["s"].segs
        of = orc.make_pred(hd.FULL_FIELD, "BETWEEN", FILT_LO, FILT_HI) if filt else None
        oh, total, _ = orc.bm25_topk(S["small"][deleted], kind, oracle_terms(S["reader"], scorer, tis),
                                     sum(len(c.U) for c in segs), k1=scorer.k, b=scorer.b, filt=of, mode=1)
        S["cache"][key] = (hd.map_hits(segs, oh), total)
    return S["cache"][key]


def _matches(S, kind, pos, excl=(), groups=None, mins=None, deleted=False, filt=False):
    """Per segment, the high doc ids the query matches (count_reference's set logic; the predicate at matched rows)."""
    out = []
    for c in S["s"].segs:
        lists = [d for _, d, _ in c.lists]
        dele = c.deleted if deleted else None
        if groups is None:
            docs = cr.match_docs(lists, kind, pos, excl, dele)
        else:
            docs = None
            for gi, grp in enumerate(groups):
                u, cnt = np.unique(np.concatenate([lists[t] for t in grp]), return_counts=True)
                ok = u[cnt >= (mins[gi] if mins is not None else 1)]
                docs = ok if docs is None else np.intersect1d(docs, ok)
            docs = cr.match_docs([docs] + [lists[t] for t in excl], "OR", [0], list(range(1, len(excl) + 1)), dele)
        if filt:
            v = c.values(docs)
            docs = docs[(v >= FILT_LO) & (v <= FILT_HI)]
        out.append(docs.astype(np.uint32))
    return out


def _restrict(ref, per_seg):
    """The oracle's hits of a wider query restricted to the matched (segment, doc) pairs, order kept."""
    oh, _ = ref
    keep = np.zeros(len(oh), bool)
    for si, docs in enumerate(per_seg):
        keep |= (oh["seg"] == si) & np.isin(oh["doc"], docs)
    return oh[keep], sum(len(d) for d in per_seg)


def _check_topk(h, n, t, ref, k, exact_total):
    oh, ototal = ref
    assert_hits_equal(h[:int(n)], oh[:k])
    assert int(t) == ototal if exact_total else int(t) <= ototal


def _queries(S, seed=9):
    nm = S["s"].names
    rng = np.random.default_rng(seed)
    sh = S["s"].shapes
    a, b = nm["spread_a"], nm["spread_b"]
    q = [("OR", [t]) for t in sh] + [("AND", [t, t + 1]) for t in sh if t not in (a, b)]
    q += [("OR", [t, t + 1]) for t in sh if t not in (a, b)] + [("AND", [a, b]), ("OR", [a, b])]
    n_terms = len(S["s"].segs[0].lists)
    for _ in range(8):
        tis = sorted(int(x) for x in rng.choice(n_terms, size=int(rng.integers(2, n_terms + 1)), replace=False))
        q.append(("OR", tis))
        q.append(("AND", [a, b] + [t for t in tis[:2] if t not in (a, b)]))
    return q


def _run_topk(S, nq, k, scorer, wand, filt=False, deleted=False):
    pf = sdb.pred(hd.FULL_FIELD, "BETWEEN", FILT_LO, FILT_HI) if filt else None
    for kind in ("OR", "AND"):
        qs = [tis for kd, tis in _queries(S) if kd == kind]
        if nq == 1:
            res = []
            for tis in qs:
                h, n, t = sdb.ExecuteTopKBatch(S["reader"], [tis], _kind(kind), scorer, k, filt=pf)
                res.append((tis, h[0], n[0], t[0]))
        else:
            batch = [qs[i % len(qs)] for i in range(nq)]
            h, n, t = sdb.ExecuteTopKBatch(S["reader"], batch, _kind(kind), scorer, k, filt=pf)
            res = [(tis, h[i], n[i], t[i]) for i, tis in enumerate(batch)]
        for tis, h, n, t in res:
            _check_topk(h, n, t, _all_hits(S, kind, tis, scorer, deleted, filt), k, wand == 0 or kind == "AND")


@pytest.mark.parametrize("kernel", ["stream", "legacy"])
@pytest.mark.parametrize("wand", [0, 1, 2])
@pytest.mark.parametrize("nq", [1, 64, 1100])
def test_topk(split, nq, wand, kernel, monkeypatch):
    if kernel == "legacy":
        monkeypatch.setenv("SDBG_STREAM", "0")
    ctx().set_wand(wand)
    for k in KS:
        if nq == 1100 and k == 8192 and wand == 1:
            continue
        _run_topk(split, nq, k, sdb.BM25(), wand)


@pytest.mark.parametrize("scorer", [sdb.BM25(b=0.0), sdb.TFIDF(True)], ids=["bm15", "tfidf_norm"])
def test_topk_other_scorers(split, scorer):
    """Scorers that read the norms differently (BM15 ignores them, normalised TFIDF divides by their root)."""
    ctx().set_wand(0)
    for nq in (1, 64):
        _run_topk(split, nq, 1000, scorer, 0)


@pytest.mark.parametrize("mode", ["filter", "deleted", "both"])
def test_topk_filter_and_deleted_docs(split, mode):
    filt, deleted = mode != "deleted", mode != "filter"
    _mask(split, deleted)
    try:
        for wand in (0, 2):
            ctx().set_wand(wand)
            for nq in (1, 64):
                for k in (10, 1000):
                    _run_topk(split, nq, k, sdb.BM25(), wand, filt=filt, deleted=deleted)
    finally:
        _mask(split, False)


def _group_queries(S):
    nm = S["s"].names
    a, b, L, D = nm["spread_a"], nm["spread_b"], nm["landmarks"], nm["dense_top"]
    return [([[a], [b, L]], None), ([[a, b, L]], [2]), ([[a, b, L, D, D + 1]], [2]), ([[a, L], [b, D, D + 1]], [1, 1]),
            ([[L, a], [b, D]], [2, 1]), ([[a, b, L, nm["tail_top"], nm["single_top"]]], [3])]


@pytest.mark.parametrize("wand", [0, 2])
@pytest.mark.parametrize("nq", [1, 64])
def test_exclusions_groups_min_match(split, nq, wand):
    ctx().set_wand(wand)
    nm = split["s"].names
    scorer = sdb.BM25()
    a, b, L = nm["spread_a"], nm["spread_b"], nm["landmarks"]
    excl_q = [("OR", [a], [L]), ("OR", [a, b], [L, nm["dense_top"]]), ("AND", [a, b], [L]),
              ("OR", [L, nm["single_top"]], [nm["tail_top"]]), ("OR", [a, b, L], [nm["single_top"]])]
    for k in (10, 1000, 8192):
        for kind in ("OR", "AND"):
            qs = [(p, x) for kd, p, x in excl_q if kd == kind]
            batch = [qs[i % len(qs)] for i in range(nq)] if nq > 1 else qs
            h, n, t = sdb.ExecuteTopKBatch(split["reader"], [p for p, _ in batch], _kind(kind), scorer, k,
                                           exclude=[x for _, x in batch])
            for i, (p, x) in enumerate(batch):
                ref = _restrict(_all_hits(split, kind, p, scorer), _matches(split, kind, p, excl=x))
                _check_topk(h[i], n[i], t[i], ref, k, wand == 0 or kind == "AND")
        gq = _group_queries(split)
        batch = [gq[i % len(gq)] for i in range(nq)] if nq > 1 else gq
        xs = [[nm["tail_top"]] if i % 2 else [] for i in range(len(batch))]
        h, n, t = sdb.ExecuteTopKGroupsBatch(split["reader"], [g for g, _ in batch], scorer, k,
                                             min_match=[m if m is not None else [1] * len(g) for g, m in batch],
                                             exclude=[x or None for x in xs])
        for i, (grp, m) in enumerate(batch):
            flat = sorted({t_ for gg in grp for t_ in gg})
            ref = _restrict(_all_hits(split, "OR", flat, scorer), _matches(split, "OR", flat, excl=xs[i], groups=grp, mins=m))
            _check_topk(h[i], n[i], t[i], ref, k, wand == 0)


@pytest.mark.parametrize("deleted", [False, True], ids=["all", "deleted"])
def test_count(split, deleted):
    pf = sdb.pred(hd.FULL_FIELD, "BETWEEN", FILT_LO, FILT_HI)
    _mask(split, deleted)
    try:
        for filt in (False, True):
            for kind in ("OR", "AND"):
                qs = [p for kd, p in _queries(split) if kd == kind]
                got = sdb.ExecuteCountBatch(split["reader"], qs, _kind(kind), filt=pf if filt else None)
                for i, p in enumerate(qs):
                    assert got[i] == sum(len(d) for d in _matches(split, kind, p, deleted=deleted, filt=filt)), (kind, p)
    finally:
        _mask(split, False)


def _check_sorted(S, got, per_seg, desc, k):
    segs = S["s"].segs
    ref = sr.sorted_hits([[c.small(d)] for c, d in zip(segs, per_seg)], "OR", [0],
                         [c.small_columns(hd.FULL_FIELD) for c in segs], desc, False, k)
    docs = np.array([segs[s].big([d])[0] for s, d in zip(ref["segs"], ref["docs"])], np.uint32)
    assert np.array_equal(got["segs"], ref["segs"]) and np.array_equal(got["docs"], docs)
    assert np.array_equal(got["values"], ref["values"]) and not got["nulls"].any()


@pytest.mark.parametrize("wand", [0, 2])
def test_sorted_scan(split, wand):
    """ORDER BY the full column LIMIT k over 2^32 - 2 docs in two segments: the keys' ordinals reach 2^32 - 3 and the
    segment of an ordinal past 2^31 is found again when the keys are turned into hits."""
    ctx().set_wand(wand)
    pf = sdb.pred(hd.FULL_FIELD, "BETWEEN", FILT_LO, FILT_HI)
    for deleted in (False, True):
        _mask(split, deleted)
        try:
            for k in (1, 100, 4096):
                for desc in (False, True):
                    for kind in ("OR", "AND"):
                        qs = [p for kd, p in _queries(split) if kd == kind]
                        for filt in (False, True):
                            r = sdb.ExecuteTopKByColumnBatch(split["reader"], qs, _kind(kind), hd.FULL_FIELD, k, desc,
                                                             filt=pf if filt else None)
                            for i, p in enumerate(qs):
                                got = {key: r[key][i] for key in ("docs", "segs", "values", "nulls")}
                                _check_sorted(split, got, _matches(split, kind, p, deleted=deleted, filt=filt), desc, k)
                    gq = _group_queries(split)
                    mins = [m if m is not None else [1] * len(g) for g, m in gq]
                    r = sdb.ExecuteTopKByColumnGroupsBatch(split["reader"], [g for g, _ in gq], hd.FULL_FIELD, k, desc,
                                                           min_match=mins)
                    for i, (grp, m) in enumerate(gq):
                        flat = sorted({t for gg in grp for t in gg})
                        got = {key: r[key][i] for key in ("docs", "segs", "values", "nulls")}
                        _check_sorted(split, got, _matches(split, "OR", flat, groups=grp, mins=m, deleted=deleted), desc, k)
        finally:
            _mask(split, False)
