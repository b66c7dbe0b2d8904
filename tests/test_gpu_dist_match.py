"""The count, facet-count, aggregate and sorted-scan passes across GPUs (sdbg_dist_match_*_batch_groups_min, DESIGN §5),
with R ranks simulated on one GPU: each rank is its own list of segments. The references are the local entries over the unsharded
corpus, which the single-GPU suites check against their Python statements of the semantics.

Sorted scan: TopKByColumnDevice writes rank r's rows into slice r and merge_topk_by_column_gathered selects the k best;
the hits must equal the unsharded sorted scan's bit for bit once (rank, ordinal within the rank) is mapped back to
(segment, doc). Count and facet counts: without sdbg_dist_init the all-reduce is a no-op, so each rank's dist call gives
that rank's local result, and the ranks' results must add up to the unsharded result. Aggregates: MatchAggregatesDevice writes rank
r's buffer into slice r of one torch buffer and merge_aggregates_gathered merges all R, as the dist entry does after its
all-gather; integer results are exact, float64 sums bit for bit the ranks' partials added in rank order. A one-rank NCCL
communicator runs the collectives themselves."""
import ctypes as C

import numpy as np
import pytest

import count_reference as cr
import serenedb_b200 as sdb
from gpu_util import ctx, metas_of
from serenedb_b200 import _native as N
from serenedb_b200._native import SdbgError
from shape_corpora import Corpus, natural_segments, uniform_segments

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
KEY64, KEY32, VAL64, VALF, VAL32, FILT = 1, 2, 3, 4, 5, 9
C_VP = C.c_void_p


def _columns(rng, n, all_null_key=False, fail_filter=False):
    f = rng.normal(size=n) * 1e3
    for v, m in ((np.nan, 5), (np.inf, 5), (-np.inf, 5), (-0.0, 40), (0.0, 40), (5e-324, 10), (-2.5e-310, 10)):
        f[rng.integers(0, n, m)] = v
    v64 = rng.integers(-1000, 1000, n).astype(np.int64)
    v64[rng.integers(0, n, n // 20)] = I64_MAX
    v64[rng.integers(0, n, n // 20)] = I64_MIN
    return {KEY64: (rng.integers(-5, 11, n).astype(np.int64), None),                            # bit-packed
            KEY32: (rng.integers(0, 16, n).astype(np.int32), np.zeros(n, bool) if all_null_key else rng.random(n) < 0.8),
            VAL64: (v64, rng.random(n) < 0.9),                                                 # raw, nullable, extremes
            VALF: (f, rng.random(n) < 0.95),
            VAL32: (rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int32), None),
            FILT: (np.full(n, 1000, np.int64) if fail_filter else rng.integers(0, 100, n).astype(np.int64), None)}


def _stage(c, oseg, cols):
    g = sdb.Segment(c, oseg.n_docs)
    if oseg.num_terms():
        g.stage_postings(oseg.doc_bytes(), metas_of(oseg))
    if oseg.has_norms:
        g.stage_norms(*oseg.norm_bytes())
    for field, (vals, valid) in cols.items():
        g.stage_column(field, vals, cr.validity_words(valid) if valid is not None else None)
    return g


def _env(c, corpus, ranks, cols):
    gsegs = [_stage(c, o, cl) for o, cl in zip(corpus.osegs, cols)]
    reader = lambda segs: sdb.IndexReader(segs, corpus.docs_with_field, corpus.total_term_freq, corpus.docs_with_term)
    gbase = np.cumsum([0] + [o.n_docs for o in corpus.osegs])[:-1]
    return dict(readers=[reader([gsegs[j] for j in rk]) for rk in ranks], one=reader(gsegs), gsegs=gsegs,
                n_terms=corpus.n_terms, ranks=ranks, gbase=gbase)


@pytest.fixture(scope="module")
def uniform8():
    """8 ranks of one segment each, cut by doc range from one corpus."""
    _, parts, _ = uniform_segments(parts=8)
    corpus = Corpus(parts)
    rng = np.random.default_rng(1)
    return _env(ctx(), corpus, [[j] for j in range(8)], [_columns(rng, o.n_docs) for o in corpus.osegs])


@pytest.fixture(scope="module")
def natural3():
    """rank 0: segments 0 + 1; rank 1: segment 2, every KEY32 NULL and deleted docs; rank 2: a segment where the queried
    terms have no postings and every doc fails the filter."""
    segs = natural_segments()
    rng = np.random.default_rng(3)
    n = 2000
    empty = [(np.zeros(0, np.uint32), np.zeros(0, np.uint32))] * 10
    extra = np.sort(rng.choice(np.arange(1, n + 1), 50, replace=False)).astype(np.uint32)
    segs.append((rng.integers(5, 50, n).astype(np.uint32), empty + [(extra, np.ones(50, np.uint32))]))
    corpus = Corpus(segs)
    cols = [_columns(rng, o.n_docs, all_null_key=(i == 2), fail_filter=(i == 3)) for i, o in enumerate(corpus.osegs)]
    env = _env(ctx(), corpus, [[0, 1], [2], [3]], cols)
    env["gsegs"][2].stage_docs_mask(np.unique(rng.integers(1, corpus.osegs[2].n_docs + 1, 5000)).astype(np.uint32))
    return env


@pytest.fixture(params=[0, 1, 2], ids=lambda v: f"wand{v}")
def level(request):
    ctx().set_wand(request.param)
    yield request.param
    ctx().set_wand(0)


def _batch(n_terms, seed):
    """(queries, exclude, min_match): flat ORs (one group), flat ANDs (single-term groups), true groups, min-match groups,
    with exclusions on some: one batch of every shape."""
    rng = np.random.default_rng(seed)
    pick = lambda k: [int(t) for t in rng.choice(n_terms, size=k, replace=False)]
    qs, xs, ms = [], [], []
    for i in range(24):
        t = pick(4)
        shape = i % 4
        if shape == 0:
            q, m = [t[:3]], [1]
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


def _shapes(n_terms, seed):
    """The mixed batch, then each shape alone (one shape writes straight into the outputs, several are scattered)."""
    qs, xs, ms = _batch(n_terms, seed)
    yield qs, xs, ms
    for s in range(4):
        yield qs[s::4], xs[s::4], ms[s::4]


FILTERS = (None, sdb.pred(FILT, "BETWEEN", 20, 59))


@pytest.mark.parametrize("corpus_name", ["uniform8", "natural3"])
def test_counts_add_up_to_unsharded(request, corpus_name, level):
    env = request.getfixturevalue(corpus_name)
    for qs, xs, ms in _shapes(env["n_terms"], 7):
        for filt in FILTERS:
            total = np.zeros(len(qs), np.uint64)
            for reader in env["readers"]:
                got = sdb.ExecuteDistCountGroupsBatch(reader, qs, filt=filt, exclude=xs, min_match=ms)
                assert np.array_equal(got, sdb.ExecuteCountGroupsBatch(reader, qs, filt=filt, exclude=xs, min_match=ms))
                total += got
            assert np.array_equal(total, sdb.ExecuteCountGroupsBatch(env["one"], qs, filt=filt, exclude=xs, min_match=ms))


@pytest.mark.parametrize("key,key_min,span", [(KEY64, -5, 16), (KEY32, 0, 16), (KEY64, -1000, 2001), (KEY32, -2048, 4096)])
@pytest.mark.parametrize("corpus_name", ["uniform8", "natural3"])
def test_facets_add_up_to_unsharded(request, corpus_name, key, key_min, span, level):
    env = request.getfixturevalue(corpus_name)
    for qs, xs, ms in _shapes(env["n_terms"], 11):
        for filt in FILTERS:
            counts, nulls = np.zeros((len(qs), span), np.uint64), np.zeros(len(qs), np.uint64)
            for reader in env["readers"]:
                got = sdb.ExecuteDistFacetCountsGroupsBatch(reader, qs, key, key_min, span, filt=filt, exclude=xs, min_match=ms)
                want = sdb.ExecuteFacetCountsGroupsBatch(reader, qs, key, key_min, span, filt=filt, exclude=xs, min_match=ms)
                assert np.array_equal(got["counts"], want["counts"]) and np.array_equal(got["nulls"], want["nulls"])
                counts += got["counts"]
                nulls += got["nulls"]
            want = sdb.ExecuteFacetCountsGroupsBatch(env["one"], qs, key, key_min, span, filt=filt, exclude=xs, min_match=ms)
            assert np.array_equal(counts, want["counts"]) and np.array_equal(nulls, want["nulls"])


def _cuda_zeros(n_words, rows=1):
    import torch
    t = torch.zeros((rows, n_words), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()      # the library works on its own non-blocking stream
    return t


def _gather(readers, qs, value, key, key_min, span, **kw):
    """Every rank's device buffer in one [R, words] buffer, as the all-gather leaves it."""
    words = sdb.match_aggregate_device_bytes(len(qs), span) // 8
    buf = _cuda_zeros(words, len(readers))
    for r, reader in enumerate(readers):
        sdb.MatchAggregatesDevice(reader, qs, value, buf[r].data_ptr(), key, key_min, span, **kw)
    return buf


def _merge(buf, nq, vt, key_min, span):
    return sdb.merge_aggregates_gathered(ctx(), buf.data_ptr(), buf.shape[0], nq, vt, key_min, span)


def _assert_agg_equal(got, want, vt, exact_float=True):
    for part in (lambda r: r, lambda r: r["null"]):
        g, w = part(got), part(want)
        for f in ("count", "count_value", "min", "max"):
            a, b = np.asarray(g[f]), np.asarray(w[f])
            assert np.array_equal(a.view(np.uint64) if vt == 1 and f in ("min", "max") else a,
                                  b.view(np.uint64) if vt == 1 and f in ("min", "max") else b), f
        if vt != 1:
            assert np.array_equal(g["sum"], w["sum"])
        elif exact_float:
            assert np.array_equal(np.asarray(g["sum"], np.float64).view(np.uint64), np.asarray(w["sum"], np.float64).view(np.uint64))


def _float_close(got, want, cv):
    """float64 sums of the same values added in another order: within cv * 2^-52 * sum(|v|), |v| < 1e4 here."""
    with np.errstate(all="ignore"):
        return np.all((np.isnan(got) & np.isnan(want)) | (got == want) | (np.abs(got - want) <= cv * cv * 2.0 ** -52 * 1e4))


AGG_CASES = [(VAL64, None, 0, 1), (VAL32, KEY64, -5, 16), (VALF, KEY32, 0, 16), (VAL64, KEY64, -1000, 2001),
             (VALF, None, 0, 1), (VALF, KEY64, -2048, 4096), (KEY64, KEY64, -5, 16)]


@pytest.mark.parametrize("value,key,key_min,span", AGG_CASES)
@pytest.mark.parametrize("corpus_name", ["uniform8", "natural3"])
def test_aggregates_merged_equal_unsharded(request, corpus_name, value, key, key_min, span, level):
    env = request.getfixturevalue(corpus_name)
    readers, vt = env["readers"], env["one"].segments[0].col_types[value]
    for qs, xs, ms in list(_shapes(env["n_terms"], 13))[:3]:
        for filt in FILTERS:
            kw = dict(filt=filt, exclude=xs, min_match=ms)
            buf = _gather(readers, qs, value, key, key_min, span, **kw)
            got = _merge(buf, len(qs), vt, key_min, span)
            want = sdb.ExecuteMatchAggregatesGroupsBatch(env["one"], qs, value, key, key_min, span, **kw)
            _assert_agg_equal(got, want, vt, exact_float=False)
            if vt != 1:
                continue
            # the float64 sums: bit for bit the ranks' partials (each rank's buffer merged alone) added in rank order
            parts = [_merge(buf[r:r + 1], len(qs), vt, key_min, span) for r in range(len(readers))]
            for sel in (lambda r: r, lambda r: r["null"]):
                acc = np.asarray(sel(parts[0])["sum"], np.float64).copy()
                with np.errstate(all="ignore"):
                    for p in parts[1:]:
                        s = np.asarray(sel(p)["sum"], np.float64)
                        acc = np.where(np.asarray(sel(p)["count_value"]) > 0, acc + s, acc)
                g = np.asarray(sel(got)["sum"], np.float64)
                real = ~np.isnan(g)   # a NaN is any NaN: NumPy's inf + -inf on the host has the sign bit set
                assert np.array_equal(real, ~np.isnan(acc)) and np.array_equal(g[real].view(np.uint64), acc[real].view(np.uint64))
                w = np.asarray(sel(want)["sum"], np.float64)
                assert _float_close(g, w, np.asarray(sel(want)["count_value"]).astype(np.float64))


@pytest.mark.parametrize("corpus_name", ["uniform8", "natural3"])
def test_dist_entries_at_world_one_equal_local(request, corpus_name):
    """Without sdbg_dist_init the all-gather is a copy and the merge of one rank the identity."""
    env = request.getfixturevalue(corpus_name)
    qs, xs, ms = _batch(env["n_terms"], 17)
    for reader in env["readers"] + [env["one"]]:
        bases = np.cumsum([0] + [g.n_docs for g in reader.segments])[:-1]
        for field in (VAL64, VALF):
            for k in (10, 1000):
                got = sdb.ExecuteDistTopKByColumnGroupsBatch(reader, qs, field, k, True, True, exclude=xs, min_match=ms)
                want = sdb.ExecuteTopKByColumnGroupsBatch(reader, qs, field, k, True, True, exclude=xs, min_match=ms)
                assert np.array_equal(got["n_out"], want["n_out"])
                for q in range(len(qs)):
                    assert np.all(got["segs"][q] == 0)
                    assert np.array_equal(got["docs"][q], bases[want["segs"][q]] + want["docs"][q])
                    assert np.array_equal(got["values"][q].view(np.uint8), want["values"][q].view(np.uint8))
                    assert np.array_equal(got["nulls"][q], want["nulls"][q])
        for value, key, key_min, span in AGG_CASES:
            vt = reader.segments[0].col_types[value]
            for filt in FILTERS:
                kw = dict(filt=filt, exclude=xs, min_match=ms)
                got = sdb.ExecuteDistMatchAggregatesGroupsBatch(reader, qs, value, key, key_min, span, **kw)
                want = sdb.ExecuteMatchAggregatesGroupsBatch(reader, qs, value, key, key_min, span, **kw)
                _assert_agg_equal(got, want, vt, exact_float=False)
                if vt == 1:   # float64 sums: the local pass adds with atomics, so only within its rounding
                    for sel in (lambda r: r, lambda r: r["null"]):
                        assert _float_close(np.asarray(sel(got)["sum"], np.float64), np.asarray(sel(want)["sum"], np.float64),
                                            np.asarray(sel(want)["count_value"]).astype(np.float64))


# ---------------------------------------------------------------- crafted buffers
def _crafted(R, nq, span, vt, rng, empty_ranks=()):
    """[R, words] device buffers with random cells: counts, 128-bit sums that carry, order keys; cells of empty_ranks
    and a random quarter of the others have no values."""
    n = nq * (span + 1)
    cells = np.zeros((R, n, 6), np.uint64)
    cells[..., 0] = rng.integers(0, 1 << 40, (R, n), dtype=np.uint64)
    cells[..., 1] = cells[..., 0] // 2
    cells[rng.random((R, n)) < 0.25, 1] = 0
    for r in empty_ranks:
        cells[r] = 0
    if vt == 1:
        cells[..., 2] = (rng.normal(size=(R, n)) * 1e6).view(np.uint64)
    else:
        cells[..., 2] = rng.integers(0, 2 ** 64, (R, n), dtype=np.uint64)                   # low words: carries
        cells[..., 3] = rng.integers(-5, 5, (R, n)).astype(np.int64).view(np.uint64)
    cells[..., 4] = rng.integers(1, 2 ** 64, (R, n), dtype=np.uint64)
    cells[..., 5] = rng.integers(1, 2 ** 64, (R, n), dtype=np.uint64)
    cells[cells[..., 1] == 0, 2:] = 0
    hdr = np.zeros((R, 8), np.uint64)
    hdr[:, 0], hdr[:, 1], hdr[:, 2] = vt, span, nq
    return hdr, cells


def _to_device(hdr, cells):
    import torch
    raw = np.concatenate([hdr, cells.reshape(cells.shape[0], -1)], axis=1).view(np.int64)
    t = torch.from_numpy(np.ascontiguousarray(raw)).cuda()
    torch.cuda.synchronize()
    return t


def _flip(o, vt):
    """Order key -> the value bits as the result reports them (sort_order_value)."""
    sign = np.uint64(1 << 63)
    if vt != 1:
        return (o ^ sign).view(np.int64)
    return np.where((o & sign) != 0, o ^ sign, ~o).view(np.int64)


@pytest.mark.parametrize("vt", [0, 1])
@pytest.mark.parametrize("R,empty", [(1, ()), (3, (1,)), (8, (0, 7)), (8, tuple(range(8)))])
def test_merge_crafted_cells(R, empty, vt):
    nq, span = 5, 16
    rng = np.random.default_rng(R * 10 + vt)
    hdr, cells = _crafted(R, nq, span, vt, rng, empty)
    got = _merge(_to_device(hdr, cells), nq, vt, 0, span)
    n = nq * (span + 1)
    cnt = cells[..., 0].sum(axis=0)
    cv = cells[..., 1].sum(axis=0)
    has = cells[..., 1] > 0
    want_min = np.where(cv > 0, _flip(~np.max(np.where(has, cells[..., 4], 0), axis=0), vt), 0)
    want_max = np.where(cv > 0, _flip(np.max(np.where(has, cells[..., 5], 0), axis=0), vt), 0)
    flat = lambda f: np.concatenate([np.asarray(got[f]).reshape(-1), np.asarray(got["null"][f]).reshape(-1)])
    assert np.array_equal(flat("count"), cnt) and np.array_equal(flat("count_value"), cv)
    assert np.array_equal(flat("min").view(np.int64), want_min) and np.array_equal(flat("max").view(np.int64), want_max)
    sums = flat("sum")
    for i in range(n):
        if vt == 1:
            acc = None
            for r in range(R):
                if cells[r, i, 1]:
                    v = cells[r, i, 2:3].view(np.float64)[0]
                    acc = v if acc is None else acc + v
            want = 0.0 if acc is None else acc
            assert np.float64(sums[i]).view(np.uint64) == np.float64(want).view(np.uint64), i
        else:
            want = sum((int(cells[r, i, 3].view(np.int64)) << 64) + int(cells[r, i, 2]) for r in range(R))
            want = (want + 2 ** 127) % 2 ** 128 - 2 ** 127
            assert (sums[i] if cv[i] else 0) == (want if cv[i] else 0), i


def test_merge_rejects_bad_headers():
    nq, span, R = 3, 4, 3
    rng = np.random.default_rng(2)
    for word, value in ((0, 1), (1, 5), (2, 4), (3, 1), (4, 1)):   # type, span, nq, failure word, out-of-range word
        hdr, cells = _crafted(R, nq, span, 0, rng)
        hdr[2, word] = value
        with pytest.raises(SdbgError, match="^EINVAL"):
            _merge(_to_device(hdr, cells), nq, 0, 0, span)
    hdr, cells = _crafted(R, nq, span, 0, rng)
    _merge(_to_device(hdr, cells), nq, 0, 0, span)


def _expect_rejected(code, fn):
    before = ctx().launches
    with pytest.raises(SdbgError, match="^" + code):
        fn()
    assert ctx().launches == before, "a rejected call queued work"


def test_scalar_errors_queue_nothing(uniform8):
    reader = uniform8["readers"][0]
    qs = [[[0, 1]]]
    buf = _cuda_zeros(sdb.match_aggregate_device_bytes(1, 4097) // 8)
    _expect_rejected("EINVAL", lambda: sdb.ExecuteDistFacetCountsGroupsBatch(reader, qs, KEY64, 0, 0))
    _expect_rejected("EINVAL", lambda: sdb.ExecuteDistFacetCountsGroupsBatch(reader, qs, KEY64, I64_MAX, 2))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.ExecuteDistFacetCountsGroupsBatch(reader, qs, KEY64, 0, 32769))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.ExecuteDistMatchAggregatesGroupsBatch(reader, qs, VAL64, KEY64, 0, 4097))
    _expect_rejected("EINVAL", lambda: sdb.ExecuteDistMatchAggregatesGroupsBatch(reader, qs, VAL64, KEY64, 0, 0))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.MatchAggregatesDevice(reader, qs, VAL64, buf.data_ptr(), KEY64, 0, 4097))
    _expect_rejected("EINVAL", lambda: sdb.merge_aggregates_gathered(ctx(), buf.data_ptr(), 0, 1, 0))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.merge_aggregates_gathered(ctx(), buf.data_ptr(), 1, 1, 0, 0, 4097))
    segs = (C_VP * 1)(reader.segments[0]._h)
    counts = np.zeros(1, np.uint64)
    _expect_rejected("EINVAL", lambda: N.check(N.lib().sdbg_dist_match_count_batch_groups_min(
        segs, 1, None, None, None, None, 1, None, None, None, counts.ctypes.data_as(C_VP)), ctx()._h))


def test_rank_failures_reach_the_merge(uniform8):
    """A rank's own failure (missing value column, bad term id, key out of range) returns its code and sets its failure
    or out-of-range word, so that the merge fails on every rank."""
    readers = uniform8["readers"][:2]
    qs = [[[0, 1]]]
    words = sdb.match_aggregate_device_bytes(1, 16) // 8
    for bad_call, code in ((lambda p: sdb.MatchAggregatesDevice(readers[1], qs, 77, p, KEY64, -5, 16), "ENOTFOUND"),
                           (lambda p: sdb.MatchAggregatesDevice(readers[1], [[[0, 999]]], VAL64, p, KEY64, -5, 16), "EINVAL")):
        buf = _cuda_zeros(words, 2)
        sdb.MatchAggregatesDevice(readers[0], qs, VAL64, buf[0].data_ptr(), KEY64, -5, 16)
        with pytest.raises(SdbgError, match="^" + code):
            bad_call(buf[1].data_ptr())
        with pytest.raises(SdbgError, match="^EINVAL"):
            _merge(buf, 1, 0, -5, 16)
    buf = _gather(readers, qs, VAL64, KEY64, 0, 4)         # keys -5 .. 10 outside [0, 4)
    with pytest.raises(SdbgError, match="^EINVAL"):
        _merge(buf, 1, 0, 0, 4)
    with pytest.raises(SdbgError, match="^EINVAL"):
        sdb.ExecuteDistFacetCountsGroupsBatch(readers[0], qs, KEY64, 0, 4)
    with pytest.raises(SdbgError, match="^EINVAL"):
        sdb.ExecuteDistCountGroupsBatch(readers[0], [[[0, 999]]])
    with pytest.raises(ValueError):                        # no per-rank default range
        sdb.ExecuteDistFacetCountsGroupsBatch(readers[0], qs, KEY64, None, None)


def test_missing_column_reaches_the_library(uniform8):
    """The Python dist wrappers check nothing about this rank's columns before the library call, so a rank without the
    column enters the collective and fails there (SdbgError), instead of raising on its own and leaving the others
    waiting."""
    reader = uniform8["readers"][0]
    qs = [[[0, 1]]]
    for call in (lambda: sdb.ExecuteDistFacetCountsGroupsBatch(reader, qs, 77, 0, 16),
                 lambda: sdb.ExecuteDistMatchAggregatesGroupsBatch(reader, qs, 77),
                 lambda: sdb.ExecuteDistMatchAggregatesGroupsBatch(reader, qs, VAL64, 77, 0, 16),
                 lambda: sdb.ExecuteDistTopKByColumnGroupsBatch(reader, qs, 77, 10)):
        with pytest.raises(SdbgError, match="^ENOTFOUND"):
            call()


# ---------------------------------------------------------------- sorted scan
SORT_COLS = (VAL64, VALF, VAL32, KEY64, KEY32)


def _sort_gather(env, qs, field, k, desc, nf, **kw):
    R = len(env["readers"])
    buf = _cuda_zeros(sdb.topk_by_column_device_bytes(len(qs), k) // 8, R)
    for r, reader in enumerate(env["readers"]):
        sdb.TopKByColumnDevice(reader, qs, field, k, r, buf[r].data_ptr(), descending=desc, nulls_first=nf, **kw)
    return buf


def _assert_sort_equal_unsharded(env, got, want):
    """Merged hits (rank, ordinal within the rank + 1) against the unsharded scan's (segment, doc)."""
    assert np.array_equal(got["n_out"], want["n_out"])
    rank_base = np.array([env["gbase"][rk[0]] for rk in env["ranks"]], np.int64)
    for q in range(len(got["n_out"])):
        g_ord = rank_base[got["segs"][q].astype(np.int64)] + got["docs"][q].astype(np.int64) - 1
        w_ord = env["gbase"][want["segs"][q].astype(np.int64)] + want["docs"][q].astype(np.int64) - 1
        assert np.array_equal(g_ord, w_ord), q
        assert np.array_equal(got["nulls"][q], want["nulls"][q]), q
        assert np.array_equal(got["values"][q].view(np.uint8), want["values"][q].view(np.uint8)), q


@pytest.mark.parametrize("k", [1, 10, 1000, 4096])
@pytest.mark.parametrize("corpus_name", ["uniform8", "natural3"])
def test_sorted_merge_equals_unsharded(request, corpus_name, k, level):
    env = request.getfixturevalue(corpus_name)
    for field in SORT_COLS:
        vt = env["one"].segments[0].col_types[field]
        for i, (desc, nf) in enumerate(((False, False), (True, False), (False, True), (True, True))):
            for qs, xs, ms in list(_shapes(env["n_terms"], 23 + i))[:2]:
                filt = FILTERS[i % 2]
                kw = dict(filt=filt, exclude=xs, min_match=ms)
                got = sdb.merge_topk_by_column_gathered(ctx(), _sort_gather(env, qs, field, k, desc, nf, **kw).data_ptr(),
                                                        len(env["readers"]), len(qs), k, vt)
                want = sdb.ExecuteTopKByColumnGroupsBatch(env["one"], qs, field, k, desc, nf, **kw)
                _assert_sort_equal_unsharded(env, got, want)


def test_sorted_merge_ties_across_ranks(uniform8):
    """KEY64 holds 16 values: at k = 1000 every hit ties with hundreds of others on every rank, so the order is decided
    by (rank, ordinal) alone."""
    qs = [[[0, 1, 4]], [[2]], [[0], [4]]]
    for desc in (False, True):
        got = sdb.merge_topk_by_column_gathered(ctx(), _sort_gather(uniform8, qs, KEY64, 1000, desc, False).data_ptr(), 8,
                                                len(qs), 1000, 0)
        want = sdb.ExecuteTopKByColumnGroupsBatch(uniform8["one"], qs, KEY64, 1000, desc)
        _assert_sort_equal_unsharded(uniform8, got, want)
        assert len(set(got["segs"][0].tolist())) > 1


def test_sorted_merge_rejects_bad_headers(uniform8):
    env = dict(uniform8, readers=uniform8["readers"][:3], ranks=uniform8["ranks"][:3])
    qs = [[[0, 1]], [[2, 3]]]
    for word, value in ((0, 1), (1, 1), (2, 1), (3, 11), (4, 3), (5, 1)):   # type, desc, nulls_first, k, nq, failure word
        buf = _sort_gather(env, qs, VAL64, 10, False, False)
        buf[2, word] = value
        import torch
        torch.cuda.synchronize()
        with pytest.raises(SdbgError, match="^EINVAL"):
            sdb.merge_topk_by_column_gathered(ctx(), buf.data_ptr(), 3, len(qs), 10, 0)
    buf = _cuda_zeros(sdb.topk_by_column_device_bytes(len(qs), 10) // 8, 2)
    sdb.TopKByColumnDevice(env["readers"][0], qs, VAL64, 10, 0, buf[0].data_ptr())
    with pytest.raises(SdbgError, match="^ENOTFOUND"):
        sdb.TopKByColumnDevice(env["readers"][1], qs, 77, 10, 1, buf[1].data_ptr())
    with pytest.raises(SdbgError, match="^EINVAL"):
        sdb.merge_topk_by_column_gathered(ctx(), buf.data_ptr(), 2, len(qs), 10, 0)


def test_sorted_scalar_errors_queue_nothing(uniform8):
    reader = uniform8["readers"][0]
    qs = [[[0, 1]]]
    buf = _cuda_zeros(sdb.topk_by_column_device_bytes(1, 4097) // 8)
    _expect_rejected("EINVAL", lambda: sdb.ExecuteDistTopKByColumnGroupsBatch(reader, qs, VAL64, 0))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.ExecuteDistTopKByColumnGroupsBatch(reader, qs, VAL64, 4097))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.TopKByColumnDevice(reader, qs, VAL64, 4097, 0, buf.data_ptr()))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.TopKByColumnDevice(reader, qs, VAL64, 10, 1 << 31, buf.data_ptr()))
    _expect_rejected("EINVAL", lambda: sdb.merge_topk_by_column_gathered(ctx(), buf.data_ptr(), 0, 1, 10, 0))
    _expect_rejected("EINVAL", lambda: sdb.merge_topk_by_column_gathered(ctx(), buf.data_ptr(), 1, 1, 0, 0))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.merge_topk_by_column_gathered(ctx(), buf.data_ptr(), 1, 1, 4097, 0))


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
    corpus = Corpus(parts)
    rng = np.random.default_rng(9)
    env = _env(c, corpus, [[0, 1]], [_columns(rng, o.n_docs) for o in corpus.osegs])
    yield env
    for g in env["gsegs"]:
        g.close()
    c.close()


def test_nccl_world_one_equals_local(nccl):
    reader = nccl["one"]
    qs, xs, ms = _batch(nccl["n_terms"], 19)
    for filt in FILTERS:
        kw = dict(filt=filt, exclude=xs, min_match=ms)
        assert np.array_equal(sdb.ExecuteDistCountGroupsBatch(reader, qs, **kw), sdb.ExecuteCountGroupsBatch(reader, qs, **kw))
        got = sdb.ExecuteDistFacetCountsGroupsBatch(reader, qs, KEY32, 0, 16, **kw)
        want = sdb.ExecuteFacetCountsGroupsBatch(reader, qs, KEY32, 0, 16, **kw)
        assert np.array_equal(got["counts"], want["counts"]) and np.array_equal(got["nulls"], want["nulls"])
        for value, key, key_min, span in AGG_CASES:
            got = sdb.ExecuteDistMatchAggregatesGroupsBatch(reader, qs, value, key, key_min, span, **kw)
            want = sdb.ExecuteMatchAggregatesGroupsBatch(reader, qs, value, key, key_min, span, **kw)
            _assert_agg_equal(got, want, reader.segments[0].col_types[value], exact_float=False)
        got = sdb.ExecuteDistTopKByColumnGroupsBatch(reader, qs, VALF, 100, True, **kw)
        want = sdb.ExecuteTopKByColumnGroupsBatch(reader, qs, VALF, 100, True, **kw)
        assert np.array_equal(got["n_out"], want["n_out"])
        bases = np.cumsum([0] + [g.n_docs for g in reader.segments])[:-1]
        for q in range(len(qs)):
            assert np.array_equal(got["docs"][q], bases[want["segs"][q]] + want["docs"][q])
            assert np.array_equal(got["values"][q].view(np.uint8), want["values"][q].view(np.uint8))


# ---------------------------------------------------------------- scale
def test_benchmark_scale_batch_at_eight_ranks(uniform8):
    """4096 two-term ORs at 8 ranks through the device forms and the merge, grouped by 2001 keys (394 MB per rank)."""
    rng = np.random.default_rng(4)
    qs = [[[int(a), int(b)]] for a, b in (rng.choice(uniform8["n_terms"], 2, replace=False) for _ in range(4096))]
    buf = _gather(uniform8["readers"], qs, VALF, KEY64, -1000, 2001)
    got = _merge(buf, len(qs), 1, -1000, 2001)
    want = sdb.ExecuteMatchAggregatesGroupsBatch(uniform8["one"], qs, VALF, KEY64, -1000, 2001)
    _assert_agg_equal(got, want, 1, exact_float=False)
    assert _float_close(np.asarray(got["sum"]), np.asarray(want["sum"]), np.asarray(want["count_value"]).astype(np.float64))
    got = sdb.merge_topk_by_column_gathered(ctx(), _sort_gather(uniform8, qs, VAL64, 1000, True, False).data_ptr(), 8,
                                            len(qs), 1000, 0)
    _assert_sort_equal_unsharded(uniform8, got, sdb.ExecuteTopKByColumnGroupsBatch(uniform8["one"], qs, VAL64, 1000, True))
    counts = sdb.ExecuteDistCountGroupsBatch(uniform8["readers"][0], qs)
    assert np.array_equal(counts, sdb.ExecuteCountGroupsBatch(uniform8["readers"][0], qs))

