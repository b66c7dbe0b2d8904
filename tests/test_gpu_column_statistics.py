"""Plans chosen from cached column statistics: the min / max (dense range, wide limbs, packed COUNT|SUM word, facet key
range), the zonemaps (skip verdicts) and the bit-packed words. Each reader is compared with NumPy over the column's current values (exact Python-int sums) after the values change in every
way the library allows, and each statistics-gated choice is placed on both sides of its limit, up to the GROUP BY's row
limit of 2^31 - 1 rows per GPU."""
import json
import math
import os
import subprocess
import sys
import time
from fractions import Fraction

import numpy as np
import pytest

import serenedb_b200 as sdb
from serenedb_b200._native import SdbgError

pytestmark = pytest.mark.gpu

INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
N = 200_000                      # 98 zonemap blocks of 2048 rows
KEY, SUBJ = 1, 2                 # the GROUP BY key column and the column whose values change
TILE = 512                       # rows per tile of the TMA GROUP BY (packed words are dealt by tile)

# GROUP BY paths: default (TMA, packed COUNT|SUM words when the statistics allow), TMA with plain words, the
# register-staged kernel, the hash table
PATHS = [{}, {"SDBG_GROUPBY_PACKED": "0"}, {"SDBG_GROUPBY_TMA": "0"}, {"SDBG_GROUPBY_FORCE_HASH": "1"}]


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
_CTX = None
_SEGMENTS = []


def ctx():
    """The module's own context (pruning off: exact totals)."""
    return _CTX


@pytest.fixture(scope="module", autouse=True)
def _own_context():
    """The module grows device buffers far beyond other tests' (the 2^26-key dense table, the hash table for a 2^24
    hint, 32 GiB of raw columns at the row limit). They belong to this context and to torch's cache, and both are given
    back when the module ends, so the tests after it find the device memory they had before it."""
    global _CTX
    _CTX = sdb.Context(0)
    _CTX.set_wand(False)
    yield
    import gc
    import torch
    for s in _SEGMENTS:
        s.close()
    _SEGMENTS.clear()
    _CTX.close()
    _CTX = None
    gc.collect()
    torch.cuda.empty_cache()


def _segment(n_docs):
    s = sdb.Segment(ctx(), n_docs)
    _SEGMENTS.append(s)                       # closed before the context at the latest
    return s


def _device_view(ptr, n, dtype):
    """A torch tensor over n values of `dtype` at device address `ptr` (no copy)."""
    import torch

    class _Mem:
        __cuda_array_interface__ = dict(shape=(int(n),), typestr=np.dtype(dtype).str, data=(int(ptr), False), version=3)
    return torch.as_tensor(_Mem(), device="cuda")


def _write_device(ptr, values):
    """Writes `values` to device address `ptr` the way a caller generating data in place would."""
    import torch
    ctx().sync()                                   # the library's queued work on the column is done
    _device_view(ptr, len(values), values.dtype).copy_(torch.from_numpy(values).cuda())
    torch.cuda.synchronize()


def _kernels_per_call(calls):
    """Names of the CUDA kernels each of `calls` launches, from one torch.profiler session; the calls are told apart by a
    fill kernel on torch's stream after each of them."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    mark = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in calls:
            fn()
            ctx().sync()
            mark.fill_(1.0)
            torch.cuda.synchronize()
    out, cur = [], []
    for e in sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start):
        if "FillFunctor" in e.name:
            out.append(cur)
            cur = []
        else:
            cur.append(e.name)
    assert len(out) == len(calls), (len(out), len(calls))
    return out


def _tma_args(names):
    """Template arguments of each filter_groupby_tma_kernel launch: [kPacked, kFor]."""
    out = []
    for n in names:
        if "filter_groupby_tma_kernel" in n:
            head = n.replace(" ", "").split("(")[0]
            out.append(head[head.index("<") + 1:head.rindex(">")].split(","))
    return out


def _env(monkeypatch, env):
    for k in ("SDBG_GROUPBY_PACKED", "SDBG_GROUPBY_TMA", "SDBG_GROUPBY_FORCE_HASH", "SDBG_GROUPBY_PACK_TABLES_MIN"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _f64_close(got, exact, count, abs_sum):
    """|got - exact| <= count * 2^-52 * sum|w| (exact Fractions: no overflow near DBL_MAX)."""
    if math.isinf(got) or math.isnan(got):
        return False
    return abs(Fraction(got) - exact) <= Fraction(max(count, 1)) * Fraction(1, 2**52) * abs_sum


def _exact_sum(w):
    """(sum w, sum |w|) as Fractions: exact near DBL_MAX, else math.fsum's correctly rounded sums (within half an ulp,
    far inside the bound they are used with)."""
    w = np.asarray(w, np.float64)
    if len(w) and np.abs(w).max() >= 2.0**1000:
        return sum(map(Fraction, w.tolist()), Fraction(0)), sum(map(Fraction, np.abs(w).tolist()), Fraction(0))
    return Fraction(math.fsum(w.tolist())), Fraction(math.fsum(np.abs(w).tolist()))


def ref_groups(keys, sel, ivals=None, ivalid=None, fvals=None, fvalid=None):
    """{key: (count, sum_int, cnt_f, exact Fraction sum_f, sum |w|)} over the selected rows."""
    out = {}
    ks = keys[sel]
    order = np.argsort(ks, kind="stable")
    ks = ks[order]
    uk, start = np.unique(ks, return_index=True)
    end = list(start[1:]) + [len(ks)]
    idx = np.nonzero(sel)[0][order]
    for k, a, b in zip(uk, start, end):
        rows = idx[a:b]
        s_i = 0
        if ivals is not None:
            r = rows if ivalid is None else rows[ivalid[rows]]
            s_i = int(ivals[r].astype(object).sum())
        cf, sf, af = len(rows), Fraction(0), Fraction(0)
        if fvals is not None:
            r = rows if fvalid is None else rows[fvalid[rows]]
            cf = len(r)
            sf, af = _exact_sum(fvals[r])
        out[int(k)] = (len(rows), s_i, cf, sf, af)
    return out


def assert_groups(got, ref, has_i, has_f):
    assert [int(k) for k in got["key"]] == sorted(ref), (list(got["key"][:8]), sorted(ref)[:8])
    sums = sdb.engine.sum_i128(got)
    for j, k in enumerate(int(x) for x in got["key"]):
        cnt, s_i, cf, sf, af = ref[k]
        assert int(got["count"][j]) == cnt, (k, int(got["count"][j]), cnt)
        if has_i:
            assert sums[j] == s_i, (k, sums[j], s_i)
        if has_f:
            assert int(got["cnt_f64"][j]) == cf, (k, int(got["cnt_f64"][j]), cf)
            assert _f64_close(float(got["sum_f64"][j]), sf, cnt, af), (k, float(got["sum_f64"][j]), float(sf))


def _bits(mask, rows):
    return np.unpackbits(mask.view(np.uint8), bitorder="little")[:rows].astype(bool)


# ---------------------------------------------------------------------------------------------------------------------
# 1. values that change, against every reader
# ---------------------------------------------------------------------------------------------------------------------
def _table():
    """A segment of N docs: one term holding every doc (so full-text readers see every row), the key column."""
    w = sdb.PostingsWriter(N, has_wand=True)
    w.add_term(np.arange(1, N + 1, dtype=np.uint32), np.ones(N, np.uint32))
    doc, metas = w.finish()
    g = _segment(N)
    g.stage_postings(doc, metas)
    keys = (np.arange(N) % 61).astype(np.int64)
    g.stage_column(KEY, keys)
    return g, sdb.IndexReader([g], N, N, [N]), keys


def _window(vals, valid):
    """A BETWEEN range holding rows 50_000 .. 52_000 of the current values (1-2 zonemap blocks), as Python scalars."""
    w = vals[50_000:52_001]
    if valid is not None:
        w = w[valid[50_000:52_001]]
    lo, hi = w.min(), w.max()
    return (float(lo), float(hi)) if vals.dtype == np.float64 else (int(lo), int(hi))


def check_readers(monkeypatch, seg, reader, keys, vals, valid=None):
    """Every reader of column SUBJ against NumPy over `vals` (NULL where valid is False)."""
    is_f = vals.dtype == np.float64
    ok = np.ones(len(vals), bool) if valid is None else valid
    lo, hi = _window(vals, valid)
    pred = [sdb.pred(SUBJ, "BETWEEN", lo, hi)]
    passing = ok & (vals >= lo) & (vals <= hi)
    assert 500 <= passing.sum() < 0.05 * N                         # zonemap-selective
    # filter_bitmap, count_sum, column_minmax
    assert np.array_equal(_bits(seg.filter_bitmap(pred), N), passing)
    scan = sdb.IResearchScan([seg])
    for preds, sel in ((pred, passing), ([], np.ones(N, bool))):
        cnt, s_i, s_f = scan.count_sum(preds, SUBJ)
        assert cnt == int(sel.sum())
        r = sel & ok
        if is_f:
            ex, ab = _exact_sum(vals[r])
            assert _f64_close(s_f, ex, cnt, ab)
        else:
            assert s_i == int(vals[r].astype(object).sum())
    if not is_f:
        assert seg.column_minmax(SUBJ) == (int(vals[ok].min()), int(vals[ok].max()))
    # GROUP BY on every path, with and without the zonemap-selective predicate; the partial + finalize pair
    si, sf = (None, SUBJ) if is_f else (SUBJ, None)
    refs = [(preds, ref_groups(keys, sel, None if is_f else vals, valid, vals if is_f else None, valid))
            for preds, sel in ((pred, passing), ([], np.ones(N, bool)))]
    for env in PATHS:
        _env(monkeypatch, env)
        for preds, ref in refs:
            assert_groups(scan.groupby(preds, KEY, sum_int_field=si, avg_f64_field=sf), ref, not is_f, is_f)
    _env(monkeypatch, {})
    import torch
    span = 61
    d_i64 = torch.zeros(4 * span, dtype=torch.int64, device="cuda")
    d_f64 = torch.zeros(span, dtype=torch.float64, device="cuda")
    scan.groupby_partial(pred, KEY, 0, span, si, sf, d_i64.data_ptr(), d_f64.data_ptr())
    assert_groups(scan.groupby_finalize(0, span, d_i64.data_ptr(), d_f64.data_ptr(), span), refs[0][1], not is_f, is_f)
    # GROUP BY the changing column itself: its min / max are the dense table's range
    if not is_f and valid is None and int(vals.max()) - int(vals.min()) < 2**20:
        for env in PATHS:
            _env(monkeypatch, env)
            got = scan.groupby([], SUBJ)
            uk, cnt = np.unique(vals, return_counts=True)
            assert np.array_equal(got["key"], uk) and np.array_equal(got["count"], cnt)
        _env(monkeypatch, {})
    # BM25 with the column filter (exact total: pruning is off in this context)
    hits, total = sdb.ExecuteTopK(reader, [0], sdb.OR, sdb.BM25(), 10, filt=sdb.pred(SUBJ, "BETWEEN", lo, hi))
    assert total == int(passing.sum()) and len(hits) == 10 and passing[hits["doc"].astype(np.int64) - 1].all()
    # sorted scan with zonemap windows (pruning level 2)
    order = np.argsort(np.where(ok, vals, np.inf if is_f else INT64_MAX), kind="stable")[:int(ok.sum())]
    try:
        ctx().set_wand(2)
        for desc in (False, True):
            got = sdb.ExecuteTopKByColumn(reader, [0], sdb.OR, SUBJ, 50, descending=desc)
            exp = (order[::-1] if desc else order)[:50]
            d = got["docs"].astype(np.int64) - 1                        # ties may come in another doc order
            assert len(set(d)) == 50 and ok[d].all() and np.array_equal(vals[d], got["values"]), desc
            assert np.array_equal(got["values"], vals[exp]), desc
    finally:
        ctx().set_wand(0)
    # facet counts over the default key range, and aggregates
    if not is_f and int(vals[ok].max()) - int(vals[ok].min()) < 32768:
        got = sdb.ExecuteFacetCounts(reader, [0], sdb.OR, SUBJ)
        uk, cnt = np.unique(vals[ok], return_counts=True)
        exp = {int(k): int(c) for k, c in zip(uk, cnt)}
        if not ok.all():
            exp[None] = int((~ok).sum())
        assert got == exp
    agg = sdb.ExecuteMatchAggregates(reader, [0], sdb.OR, SUBJ)
    v = vals[ok]
    assert agg["count"] == N and agg["count_value"] == len(v)
    assert agg["min"] == v.min() and agg["max"] == v.max()
    if is_f:
        ex, ab = _exact_sum(v)
        assert _f64_close(float(agg["sum"]), ex, len(v), ab)
    else:
        assert agg["sum"] == int(v.astype(object).sum())
    # gather
    docs = np.random.default_rng(3).integers(1, N + 1, 3000).astype(np.uint32)
    gv, gok = seg.gather(SUBJ, docs, vals.dtype)
    assert np.array_equal(gok, ok[docs - 1]) and np.array_equal(gv[gok], vals[docs - 1][gok])


def _old_new(dtype):
    """(old, new): old ascends in clusters of 100 from 1000 to 2999; new descends in clusters of 8 from 12_999 to
    -12_000. The new values move the min and the max and every zonemap block, and a stale plan
    gives a different answer rather than an error (a stale packing bias above the new minimum carries the sum field into
    the count). Both ranges fit the facet bins."""
    i = np.arange(N)
    old = (i // 100 + 1000).astype(dtype)
    new = ((N - 1 - i) // 8 - 12_000).astype(dtype)
    if dtype == np.float64:
        old = old + 0.25
        new = new * 1.5 + 0.5
    return old, new


def _nulls():
    v = np.ones(N, bool)
    v[np.random.default_rng(11).choice(N, N // 10, replace=False)] = False
    v[50_000] = v[52_000] = True
    return v


def _validity(valid):
    return np.packbits(valid, bitorder="little").view(np.uint64)      # N is a multiple of 64


@pytest.mark.parametrize("how", ["packed_i64", "raw_i64", "i32", "f64", "nullable_i64"])
def test_writes_through_column_device_ptr(monkeypatch, how):
    """sdbg_column_device_ptr is the way to write a column in place: every statistic of the old values is dropped, and a
    packed column is read through its raw view from then on."""
    seg, reader, keys = _table()
    dtype = {"i32": np.int32, "f64": np.float64}.get(how, np.int64)
    old, new = _old_new(dtype)
    valid = _nulls() if how == "nullable_i64" else None
    if how == "raw_i64":      # full 64-bit values: not smaller packed, held raw
        old = np.random.default_rng(5).integers(INT64_MIN, INT64_MAX, N, dtype=np.int64, endpoint=True)
        old[50_000:52_001] = np.arange(2001)
    seg.stage_column(SUBJ, old, None if valid is None else _validity(valid))
    assert (seg.column_packed(SUBJ, N) is not None) == (how == "packed_i64")
    check_readers(monkeypatch, seg, reader, keys, old, valid)          # the statistics of the old values are cached
    ptr, rows = seg.column_device_ptr(SUBJ)
    assert rows == N
    _write_device(ptr, new)
    check_readers(monkeypatch, seg, reader, keys, new, valid)
    assert seg.column_packed(SUBJ, N) is None                          # the raw view is the column now
    ptr2, _ = seg.column_device_ptr(SUBJ)                              # a second write: announced the same way
    _write_device(ptr2, old)
    check_readers(monkeypatch, seg, reader, keys, old, valid)
    seg.stage_column(SUBJ, new, None if valid is None else _validity(valid))   # restaging packs it again
    assert (seg.column_packed(SUBJ, N) is not None) == (how in ("packed_i64", "raw_i64"))   # the new values are narrow
    check_readers(monkeypatch, seg, reader, keys, new, valid)
    seg.close()


def test_borrowed_buffer_restaged_after_a_write(monkeypatch):
    """A borrowed device column that its owner rewrites is restaged with sdbg_stage_column_device: that resets every
    statistic of the old values."""
    import torch
    seg, reader, keys = _table()
    for dtype in (np.int64, np.int32, np.float64):
        old, new = _old_new(dtype)
        t = torch.from_numpy(old).cuda()
        torch.cuda.synchronize()
        seg.stage_column_device(SUBJ, t.data_ptr(), dtype, N)
        check_readers(monkeypatch, seg, reader, keys, old)
        ctx().sync()
        t.copy_(torch.from_numpy(new).cuda())
        torch.cuda.synchronize()
        seg.stage_column_device(SUBJ, t.data_ptr(), dtype, N)
        check_readers(monkeypatch, seg, reader, keys, new)
        del t
    seg.close()


def test_restaging_paths(monkeypatch):
    """Restaging from the host with the same shape, another type or another length, from the bit-packed form, and by
    generating the values on the device over an existing field."""
    import orc
    seg, reader, keys = _table()
    old, new = _old_new(np.int64)
    seg.stage_column(SUBJ, old)
    check_readers(monkeypatch, seg, reader, keys, old)
    seg.stage_column(SUBJ, new)                                         # same shape
    check_readers(monkeypatch, seg, reader, keys, new)
    for dtype in (np.int32, np.float64):                                # another type
        o, n = _old_new(dtype)
        seg.stage_column(SUBJ, o)
        check_readers(monkeypatch, seg, reader, keys, o)
        seg.stage_column(SUBJ, n)
        check_readers(monkeypatch, seg, reader, keys, n)
    short = new[:N // 2 + 2048 * 3 + 5] - 10**6                         # another length (rows past it are not read)
    seg.stage_column(SUBJ, short)
    assert seg.column_minmax(SUBJ) == (int(short.min()), int(short.max()))
    assert sdb.IResearchScan([seg]).count_sum([sdb.pred(SUBJ, "LT", -10**6)], SUBJ)[:2] == \
        (int((short < -10**6).sum()), int(short[short < -10**6].sum()))
    seg.stage_column(SUBJ, old)
    check_readers(monkeypatch, seg, reader, keys, old)
    seg.stage_column_for(SUBJ, sdb.pack_for(new))                      # from the bit-packed form
    assert seg.column_packed(SUBJ, N) is not None
    check_readers(monkeypatch, seg, reader, keys, new)
    seg.synth_column(SUBJ, 0, 7, 10**7, N)                              # generated on the device: (row0 + i) // 100
    check_readers(monkeypatch, seg, reader, keys, orc.synth_column(0, 7, 10**7, N))
    seg.stage_column_for(SUBJ, sdb.pack_for(new))
    check_readers(monkeypatch, seg, reader, keys, new)
    seg.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. statistics-gated choices at their limits
# ---------------------------------------------------------------------------------------------------------------------
def _segments(cols_per_seg):
    segs = []
    for cols in cols_per_seg:
        s = _segment(len(next(iter(cols.values()))))
        for f, v in cols.items():
            s.stage_column(f, v)
        segs.append(s)
    return segs


def _run_groupby(segs, cols_per_seg, key, si=None, sf=None, hint=0):
    """GROUP BY over the segments against the reference."""
    keys = np.concatenate([c[key] for c in cols_per_seg])
    iv = np.concatenate([c[si] for c in cols_per_seg]) if si is not None else None
    fv = np.concatenate([c[sf] for c in cols_per_seg]) if sf is not None else None
    got = sdb.IResearchScan(segs).groupby([], key, sum_int_field=si, avg_f64_field=sf, n_groups_hint=hint)
    assert_groups(got, ref_groups(keys, np.ones(len(keys), bool), iv, None, fv, None), si is not None, sf is not None)


def _pack_fill(tiles, nt, shift):
    """Sum column values: one key's rows fill word 0 of its slot to within one range (nt > 1) or two (nt = 1) of
    2^shift. Returns (cols per segment, range)."""
    cap = sum(-(-t // nt) for t in tiles) * TILE
    rng_ = (2**shift - 1) // cap                                        # range * cap < 2^shift <= range * (cap + 1)
    assert rng_ * cap < 2**shift <= rng_ * (cap + 1) and rng_ <= 2**32 - 1
    mn = INT32_MIN
    cols = []
    for si, t in enumerate(tiles):
        rows = t * TILE
        v = np.full(rows, mn + rng_, np.int64)
        k = np.full(rows, 3, np.int64)
        if si == 0:                                                     # the row that sets the minimum: another key, in
            r = TILE + 7 if nt > 1 else 7                               # a tile dealt to word 1 when there is one
            v[r], k[r] = mn, 4
        cols.append({1: k, 2: v})
    return cols, rng_


@pytest.mark.parametrize("nt", [1, 2, 3])
def test_packed_word_filled_to_its_limit(monkeypatch, nt):
    """COUNT << shift | SUM(v - min) in 1, 2 and 3 words per slot, over segments of ragged tile counts, with one key's
    rows filling its sum field to within a row or two of 2^shift: nothing carries into the count."""
    tiles = [7, 5, 1, 2]
    for shift in (34, 40, 43):                                          # 43: range near 2^32 - 1
        cols, _ = _pack_fill(tiles, nt, shift)
        segs = _segments(cols)
        _env(monkeypatch, {"SDBG_GROUPBY_PACK_TABLES_MIN": str(nt)})
        _run_groupby(segs, cols, 1, si=2)
        _env(monkeypatch, {})
        for s in segs:
            s.close()


def _shift_of(max_sum):
    s = 1
    while s < 63 and (1 << s) <= max_sum:
        s += 1
    return s


def test_packed_count_field_at_its_limit(monkeypatch):
    """cap_rows < 2^(64 - shift) for a range of 2^32 - 1 just holding and just failing for one word: every row of one
    key, the sum at its widest."""
    ok = [t for t in range(1, 200) if t * TILE < 2**(64 - _shift_of((2**32 - 1) * t * TILE))]
    t1 = max(ok)
    assert t1 + 1 not in ok and t1 == 127                               # 65_024 rows
    for tiles in (t1, t1 + 1):
        rows = tiles * TILE
        v = np.full(rows, INT32_MAX, np.int64)
        v[1] = INT32_MIN
        cols = [{1: np.zeros(rows, np.int64), 2: v}]
        segs = _segments(cols)
        _env(monkeypatch, {})
        _run_groupby(segs, cols, 1, si=2)
        segs[0].close()


@pytest.mark.parametrize("mn,mx,wide", [(INT32_MIN, INT32_MAX, False), (INT32_MIN, INT32_MAX + 1, True),
                                        (INT32_MIN - 1, INT32_MAX, True), (-5, INT32_MAX, False)])
def test_wide_limbs_at_int32_edges(monkeypatch, mn, mx, wide):
    """The wide-integer limbs switch on exactly past the int32 range; sums are exact on every path either way."""
    rows = 70_002
    rng = np.random.default_rng(mx & 0xFFFF)
    v = rng.choice(np.array([mn, mx, mn + 1, mx - 1, 0], np.int64), rows)
    v[:2] = mn, mx
    cols = [{1: rng.integers(0, 50, rows).astype(np.int64), 2: v}]
    segs = _segments(cols)
    for env in PATHS:
        _env(monkeypatch, env)
        _run_groupby(segs, cols, 1, si=2)
    _env(monkeypatch, {})
    segs[0].close()


@pytest.mark.parametrize("span,hint,dense", [(2**20, 0, True), (2**20 + 1, 0, False), (2**21, 2**18, True),
                                             (2**21 + 1, 2**18, False), (2**26, 2**23, True), (2**26 + 1, 2**24, False)])
def test_dense_or_hash_at_the_span_limits(monkeypatch, span, hint, dense):
    """Dense table up to a key span of max(2^20, 8 x hint) and 2^26, hash table past either."""
    rows = 8192
    rng = np.random.default_rng(span & 0xFFFF)
    k0 = -(2**40) + 17
    k = k0 + rng.integers(0, span, rows).astype(np.int64)
    k[:2] = k0, k0 + span - 1
    cols = [{1: k, 2: rng.integers(-1000, 1000, rows).astype(np.int64)}]
    segs = _segments(cols)
    _env(monkeypatch, {})
    _run_groupby(segs, cols, 1, si=2, hint=hint)
    segs[0].close()


def _plan_checks():
    """(ok, detail) per limit case: the kernels it launches, from one profiler session. The packed COUNT|SUM word at its
    fill limit in 1, 2 and 3 words and on both sides of the count-field limit; wide limbs (no packed word) exactly past
    the int32 range; the dense table up to max(2^20, 8 x hint) and 2^26 keys, the hash table past them."""
    cases = []                                            # (segments, groupby kwargs, env, check of the kernel names)

    def packed(flag):
        return lambda names: bool(_tma_args(names)) and all(a[0] == flag for a in _tma_args(names))
    for nt in (1, 2, 3):
        cases.append((_segments(_pack_fill([7, 5, 1, 2], nt, 43)[0]), dict(sum_int_field=2),
                      {"SDBG_GROUPBY_PACK_TABLES_MIN": str(nt)}, packed("true")))
    for tiles in (127, 128):                              # one word at 127 tiles, two past it
        v = np.full(tiles * TILE, INT32_MAX, np.int64)
        v[1] = INT32_MIN
        cases.append((_segments([{1: np.zeros(tiles * TILE, np.int64), 2: v}]), dict(sum_int_field=2), {}, packed("true")))
    for mn, mx, wide in ((INT32_MIN, INT32_MAX, False), (INT32_MIN, INT32_MAX + 1, True), (INT32_MIN - 1, INT32_MAX, True)):
        v = np.zeros(4096, np.int64)
        v[:2] = mn, mx
        cases.append((_segments([{1: np.arange(4096, dtype=np.int64) % 5, 2: v}]), dict(sum_int_field=2), {},
                      packed("false" if wide else "true")))
    for span, hint, dense in ((2**20, 0, True), (2**20 + 1, 0, False), (2**21, 2**18, True), (2**21 + 1, 2**18, False),
                              (2**26, 2**23, True), (2**26 + 1, 2**24, False)):
        k = np.zeros(4096, np.int64)
        k[1] = span - 1
        cases.append((_segments([{1: k, 2: np.ones(4096, np.int64)}]), dict(sum_int_field=2, n_groups_hint=hint), {},
                      (lambda d: lambda names: bool(_tma_args(names)) == d and
                       any("filter_groupby_hash_kernel" in n for n in names) != d)(dense)))

    def call(segs, kw, env):
        def fn():
            os.environ.update(env)
            try:
                sdb.IResearchScan(segs).groupby([], 1, **kw)
            finally:
                for k in env:
                    del os.environ[k]
        return fn
    names = _kernels_per_call([call(*c[:3]) for c in cases])
    out = [(bool(c[3](n)), [c[2], sorted(set(x[:70] for x in n))]) for c, n in zip(cases, names)]
    for c in cases:
        for s in c[0]:
            s.close()
    return out


def test_plans_flip_at_their_limits():
    """The plan of each limit case above, read from the kernel names torch.profiler records. The profiler runs in a
    child process: once a process has opened a profiler session, a later session in it can miss kernel records, and
    the other test modules that read kernel names must not inherit that."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys; sys.path[:0] = [%r, %r]; import json, serenedb_b200 as sdb, test_gpu_column_statistics as t; "
            "t._CTX = sdb.Context(0); print(json.dumps(t._plan_checks()))" % (os.path.dirname(here), here))
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    res = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    out = json.loads(res.stdout.strip().splitlines()[-1])
    assert len(out) == 14 and all(ok for ok, _ in out), [(i, detail) for i, (ok, detail) in enumerate(out) if not ok]


# ---------------------------------------------------------------------------------------------------------------------
# 3. the row limit: 2^31 - 1 rows per GPU in one GROUP BY
# ---------------------------------------------------------------------------------------------------------------------
def _for_constant(rows, value):
    """The bit-packed form of a column whose every row is `value`: headers only (bit width 0)."""
    hd = np.zeros((rows + 2047) // 2048, sdb.engine.FOR_BLOCK_DTYPE)
    hd["base"] = value
    return hd, np.zeros(1, np.uint64), rows


WIDE = 2**33 - 1                        # low 32 bits 0xFFFFFFFF: the lo limb gains 2^32 - 1 per row


def _used_gib():
    import torch
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 2**30


def _expect_row_limit(fn):
    with pytest.raises(SdbgError, match="^EUNSUPPORTED"):
        fn()


def test_groupby_row_limit(monkeypatch):
    """One GROUP BY over 2^31 - 1 rows in one key whose values have all-ones low limbs, bit-packed and raw, on the TMA,
    register and hash paths; 2^31 rows are refused on every path and the context answers correctly afterwards.
    Measured on an H100 80GB HBM3 at a 700 W power limit: 43 s, peak device memory in use 37.7 GiB (the raw views of the
    two bit-packed columns, then the two borrowed raw columns: 16 GiB each)."""
    import torch
    t0, peak = time.time(), _used_gib()
    limit = 2**31 - 1
    seg = _segment(limit)
    seg.stage_column_for(1, _for_constant(limit, 7))
    seg.stage_column_for(2, _for_constant(limit, WIDE))
    assert seg.column_packed(2, limit) is not None

    def expect(segs, rows, preds=()):
        got = sdb.IResearchScan(segs).groupby(list(preds), 1, sum_int_field=2)
        assert len(got) == 1 and int(got["key"][0]) == 7 and int(got["count"][0]) == rows
        assert sdb.engine.sum_i128(got)[0] == rows * WIDE

    for env in PATHS:
        _env(monkeypatch, env)
        expect([seg], limit)
        peak = max(peak, _used_gib())
    _env(monkeypatch, {})
    expect([seg], limit, [sdb.pred(2, "GE", WIDE)])
    one = _segment(1)
    one.stage_column(1, np.array([7], np.int64))
    one.stage_column(2, np.array([WIDE], np.int64))
    over = _segment(2**31)
    over.stage_column_for(1, _for_constant(2**31, 7))
    over.stage_column_for(2, _for_constant(2**31, WIDE))
    for env in PATHS:
        _env(monkeypatch, env)
        _expect_row_limit(lambda: sdb.IResearchScan([seg, one]).groupby([], 1, sum_int_field=2))
        _expect_row_limit(lambda: sdb.IResearchScan([over]).groupby([], 1, sum_int_field=2))
    _env(monkeypatch, {})
    seg.close(); over.close()
    expect([one], 1)                                                    # the context still answers
    # raw: borrowed even-length device columns, 2^31 - 2 rows
    rows = 2**31 - 2
    k = torch.full((rows,), 7, dtype=torch.int64, device="cuda")
    v = torch.full((rows,), WIDE, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()                                            # filled before the library reads them
    raw = _segment(rows)
    raw.stage_column_device(1, k.data_ptr(), np.int64, rows)
    raw.stage_column_device(2, v.data_ptr(), np.int64, rows)
    for env in PATHS:
        _env(monkeypatch, env)
        expect([raw], rows)
        peak = max(peak, _used_gib())
        _expect_row_limit(lambda: sdb.IResearchScan([raw, one, one]).groupby([], 1, sum_int_field=2))
    _env(monkeypatch, {})
    raw.close()
    del k, v
    torch.cuda.empty_cache()
    expect([one], 1)
    one.close()
    print("row-limit GROUP BY: %.1f s, peak device memory in use %.1f GiB (%s)"
          % (time.time() - t0, peak, torch.cuda.get_device_name()))
