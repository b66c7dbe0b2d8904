"""Bit-packed int64 columns in HBM: the device packer writes sdbg_pack_for's bytes, the GROUP BY scan over packed columns
equals the same values staged as borrowed raw device columns, every other reader sees the raw values, and columns whose
packed form is not smaller stay raw."""
import numpy as np
import pytest

import serenedb_b200 as sdb
from gpu_util import ctx

pytestmark = pytest.mark.gpu

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


def widths_column(rows, widths, seed, base0=-1_000_003):
    """int64 values whose 2048-row group g has bit width widths[g % len(widths)] exactly and a negative base."""
    rng = np.random.default_rng(seed)
    out = np.empty(rows, np.int64)
    for g in range((rows + 2047) // 2048):
        r0, r1 = g * 2048, min(rows, g * 2048 + 2048)
        w = widths[g % len(widths)]
        if w == 64:
            v = rng.integers(INT64_MIN, INT64_MAX, r1 - r0, dtype=np.int64, endpoint=True)
            v[0], v[-1] = INT64_MIN, INT64_MAX
        else:
            base = base0 * (g + 1) if w < 40 else INT64_MIN + g
            hi = (1 << w) - 1
            d = rng.integers(0, hi, r1 - r0, dtype=np.uint64, endpoint=True) if w else np.zeros(r1 - r0, np.uint64)
            d[0], d[-1] = 0, hi
            v = (np.uint64(base & (2**64 - 1)) + d).view(np.int64)
        out[r0:r1] = v
    return out


def test_device_packer_writes_the_host_writers_bytes():
    rows = 2048 * 65 + 777                       # every width 0..64 once, then a partial group
    vals = widths_column(rows, list(range(65)) + [3], seed=1)
    seg = sdb.Segment(ctx(), rows)
    seg.stage_column(1, vals)
    got = seg.column_packed(1, rows)
    assert got is not None
    hd, wd, _ = sdb.pack_for(vals)
    assert np.array_equal(got[0], hd) and np.array_equal(got[1], wd)
    assert all(int(h) % 2 == 0 for h in got[0]["off8"])          # every group 16-byte aligned
    out = np.zeros(rows, np.int64)
    seg.column_to_host(1, out.ctypes.data, rows)
    assert np.array_equal(out, vals)
    seg.close()


def test_wide_columns_stay_raw():
    rows = 10_000
    seg = sdb.Segment(ctx(), rows)
    seg.synth_column(1, 5, 5, 0, rows)                           # full 64-bit hashes
    seg.stage_column(2, np.random.default_rng(2).integers(INT64_MIN, INT64_MAX, rows, dtype=np.int64))
    seg.stage_column(3, np.arange(rows, dtype=np.int64))          # 11 bits: packed
    seg.stage_column(4, np.arange(rows, dtype=np.int32))          # int32: raw
    assert seg.column_packed(1, rows) is None and seg.column_packed(2, rows) is None and seg.column_packed(4, rows) is None
    assert seg.column_packed(3, rows) is not None
    seg.close()


def _tables(sizes, kw, aw, vw, seed):
    """(packed segments, borrowed raw segments, host columns) of k, a, v (int64 of the given widths), b (float64)."""
    import torch
    packed, raw, host, keep = [], [], [], []
    for i, rows in enumerate(sizes):
        rng = np.random.default_rng(seed + i)
        cols = {1: widths_column(rows, kw, seed + 10 * i, base0=-7) if kw != [None] else rng.integers(-50, 50, rows).astype(np.int64),
                2: widths_column(rows, aw, seed + 10 * i + 1),
                3: rng.random(rows),
                4: widths_column(rows, vw, seed + 10 * i + 2)}
        ps, rs = sdb.Segment(ctx(), rows), sdb.Segment(ctx(), rows)
        for f, v in cols.items():
            ps.stage_column(f, v)
            t = torch.from_numpy(v).cuda()
            keep.append(t)
            rs.stage_column_device(f, t.data_ptr(), v.dtype, rows)
        packed.append(ps); raw.append(rs); host.append(cols)
    return packed, raw, host, keep


def _same_groups(a, b):
    for f in ("key", "count", "sum_lo", "sum_hi", "cnt_f64"):
        assert np.array_equal(a[f], b[f]), f
    assert np.allclose(a["sum_f64"], b["sum_f64"], rtol=1e-12, atol=1e-9)


SIZES = [70_002, 514, 2]
WIDTHS = [([0, 5, 9], [0, 1, 17, 20, 33], [11, 0, 31]),      # narrow sums: packed accumulators
          ([12], [64, 40, 63, 2], [0, 37, 64, 1]),            # wide predicate and sum columns (two-limb sums)
          ([None], [31, 32], [62])]


@pytest.mark.parametrize("kw,aw,vw", WIDTHS)
def test_groupby_over_packed_equals_raw(kw, aw, vw):
    packed, raw, host, keep = _tables(SIZES, kw, aw, vw, seed=len(kw) + len(aw))
    assert packed[0].column_packed(2, SIZES[0]) is not None or 64 in aw
    a_all = np.concatenate([h[2] for h in host])
    q = [int(x) for x in np.quantile(a_all, [0.2, 0.5, 0.8], method="nearest")]
    cases = [[sdb.pred(2, "LT", q[1])], [sdb.pred(2, "LE", q[0]), sdb.pred(3, "GE", 0.25)], [sdb.pred(2, "GT", q[2])],
             [sdb.pred(2, "GE", q[0])], [sdb.pred(2, "EQ", int(a_all[5]))], [sdb.pred(2, "NE", int(a_all[5]))],
             [sdb.pred(2, "BETWEEN", q[0], q[2]), sdb.pred(4, "NE", int(host[0][4][0]))], []]
    for preds in cases:
        got = sdb.IResearchScan(packed).groupby(preds, 1, sum_int_field=4, avg_f64_field=3)
        exp = sdb.IResearchScan(raw).groupby(preds, 1, sum_int_field=4, avg_f64_field=3)
        _same_groups(got, exp)
        for seg_p, seg_r in zip(packed, raw):     # one segment at a time as well
            _same_groups(sdb.IResearchScan([seg_p]).groupby(preds, 1, sum_int_field=4, avg_f64_field=3),
                         sdb.IResearchScan([seg_r]).groupby(preds, 1, sum_int_field=4, avg_f64_field=3))
    for s in packed + raw:
        s.close()
    del keep


def test_out_of_range_keys_fail_alike():
    import torch
    packed, raw, host, keep = _tables([70_002], [9], [20], [11], seed=5)
    kmin = int(host[0][1].min())
    d_i64 = torch.zeros(4 * 100, dtype=torch.int64, device="cuda")
    d_f64 = torch.zeros(100, dtype=torch.float64, device="cuda")
    for segs in (packed, raw):
        scan = sdb.IResearchScan(segs)
        scan.groupby_partial([sdb.pred(2, "GE", 0)], 1, kmin, 100, 4, 3, d_i64.data_ptr(), d_f64.data_ptr())
        with pytest.raises(Exception):
            scan.groupby_finalize(kmin, 100, d_i64.data_ptr(), d_f64.data_ptr(), 100)
    for s in packed + raw:
        s.close()


def test_zonemap_scan_stats_match_raw():
    import torch
    rows = 1_000_002
    ts = (np.arange(rows) // 100).astype(np.int64)              # clustered: 5 bits per group
    k = (np.arange(rows) * 7919 % 1000).astype(np.int64)
    w = np.random.default_rng(9).random(rows)
    p, r = sdb.Segment(ctx(), rows), sdb.Segment(ctx(), rows)
    keep = []
    for f, v in ((1, k), (2, ts), (3, w)):
        p.stage_column(f, v)
        t = torch.from_numpy(v).cuda()
        keep.append(t)
        r.stage_column_device(f, t.data_ptr(), v.dtype, rows)
    assert p.column_packed(2, rows) is not None
    preds = [sdb.pred(2, "BETWEEN", 2000, 2099)]
    got = sdb.IResearchScan([p]).groupby(preds, 1, avg_f64_field=3)
    st_p = ctx().scan_stats()
    exp = sdb.IResearchScan([r]).groupby(preds, 1, avg_f64_field=3)
    st_r = ctx().scan_stats()
    _same_groups(got, exp)
    assert st_p == st_r and st_p[1] > 0.9 * st_p[0]
    p.close(); r.close()


def test_raw_view_readers_see_the_values():
    rows = 100_000
    vals = widths_column(rows, [7, 0, 19], seed=4)
    b = np.random.default_rng(4).random(rows)
    seg = sdb.Segment(ctx(), rows)
    seg.stage_column(1, vals)
    seg.stage_column(2, b)
    assert seg.column_packed(1, rows) is not None
    docs = np.random.default_rng(5).integers(1, rows + 1, 3000).astype(np.uint32)
    v, ok = seg.gather(1, docs, np.int64)
    assert ok.all() and np.array_equal(v, vals[docs - 1])
    scan = sdb.IResearchScan([seg])
    lo = int(np.median(vals))
    cnt, s, _ = scan.count_sum([sdb.pred(1, "LT", lo)], 1)
    assert cnt == int((vals < lo).sum()) and s == int(vals[vals < lo].sum())
    mask = seg.filter_bitmap([sdb.pred(1, "GE", lo)])
    bits = np.unpackbits(mask.view(np.uint8), bitorder="little")[:rows].astype(bool)
    assert np.array_equal(bits, vals >= lo)
    ptr, n = seg.column_device_ptr(1)                             # the raw view, decoded once
    seg.stage_column_device(9, ptr, np.int64, n)
    out = np.zeros(rows, np.int64)
    seg.column_to_host(9, out.ctypes.data, rows)
    assert np.array_equal(out, vals)
    assert seg.column_minmax(1) == (int(vals.min()), int(vals.max()))
    seg.close()


def test_hash_groupby_over_packed_columns(monkeypatch):
    rows = 50_000
    rng = np.random.default_rng(6)
    key = (rng.integers(0, 3000, rows) * 10**9).astype(np.int64)      # too wide for the dense table
    v = rng.integers(-1000, 1000, rows).astype(np.int64)
    seg = sdb.Segment(ctx(), rows)
    seg.stage_column(1, key)
    seg.stage_column(2, v)
    assert seg.column_packed(2, rows) is not None
    got = sdb.IResearchScan([seg]).groupby([sdb.pred(2, "GT", 0)], 1, sum_int_field=2)
    sel = v > 0
    uk = np.unique(key[sel])
    assert np.array_equal(got["key"], uk)
    assert np.array_equal(got["count"], [int((key[sel] == x).sum()) for x in uk])
    tot = sdb.engine.sum_i128(got)
    assert tot == [int(v[sel][key[sel] == x].sum()) for x in uk]
    seg.close()


def test_bm25_filter_on_packed_int64_column():
    import orc
    from gpu_util import assert_hits_equal, oracle_terms, to_gpu
    n = 50_000
    oseg, dl, lists = orc.synth_segment(n, [5, 40, 0])
    col = widths_column(n, [12, 3], seed=8)
    g_packed = to_gpu(oseg, columns={7: (col, None)})
    assert g_packed.column_packed(7, n) is not None
    scorer = sdb.BM25()
    reader = sdb.IndexReader([g_packed], n, int(dl.sum()), [len(d) for d, _ in lists])
    lo, hi = int(np.quantile(col, 0.3)), int(np.quantile(col, 0.7))
    hits, total = sdb.ExecuteTopK(reader, [0, 1], sdb.OR, scorer, 100, filt=sdb.pred(7, "BETWEEN", lo, hi))
    oseg.add_column(7, col)
    oh, ototal, _ = orc.bm25_topk([oseg], "OR", oracle_terms(reader, scorer, [0, 1]), 100, mode=1,
                                 filt=orc.make_pred(7, "BETWEEN", lo, hi))
    assert_hits_equal(hits, oh)
    assert total == ototal
    g_packed.close()


def _kernels_of(fn):
    """Names of the CUDA kernels `fn` launches (torch.profiler with CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        ctx().sync()
    return [e.name for e in prof.events() if e.device_type.name == "CUDA"]


def test_groupby_reads_the_packed_words():
    """The TMA GROUP BY over packed columns runs the kFor instantiation and never decodes a raw view."""
    packed, raw, host, keep = _tables([70_002], [9], [20], [11], seed=7)
    preds = [sdb.pred(2, "LT", int(np.median(host[0][2])))]
    names = _kernels_of(lambda: sdb.IResearchScan(packed).groupby(preds, 1, sum_int_field=4, avg_f64_field=3))
    tma = [n for n in names if "filter_groupby_tma_kernel" in n]
    assert tma and all(n.replace(" ", "").split("(")[0].endswith(",true>") for n in tma), tma
    assert not any("for_unpack_kernel" in n for n in names)
    names = _kernels_of(lambda: sdb.IResearchScan(raw).groupby(preds, 1, sum_int_field=4, avg_f64_field=3))
    assert not any(n.replace(" ", "").split("(")[0].endswith(",true>") for n in names if "filter_groupby_tma_kernel" in n)
    for s in packed + raw:
        s.close()


def test_stage_column_for_keeps_aligned_streams_and_decodes_the_rest():
    rows = 70_001
    vals = widths_column(rows, [13, 0, 33, 5], seed=11)
    hd, wd, _ = sdb.pack_for(vals)
    seg = sdb.Segment(ctx(), rows)
    seg.stage_column_for(1, (hd, wd, rows))
    got = seg.column_packed(1, rows)
    assert got is not None and np.array_equal(got[0], hd) and np.array_equal(got[1], wd)
    # the same values with every group one word further: odd word offsets are not 16-byte aligned -> decoded to raw
    hd2 = hd.copy()
    hd2["off8"] += 1
    wd2 = np.concatenate([np.zeros(1, np.uint64), wd])
    seg.stage_column_for(2, (hd2, wd2, rows))
    assert seg.column_packed(2, rows) is None
    for f in (1, 2):
        out = np.zeros(rows, np.int64)
        seg.column_to_host(f, out.ctypes.data, rows)
        assert np.array_equal(out, vals)
    seg.stage_column(3, np.random.default_rng(1).random(rows))
    lo = int(np.quantile(vals, 0.4))
    g1 = sdb.IResearchScan([seg]).groupby([sdb.pred(1, "GE", lo)], 1, avg_f64_field=3)
    seg.stage_column(4, vals)
    g2 = sdb.IResearchScan([seg]).groupby([sdb.pred(2, "GE", lo)], 4, avg_f64_field=3)
    _same_groups(g1, g2)
    seg.close()


@pytest.mark.parametrize("dtype", [np.int32, np.float64, np.int64])
def test_zonemaps_follow_restaged_values(dtype):
    """Restaging a column with new values of the same shape must not leave the old zonemap's skip verdicts behind."""
    rows = 400_000
    asc = (np.arange(rows) // 100).astype(dtype)
    seg = sdb.Segment(ctx(), rows)
    seg.stage_column(1, np.zeros(rows, np.int64))
    lo, hi = (2000, 2099) if dtype != np.float64 else (2000.0, 2099.0)
    preds = [sdb.pred(2, "BETWEEN", lo, hi)]
    for vals in (asc, asc[::-1].copy()):
        seg.stage_column(2, vals)
        got = sdb.IResearchScan([seg]).groupby(preds, 1)
        assert int(got["count"].sum()) == int(((vals >= lo) & (vals <= hi)).sum()) == 10_000
        total, skipped = ctx().scan_stats()
        assert skipped >= total - 8                                 # only the blocks that hold 2000..2099 are read
    seg.close()
