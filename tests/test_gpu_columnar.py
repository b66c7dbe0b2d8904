"""GPU parity: columnar filter bitmap / COUNT / SUM / GROUP BY through the C ABI vs the CPU oracle."""
import json
import os

import numpy as np
import pytest

import orc
import serenedb_b200 as sdb
from gpu_util import ctx

pytestmark = pytest.mark.gpu
G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bm25_goldens.json")))
K, A, B, V, W = 10, 11, 12, 13, 14


def _table(rows, row0=0):
    cols = {K: orc.synth_column(10, 0, row0, rows), A: orc.synth_column(11, 1, row0, rows),
            B: orc.synth_column(12, 2, row0, rows), V: orc.synth_column(13, 3, row0, rows),
            W: orc.synth_column(14, 4, row0, rows)}
    oseg = orc.Segment(rows, has_wand=False)
    gseg = sdb.Segment(ctx(), rows)
    for f, v in cols.items():
        oseg.add_column(f, v)
        gseg.stage_column(f, v)
    return oseg, gseg, cols


def test_synth_column_kernel_matches_oracle_generator():
    rows = 100_001
    g = sdb.Segment(ctx(), rows)
    import torch
    for field, (stream, kind) in {K: (10, 0), A: (11, 1), B: (12, 2), V: (13, 3), W: (14, 4), 20: (15, 5), 21: (2, 6)}.items():
        g.synth_column(field, stream, kind, 7, rows)
    ctx().sync()
    exp = {K: orc.synth_column(10, 0, 7, rows), B: orc.synth_column(12, 2, 7, rows), W: orc.synth_column(14, 4, 7, rows)}
    # read back through a filter-free count/sum: SUM(int) exact, and bitmaps of thresholds exact
    scan = sdb.IResearchScan([g])
    cnt, si, _ = scan.count_sum([], K)
    assert cnt == rows and si == int(exp[K].sum())
    m = g.filter_bitmap([sdb.pred(B, "LT", 0.25)], rows)
    assert np.array_equal(np.unpackbits(m.view(np.uint8), bitorder="little")[:rows].astype(bool), exp[B] < 0.25)
    m = g.filter_bitmap([sdb.pred(W, "GE", 500.0)], rows)
    assert np.array_equal(np.unpackbits(m.view(np.uint8), bitorder="little")[:rows].astype(bool), exp[W] >= 500.0)


@pytest.mark.parametrize("rows", [1, 2, 63, 64, 65, 1000, 1 << 20, (1 << 20) + 3])
def test_filter_bitmap_and_count_sum(rows):
    """config 1 shape: single filter + COUNT/SUM over int64 and float64 columns; bit-exact bitmaps."""
    oseg, gseg, cols = _table(rows)
    scan = sdb.IResearchScan([gseg])
    for preds_g, preds_o in [([sdb.pred(A, "LT", 250000)], [orc.make_pred(A, "LT", 250000)]),
                             ([sdb.pred(B, "LT", 0.25)], [orc.make_pred(B, "LT", 0.25, is_float=True)]),
                             ([sdb.pred(A, "LT", 500000), sdb.pred(B, "GE", 0.25)],
                              [orc.make_pred(A, "LT", 500000), orc.make_pred(B, "GE", 0.25, is_float=True)]),
                             ([sdb.pred(V, "BETWEEN", -10, 10), sdb.pred(A, "NE", 7), sdb.pred(K, "GT", 100), sdb.pred(W, "LE", 999.0)],
                              [orc.make_pred(V, "BETWEEN", -10, 10), orc.make_pred(A, "NE", 7), orc.make_pred(K, "GT", 100),
                               orc.make_pred(W, "LE", 999.0, is_float=True)])]:
        gm = gseg.filter_bitmap(preds_g, rows)
        om = orc.filter_bitmap(oseg, preds_o, rows)
        assert np.array_equal(gm, om)
        c1, s1, _ = scan.count_sum(preds_g, A)
        c2, s2, _ = orc.filter_count_sum([oseg], preds_o, A)
        assert (c1, s1) == (c2, s2)
        c1, _, f1 = scan.count_sum(preds_g, W)
        c2, _, f2 = orc.filter_count_sum([oseg], preds_o, W)
        assert c1 == c2 and f1 == pytest.approx(f2, rel=1e-9, abs=1e-9)


def test_sum_int64_is_exact_128_bit():
    rows = 300_000
    big = np.full(rows, np.iinfo(np.int64).max - 5, np.int64)
    big[::3] = np.iinfo(np.int64).min + 9
    oseg = orc.Segment(rows, has_wand=False)
    gseg = sdb.Segment(ctx(), rows)
    key = (np.arange(rows) % 7).astype(np.int64)
    for f, v in ((1, big), (2, key)):
        oseg.add_column(f, v)
        gseg.stage_column(f, v)
    scan = sdb.IResearchScan([gseg])
    c, s, _ = scan.count_sum([], 1)
    assert c == rows and s == int(big.astype(object).sum())
    rows_g = scan.groupby([], 2, sum_int_field=1)
    exp = {int(k): int(big[key == k].astype(object).sum()) for k in range(7)}
    assert {int(r["key"]): v for r, v in zip(rows_g, sdb.sum_i128(rows_g))} == exp


def test_scan_10k_goldens_on_gpu():
    segs = []
    for s in range(3):
        x = np.arange(8000 * s, 8000 * (s + 1), dtype=np.int64)
        g = sdb.Segment(ctx(), 8000)
        g.stage_column(1, x)
        if s == 0:
            g.stage_column(3, np.zeros(8000, np.int64), validity=np.zeros(125, np.uint64))
        else:
            g.stage_column(3, x)
        segs.append(g)
    scan = sdb.IResearchScan(segs)
    P = sdb.pred
    assert scan.count_sum([])[0] == 24000
    assert scan.count_sum([P(1, "GE", 20000)])[0] == 4000
    assert scan.count_sum([P(1, "LT", 0)])[0] == 0
    assert scan.count_sum([P(3, "IS_NULL")])[0] == 8000
    assert scan.count_sum([P(3, "IS_NOT_NULL")])[0] == 16000
    assert scan.count_sum([P(1, "BETWEEN", 12000, 12099)], 1)[:2] == (100, 1204950)
    assert scan.count_sum([P(1, "GE", 8000), P(3, "IS_NOT_NULL")])[0] == 16000


@pytest.mark.parametrize("rows", [1000, 2_000_001])
def test_groupby_matches_oracle(rows):
    """config 2 shape: 2 predicates -> GROUP BY k -> COUNT, SUM(v) exact, AVG(w) within 1e-5 rel."""
    oseg, gseg, cols = _table(rows)
    scan = sdb.IResearchScan([gseg])
    gp = [sdb.pred(A, "LT", 500000), sdb.pred(B, "GE", 0.25)]
    op = [orc.make_pred(A, "LT", 500000), orc.make_pred(B, "GE", 0.25, is_float=True)]
    got = scan.groupby(gp, K, sum_int_field=V, avg_f64_field=W, n_groups_hint=100000)
    exp = orc.filter_groupby([oseg], op, K, V, W, cap=100001)
    assert np.array_equal(got["key"], exp["key"])
    assert np.array_equal(got["count"], exp["count"])
    assert np.array_equal(got["sum_lo"], exp["sum_lo"]) and np.array_equal(got["sum_hi"], exp["sum_hi"])
    assert np.array_equal(got["cnt_f64"], exp["cnt_f64"])
    avg_g = got["sum_f64"] / got["cnt_f64"]
    avg_o = exp["sum_f64"] / exp["cnt_f64"]
    assert np.allclose(avg_g, avg_o, rtol=1e-5, atol=0)   # north_star tolerance for AVG
    sel = (cols[A] < 500000) & (cols[B] >= 0.25)
    assert int(got["count"].sum()) == int(sel.sum())


@pytest.mark.parametrize("env", [{"SDBG_GROUPBY_PACKED": "0"}, {}, {"SDBG_GROUPBY_PACK_TABLES_MIN": "2"},
                                 {"SDBG_GROUPBY_PACK_TABLES_MIN": "3"}])
@pytest.mark.parametrize("sum_dtype", [np.int64, np.int32])
def test_groupby_packed_accumulators(env, sum_dtype, monkeypatch):
    """COUNT and SUM(int) sharing one RED word (stats-gated) must give the same result as separate
    accumulators: negative values, several segments of ragged size, 1..3 words per slot."""
    for k_, v_ in env.items():
        monkeypatch.setenv(k_, v_)
    rng = np.random.default_rng(17)
    segs_o, segs_g = [], []
    for rows in (70_001, 513, 1):
        key = rng.integers(-7, 300, size=rows).astype(np.int64)
        v = rng.integers(-1000, 1001, size=rows).astype(sum_dtype)
        a = rng.integers(0, 100, size=rows).astype(np.int32)
        w = rng.random(rows) * 1000.0
        o = orc.Segment(rows, has_wand=False)
        g = sdb.Segment(ctx(), rows)
        for f, vals in {1: key, 2: v, 3: a, 4: w}.items():
            o.add_column(f, vals)
            g.stage_column(f, vals)
        segs_o.append(o)
        segs_g.append(g)
    got = sdb.IResearchScan(segs_g).groupby([sdb.pred(3, "LT", 60)], 1, sum_int_field=2, avg_f64_field=4)
    exp = orc.filter_groupby(segs_o, [orc.make_pred(3, "LT", 60)], 1, 2, 4, cap=1000)
    for f in ("key", "count", "sum_lo", "sum_hi", "cnt_f64"):
        assert np.array_equal(got[f], exp[f]), f
    assert np.allclose(got["sum_f64"], exp["sum_f64"], rtol=1e-9)
    # a constant column (range 0) and a column at the int32 extremes (range 2^32: too wide to pack at scale)
    for lo, hi in ((5, 6), (-2**31, 2**31)):
        rows = 4097
        key = rng.integers(0, 50, size=rows).astype(np.int64)
        v = rng.integers(lo, hi, size=rows).astype(np.int64)
        o = orc.Segment(rows, has_wand=False)
        g = sdb.Segment(ctx(), rows)
        for f, vals in {1: key, 2: v}.items():
            o.add_column(f, vals)
            g.stage_column(f, vals)
        got = sdb.IResearchScan([g]).groupby([], 1, sum_int_field=2)
        exp = orc.filter_groupby([o], [], 1, 2, 999, cap=100)   # 999: no such column = no AVG
        for f in ("key", "count", "sum_lo", "sum_hi"):
            assert np.array_equal(got[f], exp[f]), (f, lo, hi)


@pytest.mark.parametrize("case", ["mixed", "tiny", "nonfinite", "zeros"])
@pytest.mark.parametrize("with_int_sum", [True, False])
def test_groupby_double_sum_edge_values(case, with_int_sum):
    """SUM(double) (one f64 RED per passing row) against the oracle's double sum: negative values, 60 binades of
    dynamic range, denormals, NaN / +-inf, and zeros."""
    rng = np.random.default_rng(23)
    rows = 40_003
    key = rng.integers(0, 97, size=rows).astype(np.int64)
    v = rng.integers(-1000, 1001, size=rows).astype(np.int64)
    if case == "mixed":
        w = rng.standard_normal(rows) * np.exp2(rng.integers(-30, 30, size=rows).astype(np.float64))
    elif case == "tiny":
        w = rng.standard_normal(rows) * 5e-324 * 1000       # denormals
    elif case == "zeros":
        w = np.zeros(rows)
    else:
        w = rng.standard_normal(rows)
        w[5] = np.inf; w[77] = np.nan; w[78] = -np.inf
    o = orc.Segment(rows, has_wand=False)
    g = sdb.Segment(ctx(), rows)
    for f, vals in {1: key, 2: v, 4: w}.items():
        o.add_column(f, vals)
        g.stage_column(f, vals)
    si = 2 if with_int_sum else None
    got = sdb.IResearchScan([g]).groupby([sdb.pred(2, "GE", -900)], 1, sum_int_field=si, avg_f64_field=4)
    exp = orc.filter_groupby([o], [orc.make_pred(2, "GE", -900)], 1, 2 if with_int_sum else 999, 4, cap=1000)
    for f in ("key", "count", "sum_lo", "sum_hi", "cnt_f64"):
        assert np.array_equal(got[f], exp[f]), f
    if case == "nonfinite":
        assert np.array_equal(np.isnan(got["sum_f64"]), np.isnan(exp["sum_f64"]))
        fin = np.isfinite(exp["sum_f64"])
        assert np.array_equal(got["sum_f64"][~fin & ~np.isnan(exp["sum_f64"])], exp["sum_f64"][~fin & ~np.isnan(exp["sum_f64"])])
        assert np.allclose(got["sum_f64"][fin], exp["sum_f64"][fin], rtol=1e-9)
    else:
        # error of either side is bounded by a few ulps of the sum of magnitudes in the group
        scale = np.zeros(len(exp))
        sel = v >= -900
        np.add.at(scale, np.searchsorted(exp["key"], key[sel]), np.abs(w[sel]))
        assert np.all(np.abs(got["sum_f64"] - exp["sum_f64"]) <= 1e-12 * scale)


def test_groupby_nulls_and_multisegment():
    rows = 50_000
    rng = np.random.default_rng(9)
    segs_o, segs_g = [], []
    for s in range(2):
        key = rng.integers(-50, 50, size=rows).astype(np.int64)
        v = rng.integers(-2**40, 2**40, size=rows).astype(np.int64)      # needs two limbs
        w = rng.random(rows)
        vv = rng.integers(0, 2**63, size=(rows + 63) // 64, dtype=np.int64).astype(np.uint64)  # ~half NULL
        wv = rng.integers(0, 2**63, size=(rows + 63) // 64, dtype=np.int64).astype(np.uint64)
        o = orc.Segment(rows, has_wand=False)
        g = sdb.Segment(ctx(), rows)
        for f, (vals, valid) in {1: (key, None), 2: (v, vv), 3: (w, wv)}.items():
            o.add_column(f, vals, valid)
            g.stage_column(f, vals, valid)
        segs_o.append(o)
        segs_g.append(g)
    got = sdb.IResearchScan(segs_g).groupby([sdb.pred(1, "NE", 0)], 1, sum_int_field=2, avg_f64_field=3)
    exp = orc.filter_groupby(segs_o, [orc.make_pred(1, "NE", 0)], 1, 2, 3, cap=1000)
    for f in ("key", "count", "sum_lo", "sum_hi", "cnt_f64"):
        assert np.array_equal(got[f], exp[f]), f
    assert np.allclose(got["sum_f64"], exp["sum_f64"], rtol=1e-9)


def test_groupby_hash_path_wide_keys():
    """Keys spread over the whole int64 range (incl. INT64_MIN, the table's reserved value) take the
    hash-table path; results equal the oracle's hash aggregate."""
    rows = 300_001
    rng = np.random.default_rng(21)
    pool = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, size=5000, dtype=np.int64)
    pool[0] = np.iinfo(np.int64).min
    pool[1] = np.iinfo(np.int64).max
    key = pool[rng.integers(0, len(pool), size=rows)]
    v = rng.integers(-2**45, 2**45, size=rows).astype(np.int64)
    w = rng.random(rows)
    a = rng.integers(0, 100, size=rows).astype(np.int64)
    oseg = orc.Segment(rows, has_wand=False)
    gseg = sdb.Segment(ctx(), rows)
    for f, vals in {1: key, 2: v, 3: w, 4: a}.items():
        oseg.add_column(f, vals)
        gseg.stage_column(f, vals)
    got = sdb.IResearchScan([gseg]).groupby([sdb.pred(4, "LT", 60)], 1, sum_int_field=2, avg_f64_field=3, cap=6000, n_groups_hint=5000)
    exp = orc.filter_groupby([oseg], [orc.make_pred(4, "LT", 60)], 1, 2, 3, cap=6000)
    for f in ("key", "count", "sum_lo", "sum_hi", "cnt_f64"):
        assert np.array_equal(got[f], exp[f]), f
    assert np.allclose(got["sum_f64"], exp["sum_f64"], rtol=1e-9)
    # a too-small hint still works (the table grows and the scan is retried)
    got2 = sdb.IResearchScan([gseg]).groupby([sdb.pred(4, "LT", 60)], 1, sum_int_field=2, avg_f64_field=3, cap=6000, n_groups_hint=1)
    assert np.array_equal(got2["key"], exp["key"]) and np.array_equal(got2["count"], exp["count"])


def test_groupby_reference_goldens_on_gpu():
    """The GROUP BY answers the reference's sqllogic tests hold (tests/golden/groupby_goldens.json: aggregates/index.test,
    query_syntax/groupby/index.test, cookbook/search/faceted-search.test), through the GPU aggregate."""
    G2 = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "groupby_goldens.json")))

    def run(keys, ints=None, floats=None):
        n = len(keys)
        seg = sdb.Segment(ctx(), n)
        seg.stage_column(1, np.asarray(keys, np.int64))
        seg.stage_column(2, np.asarray(ints if ints is not None else [0] * n, np.int64))
        seg.stage_column(3, np.asarray(floats if floats is not None else [0.0] * n, np.float64))
        out = sdb.IResearchScan([seg]).groupby([], 1, sum_int_field=2, avg_f64_field=3)
        seg.close()
        return out

    g = G2["sales_sum_by_region"]
    out = run(g["rows"]["key"], ints=g["rows"]["amount"])
    assert {g["key_names"][int(k)]: int(s) for k, s in zip(out["key"], out["sum_lo"])} == g["expect_sum"]
    g = G2["addresses_count_by_city"]
    out = run(g["rows"]["key"])
    assert {g["key_names"][int(k)]: int(c) for k, c in zip(out["key"], out["count"])} == g["expect_count"]
    g = G2["addresses_avg_income_by_city_street"]
    out = run(g["rows"]["key"], floats=g["rows"]["income"])
    assert {g["key_names"][int(k)]: float(s / c) for k, s, c in zip(out["key"], out["sum_f64"], out["cnt_f64"])} == {k: float(v) for k, v in g["expect_avg"].items()}
    g = G2["products_facets"]
    for col, names, exp in (("category", "category_names", "expect_category"), ("brand", "brand_names", "expect_brand"), ("band", "band_names", "expect_band")):
        out = run(g["rows"][col])
        assert {g[names][int(k)]: int(c) for k, c in zip(out["key"], out["count"])} == g[exp]


def test_zonemaps_skip_dead_blocks_and_keep_results():
    """Per-block min / max verdicts (ColFilterChain::FilterWindow / DeadUntil, table_filter_iterator.cpp:147-286): on a
    clustered column most 2048-row blocks cannot pass a selective range and are never read; results stay those of the
    oracle, and an unclustered column skips nothing."""
    rows = 1_000_000
    rng = np.random.default_rng(11)
    k = rng.integers(0, 1000, rows).astype(np.int64)
    a = (np.arange(rows) // 100).astype(np.int64)            # clustered: 0 .. 9999
    b = rng.random(rows)
    v = rng.integers(-1000, 1001, rows).astype(np.int64)
    w = rng.random(rows) * 1000.0
    oseg = orc.Segment(rows, has_wand=False)
    gseg = sdb.Segment(ctx(), rows)
    for f, arr in {1: k, 2: a, 3: b, 4: v, 5: w}.items():
        oseg.add_column(f, arr)
        gseg.stage_column(f, arr)
    scan = sdb.IResearchScan([gseg])
    cases = [([("LT", 2, 1000)], 0.85), ([("BETWEEN", 2, 5000, 5100)], 0.95), ([("GE", 2, 9990), ("GEF", 3, 0.25)], 0.95),
             ([("NE", 2, 7)], 0.0), ([("GEF", 3, 0.25)], 0.0), ([("EQ", 2, 123456)], 1.0)]
    for spec, min_skipped in cases:
        gp, op = [], []
        for sp in spec:
            if sp[0] == "GEF":
                gp.append(sdb.pred(sp[1], "GE", sp[2])); op.append(orc.make_pred(sp[1], "GE", sp[2], is_float=True))
            elif sp[0] == "BETWEEN":
                gp.append(sdb.pred(sp[1], "BETWEEN", sp[2], sp[3])); op.append(orc.make_pred(sp[1], "BETWEEN", sp[2], sp[3]))
            else:
                gp.append(sdb.pred(sp[1], sp[0], sp[2])); op.append(orc.make_pred(sp[1], sp[0], sp[2]))
        got = scan.groupby(gp, 1, sum_int_field=4, avg_f64_field=5)
        exp = orc.filter_groupby([oseg], op, 1, 4, 5, cap=2000)
        assert len(got) == len(exp)
        for f in ("key", "count", "sum_lo", "sum_hi"):
            assert np.array_equal(got[f], exp[f]), (spec, f)
        if len(exp):
            assert np.allclose(got["sum_f64"], exp["sum_f64"], rtol=1e-9)
        total, skipped = ctx().scan_stats()
        if min_skipped > 0:
            assert total == (rows + 2047) // 2048 and skipped >= min_skipped * total, (spec, total, skipped)
        elif len(exp):
            assert skipped == 0, (spec, skipped)
    gseg.close()


def test_gather_hit_rows():
    """Late materialisation (HitBatcher::MaterializeColumn): projected column values for hit docs only -- int64, float64,
    int32, a nullable column, unsorted / repeated / out-of-range doc ids."""
    rows = 200_000
    rng = np.random.default_rng(3)
    a = rng.integers(-2**40, 2**40, rows).astype(np.int64)
    b = rng.random(rows)
    c32 = rng.integers(-10**6, 10**6, rows).astype(np.int32)
    valid = rng.random(rows) < 0.8
    gseg = sdb.Segment(ctx(), rows)
    gseg.stage_column(1, a)
    gseg.stage_column(2, b)
    gseg.stage_column(3, c32)
    words = np.packbits(np.concatenate([valid, np.zeros((-rows) % 64, bool)]), bitorder="little").view(np.uint64)
    gseg.stage_column(4, a, validity=words)
    docs = np.concatenate([rng.integers(1, rows + 1, 5000), [1, rows, rows, 7, 7]]).astype(np.uint32)
    for f, col, dt in ((1, a, np.int64), (2, b, np.float64), (3, c32, np.int32)):
        v, ok = gseg.gather(f, docs, dt)
        assert ok.all() and np.array_equal(v, col[docs - 1])
    v, ok = gseg.gather(4, docs, np.int64)
    assert np.array_equal(ok, valid[docs - 1]) and np.array_equal(v, np.where(valid[docs - 1], a[docs - 1], 0))
    v, ok = gseg.gather(1, np.array([rows + 5, 3], np.uint32), np.int64)
    assert list(ok) == [False, True] and v[0] == 0 and v[1] == a[2]
    v, ok = gseg.gather(1, np.zeros(0, np.uint32), np.int64)
    assert len(v) == 0
    gseg.close()


def test_bitpacked_int_columns_decode_on_the_gpu():
    """sdbg_stage_column_for: only the packed stream crosses PCIe, the GPU unpacks it into the staged int64 column. The
    staged values equal the raw ones bit for bit, a GROUP BY over packed-staged columns equals the oracle's, and a
    corrupt stream is rejected."""
    rows = 300_001
    rng = np.random.default_rng(9)
    k = rng.integers(0, 5000, rows).astype(np.int64)
    a = (np.arange(rows) // 50).astype(np.int64)
    v = rng.integers(-2**40, 2**40, rows).astype(np.int64)
    w = rng.random(rows) * 100.0
    i64 = np.iinfo(np.int64)
    wild = rng.integers(i64.min, i64.max, rows, dtype=np.int64)
    const = np.full(rows, -12345, np.int64)
    gseg = sdb.Segment(ctx(), rows)
    oseg = orc.Segment(rows, has_wand=False)
    for f, col in {1: k, 2: a, 4: v, 6: wild, 7: const}.items():
        packed = sdb.pack_for(col)
        gseg.stage_column_for(f, packed)
        back = np.zeros(rows, np.int64)
        gseg.column_to_host(f, back.ctypes.data, rows)
        assert np.array_equal(back, col), f
        assert packed[1].nbytes < col.nbytes or f == 6
    gseg.stage_column(5, w)
    for f, col in {1: k, 2: a, 4: v, 5: w}.items():
        oseg.add_column(f, col)
    got = sdb.IResearchScan([gseg]).groupby([sdb.pred(2, "BETWEEN", 1000, 3999)], 1, sum_int_field=4, avg_f64_field=5, cap=6000)
    exp = orc.filter_groupby([oseg], [orc.make_pred(2, "BETWEEN", 1000, 3999)], 1, 4, 5, cap=6000)
    for f in ("key", "count", "sum_lo", "sum_hi", "cnt_f64"):
        assert np.array_equal(got[f], exp[f]), f
    assert np.allclose(got["sum_f64"], exp["sum_f64"], rtol=1e-12)
    h, wd, _ = sdb.pack_for(k)
    bad = h.copy()
    bad["off8"][-1] = len(wd)                    # last group points past the stream
    with pytest.raises(Exception, match="EFORMAT"):
        gseg.stage_column_for(1, (bad, wd, rows))
    gseg.close()
