"""The shipped configuration (block-max pruning level 2: MaxScore demotion, single-list block skip, lead mode with claim
words, conjunctions as lead list + probes) against the exhaustive CPU oracle: identical hits (docs, order, fp32 score
bits), total_matches a lower bound for disjunctions and exact for conjunctions. Also: a scorer whose b differs from
the segment's wand_b must NOT prune (the reference's Scorer::equals gate, reader.hpp:457-501), the kernel switches
(SDBG_STREAM / SDBG_STREAM_LEAD) must not change results, and the NCCL entry points at world size 1."""
import os

import numpy as np
import pytest

import orc
import serenedb_b200 as sdb
from gpu_util import assert_hits_equal, ctx, oracle_terms

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus():
    n = 3_000_000
    g = sdb.Segment(ctx(), n)
    dc, sum_dl = g.synth_corpus(0, 0, 96, threads=8)
    oseg, odc, osdl = orc.synth_segment_mt(n, 0, 96, threads=8)
    assert np.array_equal(dc, odc) and sum_dl == osdl
    nn = orc.synth_column(2, 1, 1, n).astype(np.int32)
    oseg.add_column(9, nn)
    g.stage_column(9, nn)
    return dict(g=g, oseg=oseg, reader=sdb.IndexReader([g], n, sum_dl, dc), dc=dc, n=n)


@pytest.fixture(autouse=True)
def shipped_pruning():
    ctx().set_wand(2)
    yield
    ctx().set_wand(0)
    for k in ("SDBG_STREAM", "SDBG_STREAM_LEAD"):
        os.environ.pop(k, None)


OR_QUERIES = [([81, 1], 100), ([5, 59], 1000), ([0, 1], 10), ([40, 41], 1000), ([0], 10), ([95], 1000), ([0, 1, 2], 100),
              ([3, 40, 70, 90], 500), ([2, 80, 90], 50), ([60, 1], 1000), ([30, 0], 300)]


@pytest.mark.parametrize("tis,k", OR_QUERIES)
def test_disjunctions_pruned_equal_exhaustive(corpus, tis, k):
    scorer = sdb.BM25()
    oh, ototal, _ = orc.bm25_topk([corpus["oseg"]], "OR", oracle_terms(corpus["reader"], scorer, tis), k, mode=1)
    for wand in (2, 0):       # the shipped level, and pruning off (exact total)
        ctx().set_wand(wand)
        hits, total = sdb.ExecuteTopK(corpus["reader"], tis, sdb.OR, scorer, k)
        assert_hits_equal(hits, oh)
        assert total <= ototal if wand else total == ototal


def test_lead_mode_engages_and_matches(corpus):
    """Pairs whose long list's bound lies below a typical posting of the short list: after the first slice the rest of
    the range streams the short list and probes the long one -- far fewer docs are looked at, same hits. A batch so
    that every query is one chain per slice (the bench shape)."""
    scorer = sdb.BM25()
    qs = [[81, 1], [60, 0], [70, 1], [50, 2]] * 16
    h, nn, tot = sdb.ExecuteTopKBatch(corpus["reader"], qs, sdb.OR, scorer, 100)
    ctx().set_wand(0)
    h0, n0, tot0 = sdb.ExecuteTopKBatch(corpus["reader"], qs, sdb.OR, scorer, 100)
    assert np.array_equal(nn, n0) and np.array_equal(h["doc"], h0["doc"]) and np.array_equal(h["score"].view(np.uint32), h0["score"].view(np.uint32))
    assert np.all(tot <= tot0) and tot[:4].sum() < tot0[:4].sum() // 2, (tot[:4], tot0[:4])
    for env in ({"SDBG_STREAM_LEAD": "0"}, {"SDBG_STREAM": "0"}):
        os.environ.update(env)
        ctx().set_wand(2)
        h1, n1, _ = sdb.ExecuteTopKBatch(corpus["reader"], qs, sdb.OR, scorer, 100)
        for k_ in env:
            os.environ.pop(k_)
        assert np.array_equal(n1, n0) and np.array_equal(h1["doc"], h0["doc"]) and np.array_equal(h1["score"].view(np.uint32), h0["score"].view(np.uint32))


@pytest.mark.parametrize("tis,k,with_filter", [([0, 1, 2, 3, 4], 1000, True), ([5, 59], 100, False), ([1, 36, 80], 100, True),
                                               ([0, 95], 10, False), ([0, 1, 2, 3, 4, 5, 6, 7], 100, False),
                                               ([0, 1, 2], 50, False)])
def test_conjunctions_by_probe_exact(corpus, tis, k, with_filter):
    scorer = sdb.BM25()
    fg = sdb.pred(9, "BETWEEN", 250000, 749999) if with_filter else None
    fo = orc.make_pred(9, "BETWEEN", 250000, 749999) if with_filter else None
    oh, ototal, _ = orc.bm25_topk([corpus["oseg"]], "AND", oracle_terms(corpus["reader"], scorer, tis), k, filt=fo, mode=1)
    for wand in (0, 2):       # exact at every pruning level
        ctx().set_wand(wand)
        hits, total = sdb.ExecuteTopK(corpus["reader"], tis, sdb.AND, scorer, k, filt=fg)
        assert_hits_equal(hits, oh)
        assert total == ototal
    os.environ["SDBG_STREAM"] = "0"          # the window kernel's conjunction must agree
    hits2, total2 = sdb.ExecuteTopK(corpus["reader"], tis, sdb.AND, scorer, k, filt=fg)
    os.environ.pop("SDBG_STREAM")
    assert_hits_equal(hits2, oh)
    assert total2 == ototal


def test_filtered_disjunction_and_deleted_docs(corpus):
    scorer = sdb.BM25()
    fg, fo = sdb.pred(9, "BETWEEN", 250000, 749999), orc.make_pred(9, "BETWEEN", 250000, 749999)
    hits, total = sdb.ExecuteTopK(corpus["reader"], [1, 30], sdb.OR, scorer, 200, filt=fg)
    oh, ototal, _ = orc.bm25_topk([corpus["oseg"]], "OR", oracle_terms(corpus["reader"], scorer, [1, 30]), 200, filt=fo, mode=1)
    assert_hits_equal(hits, oh)
    assert total <= ototal
    deleted = np.unique(np.concatenate([oh["doc"][:50], np.arange(1000, 3000, 7, dtype=np.uint32)])).astype(np.uint32)
    corpus["g"].stage_docs_mask(deleted)
    corpus["oseg"].set_docs_mask(deleted)
    try:
        for kind, okind, tis in ((sdb.OR, "OR", [1, 30]), (sdb.AND, "AND", [0, 1, 2]), (sdb.OR, "OR", [0])):
            hits, total = sdb.ExecuteTopK(corpus["reader"], tis, kind, scorer, 100)
            oh2, ototal2, _ = orc.bm25_topk([corpus["oseg"]], okind, oracle_terms(corpus["reader"], scorer, tis), 100, mode=1)
            assert_hits_equal(hits, oh2)
            assert total <= ototal2 if okind == "OR" else total == ototal2
            assert not np.isin(hits["doc"], deleted).any()
    finally:
        corpus["g"].stage_docs_mask(np.zeros(0, np.uint32))
        corpus["oseg"].set_docs_mask(np.zeros(0, np.uint32))


def test_other_b_never_prunes(corpus):
    """The block-max pairs were chosen for b = 0.75: BM25(1.2, 0.5) gets bounds that are not upper bounds, so pruning has
    to stay off for it (exact totals prove nothing was skipped), as the reference's Scorer::equals check does."""
    scorer = sdb.BM25(1.2, 0.5)
    for tis, k in (([0], 10), ([81, 1], 100), ([0, 1, 2], 100)):
        hits, total = sdb.ExecuteTopK(corpus["reader"], tis, sdb.OR, scorer, k)
        oh, ototal, _ = orc.bm25_topk([corpus["oseg"]], "OR", oracle_terms(corpus["reader"], scorer, tis), k, mode=1, b=0.5)
        assert_hits_equal(hits, oh)
        assert total == ototal


def test_collectives_at_world_size_one(corpus):
    """sdbg_dist_* with a one-rank communicator: the merged GROUP BY partials and the distributed top-k equal the local
    results (the N > 1 path is the same code with more ranks: bench.py --gpus N)."""
    import torch
    c = sdb.Context(0)
    try:
        c.dist_init(sdb.Context.dist_unique_id(), 0, 1)
    except Exception as e:   # no NCCL library on this box
        pytest.skip("NCCL not available: %s" % e)
    rows = 500_000
    seg = sdb.Segment(c, rows)
    for f, (stream, kind) in {10: (10, 0), 11: (11, 1), 12: (12, 2), 13: (13, 3), 14: (14, 4)}.items():
        seg.synth_column(f, stream, kind, 0, rows)
    scan = sdb.IResearchScan([seg])
    preds = [sdb.pred(11, "LT", 500000), sdb.pred(12, "GE", 0.25)]
    span = 100000
    d_i64 = torch.zeros(4 * span, dtype=torch.int64, device="cuda:0")
    d_f64 = torch.zeros(span, dtype=torch.float64, device="cuda:0")
    scan.groupby_partial(preds, 10, 0, span, 13, 14, d_i64.data_ptr(), d_f64.data_ptr())
    c.sync()
    before_i, before_f = d_i64.clone(), d_f64.clone()
    c.dist_groupby_merge(d_i64.data_ptr(), d_f64.data_ptr(), span, 1000.0 * rows)
    c.sync()
    total_before = before_i[span:2 * span] + (before_i[2 * span:3 * span] << 32)
    total_after = d_i64[span:2 * span] + (d_i64[2 * span:3 * span] << 32)
    assert torch.equal(before_i[:span], d_i64[:span]) and torch.equal(total_before, total_after) and torch.equal(before_i[3 * span:], d_i64[3 * span:])
    assert torch.equal(before_f, d_f64)          # 120-bit fixed point round trip of a double is exact
    n = 400_000
    g = sdb.Segment(c, n)
    dc, sum_dl = g.synth_corpus(0, 0, 32, threads=8)
    reader = sdb.IndexReader([g], n, sum_dl, dc)
    qs = [[0, 5], [3], [1, 20, 30]]
    batch = sdb.PreparedBatch(reader, qs, sdb.OR, sdb.BM25(), 50)
    hd, nd = batch.run_dist()
    hl, nl, _ = batch.run_host()
    assert np.array_equal(nd, nl) and np.array_equal(hd["doc"], hl["doc"]) and np.array_equal(hd["score"].view(np.uint32), hl["score"].view(np.uint32))
    seg.close(); g.close(); c.close()
