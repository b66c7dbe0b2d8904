"""The multi-GPU merges (DESIGN §5) against exact references, with R ranks simulated on one GPU.

Top-k: each rank is its own list of segments with an IndexReader that carries the corpus-wide statistics (what
dist.global_term_stats gives every rank). PreparedBatch.run_device writes rank r's keys into keys_all[r] and
merge_gathered selects the global top-k from them, as sdbg_dist_bm25_topk_batch does after its all-gather. Crafted keys
check the merge kernel against dist.select_topk_host bit for bit; real per-rank scans check the whole path against the
oracle on the unsharded corpus, including queries with fewer than k matches in all.

GROUP BY: sdbg_dist_groupby_merge with a one-rank NCCL communicator. The pack, all-reduce and unpack run there as they
do at N ranks; its results are checked against fractions.Fraction arithmetic and against the local GROUP BY."""
import math
from fractions import Fraction

import numpy as np
import pytest

import orc
import serenedb_b200 as sdb
from gpu_util import ctx, oracle_terms, to_gpu
from serenedb_b200 import dist
from serenedb_b200._native import SdbgError
from shape_corpora import Corpus, natural_segments, uniform_segments

pytestmark = pytest.mark.gpu

RANK_BITS = dist.RANK_SLOT_BITS
MAX_FINITE_F32 = 0x7F7FFFFF      # score bits of the largest finite float
MIN_DENORMAL_F32 = 0x00000001    # score bits of the smallest positive denormal


def _cuda(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()      # the library works on its own non-blocking stream
    return t


def _zeros(*shape):
    import torch
    t = torch.zeros(shape, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    return t


def _assert_merge_equals_host(keys_all, k):
    """merge_gathered of [R, nq, k] uint64 keys against dist.select_topk_host: n_out, then each hit's key, score bits,
    rank and ordinal bit for bit."""
    R, nq, _ = keys_all.shape
    hits, n_out = sdb.merge_gathered(ctx(), _cuda(keys_all.view(np.int64)).data_ptr(), R, nq, k)
    ref = dist.select_topk_host(keys_all.view(np.int64), R, nq, k)
    m32 = np.uint64(0xFFFFFFFF)
    for q in range(nq):
        want, h = ref[q], hits[q, :n_out[q]]
        assert n_out[q] == len(want), (q, int(n_out[q]), len(want))
        ordinal = ~want & m32
        assert np.array_equal(h["score"].view(np.uint32), (want >> np.uint64(32)).astype(np.uint32)), q
        assert np.array_equal(h["seg"], (ordinal >> np.uint64(RANK_BITS)).astype(np.uint32)), q
        assert np.array_equal(h["doc"], (ordinal & np.uint64((1 << RANK_BITS) - 1)).astype(np.uint32)), q
        got_ord = (h["seg"].astype(np.uint64) << np.uint64(RANK_BITS)) | h["doc"].astype(np.uint64)
        got = (h["score"].view(np.uint32).astype(np.uint64) << np.uint64(32)) | (~got_ord & m32)
        assert np.array_equal(got, want), q
    return n_out


# ---------------------------------------------------------------- (a) merge kernel on crafted keys
def _crafted_keys(rng, R, nq, k, counts):
    """[R, nq, k] uint64: list (r, q) holds counts[r, q] unique keys sorted descending, then zeros. Ordinals are
    rank << 28 | doc with distinct docs per list; half of the scores come from a small per-query pool (ties across and
    within ranks, broken by rank, then doc) that holds the smallest denormal and the largest finite float."""
    pool = rng.integers(0x00800000, MAX_FINITE_F32, size=(1, nq, 6), dtype=np.int64).astype(np.uint64)
    pool[..., 0], pool[..., 1] = MIN_DENORMAL_F32, MAX_FINITE_F32
    pick = np.take_along_axis(np.broadcast_to(pool, (R, nq, 6)), rng.integers(0, 6, size=(R, nq, k)), axis=2)
    free = rng.integers(1, MAX_FINITE_F32 + 1, size=(R, nq, k), dtype=np.int64).astype(np.uint64)
    score = np.where(rng.random((R, nq, k)) < 0.5, pick, free)
    doc = np.cumsum(rng.integers(1, 1 << 15, size=(R, nq, k), dtype=np.int64), axis=2).astype(np.uint64)   # < 2^28, distinct
    ordinal = (np.arange(R, dtype=np.uint64)[:, None, None] << np.uint64(RANK_BITS)) | doc
    keys = (score << np.uint64(32)) | (~ordinal & np.uint64(0xFFFFFFFF))
    keys[np.arange(k)[None, None, :] >= counts[:, :, None]] = 0
    return np.sort(keys, axis=2)[:, :, ::-1].copy()


@pytest.mark.parametrize("nq", [1, 7, 300])
@pytest.mark.parametrize("k", [1, 10, 1000, 3072, 4096, 8192])
@pytest.mark.parametrize("R", [1, 2, 3, 8, 15])
def test_merge_crafted_keys(R, k, nq):
    rng = np.random.default_rng(R * 100003 + k * 31 + nq)
    sizes = np.array(sorted({0, 1, k // 3, k - 1, k}))
    counts = sizes[rng.integers(0, len(sizes), size=(R, nq))]
    if nq >= 7:
        counts[:, 0] = 0                                  # a query no rank matched
        counts[:, 1] = k                                  # every rank full
        counts[:, 2] = np.where(np.arange(R) == R - 1, k, 0)   # one full rank, the last
        counts[:, 3] = max(k // (2 * R), 1)               # under k in all (R * k may still fill the merge buffer)
        counts[:, 4] = 1
    _assert_merge_equals_host(_crafted_keys(rng, R, nq, k, counts), k)


@pytest.mark.parametrize("R,k,per_rank", [(2, 8192, [300, 300]), (8, 1000, [100] * 8), (3, 4096, [1365, 1365, 0]),
                                          (15, 1000, [60] * 15), (8, 3072, [1000, 0, 1, 500, 0, 700, 1, 0]),
                                          (2, 8192, [8191, 0]), (2, 8192, [0, 8191]), (4, 1000, [999, 0, 0, 0]),
                                          (2, 10, [2, 2]), (3, 1000, [10, 10, 10])])
def test_merge_fewer_than_k_in_all(R, k, per_rank):
    """Fewer than k keys over all ranks: every rank's keys must come back, none lost behind another rank's zero tail --
    whether R * k fills the merge buffer (cap = max(next_pow2(k + 1024), 4096)) or only exceeds k, so that the final
    select finds fewer than k keys."""
    nq = 7
    rng = np.random.default_rng(k + R)
    counts = np.repeat(np.asarray(per_rank)[:, None], nq, axis=1)
    n_out = _assert_merge_equals_host(_crafted_keys(rng, R, nq, k, counts), k)
    assert np.all(n_out == min(sum(per_rank), k))


def test_merge_threaded_host_conversion():
    """nq * k >= 131072: the keys are turned into hits by several host threads."""
    R, k, nq = 3, 2048, 96
    assert nq * k >= 131072
    rng = np.random.default_rng(7)
    counts = rng.choice(np.array([0, 5, 700, k]), size=(R, nq))
    _assert_merge_equals_host(_crafted_keys(rng, R, nq, k, counts), k)


# ---------------------------------------------------------------- (b) real per-rank scans against the oracle
FILTER_FIELD = 9
FILTER_LO, FILTER_HI = 20, 59


def _ranked(corpus, ranks, filter_values):
    """ranks: the corpus segments of each rank (in corpus order). Every segment gets the filter column."""
    for o, v in zip(corpus.osegs, filter_values):
        o.add_column(FILTER_FIELD, v)
    gsegs = [to_gpu(o, columns={FILTER_FIELD: (v, None)}) for o, v in zip(corpus.osegs, filter_values)]
    readers = [sdb.IndexReader([gsegs[j] for j in rk], corpus.docs_with_field, corpus.total_term_freq, corpus.docs_with_term)
               for rk in ranks]
    bases = [np.cumsum([0] + [corpus.osegs[j].n_docs for j in rk])[:-1] for rk in ranks]
    one = sdb.IndexReader(gsegs, corpus.docs_with_field, corpus.total_term_freq, corpus.docs_with_term)
    return dict(corpus=corpus, ranks=ranks, readers=readers, bases=bases, one=one, gsegs=gsegs)


def _filter_values(rng, osegs, fail_all=()):
    return [np.full(o.n_docs, 1000, np.int64) if i in fail_all else rng.integers(0, 100, o.n_docs).astype(np.int64)
            for i, o in enumerate(osegs)]


@pytest.fixture(scope="module")
def uniform8():
    """8 ranks of one segment each; term 5 (p = 0.005) matches about 600 docs in all."""
    _, parts, _ = uniform_segments(parts=8)
    corpus = Corpus(parts)
    return _ranked(corpus, [[j] for j in range(8)], _filter_values(np.random.default_rng(1), corpus.osegs))


@pytest.fixture(scope="module")
def natural3():
    """rank 0: segments 0 + 1 (ordinals cross a segment base), rank 1: segment 2, rank 2: a segment where the queried
    terms have no postings (only term 10, never queried, has any) and every doc fails the filter."""
    segs = natural_segments()
    rng = np.random.default_rng(3)
    n = 2000
    empty = [(np.zeros(0, np.uint32), np.zeros(0, np.uint32))] * 10
    extra = np.sort(rng.choice(np.arange(1, n + 1), 50, replace=False)).astype(np.uint32)
    segs.append((rng.integers(5, 50, n).astype(np.uint32), empty + [(extra, np.ones(50, np.uint32))]))
    corpus = Corpus(segs)
    return _ranked(corpus, [[0, 1], [2], [3]], _filter_values(rng, corpus.osegs, fail_all=(3,)))


def _to_global(env, hits):
    """(rank, ordinal within the rank) -> (corpus segment, doc)."""
    seg = np.zeros(len(hits), np.uint32)
    doc = np.zeros(len(hits), np.uint32)
    for i, h in enumerate(hits):
        r, o = int(h["seg"]), int(h["doc"])
        b = env["bases"][r]
        j = int(np.searchsorted(b, o - 1, side="right")) - 1
        seg[i], doc[i] = env["ranks"][r][j], o - int(b[j])
    return seg, doc


def _run_ranks(env, queries, kind, k, filt, thr):
    R, nq = len(env["readers"]), len(queries)
    keys, totals = _zeros(R, nq, k), _zeros(R, nq)
    for r, reader in enumerate(env["readers"]):
        sdb.PreparedBatch(reader, queries, kind, sdb.BM25(), k, filt=filt, threshold=thr).run_device(
            r, keys[r].data_ptr(), totals[r].data_ptr())
    hits, n_out = sdb.merge_gathered(ctx(), keys.data_ptr(), R, nq, k)
    return hits, n_out, totals.cpu().numpy().sum(axis=0)


def _check_queries(env, queries, kind, k, level, with_filter=False, thr=None):
    okind = "AND" if kind == sdb.AND else "OR"
    fg = sdb.pred(FILTER_FIELD, "BETWEEN", FILTER_LO, FILTER_HI) if with_filter else None
    fo = orc.make_pred(FILTER_FIELD, "BETWEEN", FILTER_LO, FILTER_HI) if with_filter else None
    hits, n_out, total = _run_ranks(env, queries, kind, k, fg, sdb.FLT_MIN if thr is None else thr)
    for q, tis in enumerate(queries):
        kw = {} if thr is None else dict(threshold_in=np.float32(thr))
        oh, ototal, _ = orc.bm25_topk(env["corpus"].osegs, okind, oracle_terms(env["readers"][0], sdb.BM25(), tis), k,
                                      filt=fo, mode=1, **kw)
        h = hits[q, :n_out[q]]
        assert len(h) == len(oh), (tis, okind, k, len(h), len(oh))
        seg, doc = _to_global(env, h)
        assert np.array_equal(seg, oh["seg"]) and np.array_equal(doc, oh["doc"]), (tis, okind, k)
        assert np.array_equal(h["score"].view(np.uint32), oh["score"].view(np.uint32)), (tis, okind, k)
        if level == 0 and thr is None:
            assert total[q] == ototal, (tis, okind, k)
        else:
            assert total[q] <= ototal if okind == "OR" else total[q] == ototal, (tis, okind, k)
    return hits, n_out


def _seed(env, tis, kind):
    """A threshold between the oracle's 20th and 21st best scores: the scans start above most of the matches."""
    oh, _, _ = orc.bm25_topk(env["corpus"].osegs, "AND" if kind == sdb.AND else "OR",
                             oracle_terms(env["readers"][0], sdb.BM25(), tis), 50, mode=1)
    assert len(oh) > 21
    return float(np.float32((float(oh["score"][20]) + float(oh["score"][21])) / 2))


SINGLE = {"uniform8": [([5], sdb.OR), ([5, 3], sdb.OR), ([0, 4], sdb.AND), ([1, 5], sdb.AND), ([0, 1, 2, 3, 4, 5], sdb.OR)],
          "natural3": [([9], sdb.OR), ([6, 9], sdb.OR), ([0, 1], sdb.AND), ([3, 4, 5], sdb.OR), ([0, 7, 2], sdb.AND)]}
SEEDED = {"uniform8": [([0, 1], sdb.OR), ([0, 4], sdb.AND)], "natural3": [([0, 7], sdb.OR), ([0, 8], sdb.AND)]}


@pytest.fixture(params=[0, 1, 2], ids=lambda v: f"wand{v}")
def level(request):
    ctx().set_wand(request.param)
    yield request.param
    ctx().set_wand(0)


@pytest.mark.parametrize("k", [1, 10, 1000, 8192])
@pytest.mark.parametrize("corpus_name", ["uniform8", "natural3"])
def test_ranks_equal_unsharded_oracle(request, corpus_name, k, level):
    env = request.getfixturevalue(corpus_name)
    for tis, kind in SINGLE[corpus_name]:
        for with_filter in (False, True):
            _check_queries(env, [tis], kind, k, level, with_filter=with_filter)
    for tis, kind in SEEDED[corpus_name]:
        _check_queries(env, [tis], kind, k, level, thr=_seed(env, tis, kind))
    if corpus_name == "uniform8" and k == 1000:    # ~600 matches in all, 8 ranks: the merge buffer fills with zero tails
        hits, n_out = _check_queries(env, [[5]], sdb.OR, k, level)
        assert 0 < n_out[0] < k and len(set(hits["seg"][0, :n_out[0]].tolist())) == 8


@pytest.mark.parametrize("k", [10, 1000])
@pytest.mark.parametrize("corpus_name", ["uniform8", "natural3"])
def test_ranks_batch_equal_unsharded_oracle(request, corpus_name, k, level):
    env = request.getfixturevalue(corpus_name)
    rng = np.random.default_rng(k + level)
    n_terms = env["corpus"].n_terms
    queries = [sorted(int(t) for t in rng.choice(n_terms, size=int(rng.integers(1, 5)), replace=False)) for _ in range(64)]
    _check_queries(env, queries, sdb.OR, k, level)
    _check_queries(env, queries, sdb.AND, k, level, with_filter=True)


@pytest.mark.parametrize("corpus_name", ["uniform8", "natural3"])
def test_run_dist_world_one_equals_run_host(request, corpus_name):
    """Without sdbg_dist_init the library's all-gather is a copy: sdbg_dist_bm25_topk_batch on all segments of the corpus
    gives run_host's hits, with the ordinal within the one rank in place of (segment, doc)."""
    env = request.getfixturevalue(corpus_name)
    one = env["one"]
    bases = np.cumsum([0] + [o.n_docs for o in env["corpus"].osegs])[:-1]
    rng = np.random.default_rng(5)
    queries = [sorted(int(t) for t in rng.choice(env["corpus"].n_terms, size=int(rng.integers(1, 4)), replace=False))
               for _ in range(64)]
    for kind in (sdb.OR, sdb.AND):
        for k in (1, 10, 1000, 8192):
            batch = sdb.PreparedBatch(one, queries, kind, sdb.BM25(), k)
            hd, nd = batch.run_dist()
            hl, nl, _ = batch.run_host()
            assert np.array_equal(nd, nl)
            for q in range(len(queries)):
                a, b = hd[q, :nd[q]], hl[q, :nl[q]]
                assert np.all(a["seg"] == 0)
                assert np.array_equal(a["doc"], bases[b["seg"]] + b["doc"]), (queries[q], kind, k)
                assert np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32))


# ---------------------------------------------------------------- (c) limits
def _expect_rejected(code, fn):
    before = ctx().launches
    with pytest.raises(SdbgError, match="^" + code):
        fn()
    assert ctx().launches == before, "a rejected call queued work"


def _single_doc_segment(n_docs):
    """A segment without norms whose only term holds the last doc (sparse: only the postings are stored)."""
    w = sdb.PostingsWriter(n_docs, has_wand=True)
    w.add_term(np.array([n_docs], np.uint32), np.array([2], np.uint32))
    doc, metas = w.finish()
    g = sdb.Segment(ctx(), n_docs)
    g.stage_postings(doc, metas)
    return g, sdb.IndexReader([g], n_docs, n_docs, [1])


def test_rank_slot_limits(uniform8):
    reader = uniform8["readers"][0]
    k, R = 10, 15
    batch = sdb.PreparedBatch(reader, [[0, 1]], sdb.OR, sdb.BM25(), k)
    keys = _zeros(R, 1, k)
    batch.run_device(14, keys[14].data_ptr())
    _expect_rejected("EUNSUPPORTED", lambda: batch.run_device(15, keys[0].data_ptr()))
    hits, n_out = sdb.merge_gathered(ctx(), keys.data_ptr(), R, 1, k)
    oh, _, _ = orc.bm25_topk([uniform8["corpus"].osegs[0]], "OR", oracle_terms(reader, sdb.BM25(), [0, 1]), k, mode=1)
    assert n_out[0] == k and np.all(hits["seg"][0] == 14)
    assert np.array_equal(hits["doc"][0], oh["doc"]) and np.array_equal(hits["score"][0].view(np.uint32), oh["score"].view(np.uint32))

    last = (1 << 28) - 1                     # the most docs a rank may hold: ordinals 1 .. 2^28 - 1
    g, big = _single_doc_segment(last)
    keys = _zeros(R, 1, k)
    sdb.PreparedBatch(big, [[0]], sdb.OR, sdb.BM25(), k).run_device(14, keys[14].data_ptr())
    hits, n_out = sdb.merge_gathered(ctx(), keys.data_ptr(), R, 1, k)
    o = orc.Segment(last, has_wand=True)
    o.add_term(np.array([last], np.uint32), np.array([2], np.uint32))
    oh, _, _ = orc.bm25_topk([o], "OR", oracle_terms(big, sdb.BM25(), [0]), k, mode=1)
    assert n_out[0] == 1 and (hits["seg"][0, 0], hits["doc"][0, 0]) == (14, last) and oh["doc"][0] == last
    assert hits["score"][0, 0].view(np.uint32) == oh["score"][0].view(np.uint32)
    g.close()

    g, over = _single_doc_segment(1 << 28)
    _expect_rejected("EUNSUPPORTED", lambda: sdb.PreparedBatch(over, [[0]], sdb.OR, sdb.BM25(), k).run_device(0, keys[0].data_ptr()))
    g.close()


def test_merge_gathered_argument_limits():
    keys = _zeros(2, 3, 8193)
    for R, nq, k in ((0, 3, 10), (2, 0, 10), (2, 3, 0)):
        _expect_rejected("EINVAL", lambda: sdb.merge_gathered(ctx(), keys.data_ptr(), R, nq, k))
    _expect_rejected("EUNSUPPORTED", lambda: sdb.merge_gathered(ctx(), keys.data_ptr(), 2, 3, 8193))
    hits, n_out = sdb.merge_gathered(ctx(), keys.data_ptr(), 2, 3, 8192)      # the largest k still runs
    assert np.all(n_out == 0)


# ---------------------------------------------------------------- (d) fixed-point GROUP BY merge
SPAN = 4096


@pytest.fixture(scope="module")
def nccl():
    c = sdb.Context(0)
    try:
        c.dist_init(sdb.Context.dist_unique_id(), 0, 1)
    except Exception as e:   # no NCCL library on this box
        c.close()
        pytest.skip("NCCL not available: %s" % e)
    seg = sdb.Segment(c, 16)   # finalize only needs the context
    yield dict(c=c, scan=sdb.IResearchScan([seg]))
    seg.close()
    c.close()


def _eunit(abs_bound):
    return math.frexp(abs_bound if abs_bound > 0 else 1.0)[1] + 1 - 117


def _merge(env, i64, f64, abs_bound):
    c = env["c"]
    d_i64, d_f64 = _cuda(i64), _cuda(f64)
    c.dist_groupby_merge(d_i64.data_ptr(), d_f64.data_ptr(), SPAN, abs_bound)
    c.sync()
    return d_i64.cpu().numpy(), d_f64.cpu().numpy(), (d_i64, d_f64)


def _finalize(env, dev):
    return env["scan"].groupby_finalize(0, SPAN, dev[0].data_ptr(), dev[1].data_ptr(), SPAN)


def _double_partials(rng, abs_bound):
    """Partial SUM(double) values, all within abs_bound, then NaN of both signs and both infinities."""
    vals = [0.0, -0.0]
    if abs_bound > 0:
        _, e = math.frexp(abs_bound)                     # abs_bound < 2^e
        vals += [abs_bound, -abs_bound, 5e-324, -5e-324, 2.2250738585072014e-308, abs_bound * 2.0 ** -200, 1e-300]
        for sh in range(0, 150, 3):                      # 53 significant bits at many exponents below the bound
            m = int(rng.integers(1 << 52, 1 << 53))
            w = math.ldexp(m, e - 53 - sh)
            if w <= abs_bound:
                vals += [w, -w]
        vals += list(rng.standard_normal(200) * abs_bound / 8)
    vals = [v for v in vals if abs(v) <= abs_bound]
    nonfinite = [float("nan"), -float("nan"), float("inf"), -float("inf")]
    return np.array(vals, np.float64), np.array(nonfinite, np.float64)


BOUNDS = {"zero": 0.0, "one": 1.0, "pow2": 2.0 ** 40, "max": float.fromhex("0x1.6a09e667f3bcdp+18"), "1e300": 1e300}


@pytest.mark.parametrize("bound", list(BOUNDS))
def test_double_partials_fixed_point(nccl, bound):
    """In-bound finite partials come back truncated toward zero to a multiple of 2^eunit (so exactly when they are such
    a multiple; a zero comes back as +0.0), NaN as NaN and infinities as themselves. 'pow2' is the frexp edge (the
    bound is 2^40 exactly); 'max' is a bound equal to the largest |partial|."""
    rng = np.random.default_rng(list(BOUNDS).index(bound))
    abs_bound = BOUNDS[bound]
    finite, special = _double_partials(rng, abs_bound)
    assert np.max(np.abs(finite)) == abs_bound
    f64 = np.zeros(SPAN)
    keys_f = rng.choice(SPAN, len(finite) + len(special), replace=False)
    f64[keys_f[:len(finite)]] = finite
    f64[keys_f[len(finite):]] = special
    i64 = np.zeros(4 * SPAN, np.int64)
    i64[:SPAN] = rng.integers(0, 5, SPAN)                # some keys have no rows at all
    i64[3 * SPAN:] = i64[:SPAN]
    got_i, got_f, dev = _merge(nccl, i64, f64, abs_bound)
    assert np.array_equal(got_i[:SPAN], i64[:SPAN]) and np.array_equal(got_i[3 * SPAN:], i64[3 * SPAN:])
    eu = Fraction(2) ** _eunit(abs_bound)
    for key, w in zip(keys_f[:len(finite)], finite):
        exact = Fraction(float(w)) / eu
        want = float(math.trunc(exact) * eu)             # truncated toward zero to a multiple of 2^eunit
        g = float(got_f[key])
        assert np.float64(g).view(np.uint64) == np.float64(want).view(np.uint64), (w, g, want)
        assert abs(Fraction(g) - Fraction(float(w))) < eu
        if exact.denominator == 1 and w != 0:
            assert np.float64(g).view(np.uint64) == np.float64(w).view(np.uint64)
    for key, w in zip(keys_f[len(finite):], special):
        g = float(got_f[key])
        assert math.isnan(g) if math.isnan(w) else g == w, (w, g)
    rows = _finalize(nccl, dev)                          # no partial beyond the bound: finalize succeeds
    assert np.array_equal(rows["key"], np.flatnonzero(i64[:SPAN]))


def test_partial_beyond_bound_fails_finalize(nccl):
    for abs_bound, w in ((0.0, 5e-324), (1.0, np.nextafter(1.0, 2.0)), (2.0 ** 40, 2.0 ** 41), (1e300, -1.7e308)):
        f64 = np.zeros(SPAN)
        f64[17] = w
        i64 = np.zeros(4 * SPAN, np.int64)
        i64[17] = 1
        c = nccl["c"]
        d_i64, d_f64 = _cuda(i64), _cuda(f64)
        c.dist_groupby_merge(d_i64.data_ptr(), d_f64.data_ptr(), SPAN, abs_bound)
        with pytest.raises(SdbgError, match="^EINVAL"):
            _finalize(nccl, (d_i64, d_f64))
        rows = _finalize(nccl, (d_i64, d_f64))           # the report is not repeated
        assert len(rows) == 1


def test_abs_bound_must_be_finite(nccl):
    c = nccl["c"]
    d_i64, d_f64 = _zeros(4 * SPAN), _cuda(np.zeros(SPAN))
    for bad in (float("inf"), float("nan"), -1.0):
        with pytest.raises(SdbgError, match="^EINVAL"):
            c.dist_groupby_merge(d_i64.data_ptr(), d_f64.data_ptr(), SPAN, bad)


def test_int_sum_limbs(nccl):
    rng = np.random.default_rng(44)
    los = [-2 ** 63, -1, 0, 2 ** 32 - 1, 2 ** 32, 2 ** 63 - 1]
    i64 = np.zeros(4 * SPAN, np.int64)
    keys = rng.choice(SPAN, 600, replace=False)
    his = rng.integers(-2 ** 62, 2 ** 62, len(keys))
    counts = rng.integers(1, 1 << 40, len(keys))
    counts[::7] = 0                                      # keys without rows are not emitted
    for j, key in enumerate(keys):
        i64[key] = counts[j]
        if counts[j]:
            i64[SPAN + key] = los[j % len(los)]
            i64[2 * SPAN + key] = his[j]
            i64[3 * SPAN + key] = counts[j] // 3
    got_i, _, dev = _merge(nccl, i64, np.zeros(SPAN), 1.0)
    rows = _finalize(nccl, dev)
    live = np.sort(keys[counts > 0])
    assert np.array_equal(rows["key"], live)
    want = {int(key): int(his[j]) * 2 ** 32 + los[j % len(los)] for j, key in enumerate(keys) if counts[j]}
    assert sdb.engine.sum_i128(rows) == [want[int(key)] for key in live]
    assert np.array_equal(rows["count"], i64[live].astype(np.uint64))
    assert np.array_equal(rows["cnt_f64"], i64[3 * SPAN + live].astype(np.uint64))
    assert np.array_equal(got_i[:SPAN], i64[:SPAN]) and np.array_equal(got_i[3 * SPAN:], i64[3 * SPAN:])


def test_groupby_partial_merge_finalize_equals_local(nccl):
    """partial -> merge -> finalize over a double column with NaN / inf in some groups equals the local GROUP BY. The
    doubles are multiples of 1/8 with small sums, so every order of addition gives the same sums."""
    c = nccl["c"]
    rng = np.random.default_rng(23)
    rows = 40_003
    key = rng.integers(0, 97, size=rows).astype(np.int64)
    v = rng.integers(-1000, 1001, size=rows).astype(np.int64)
    w = rng.integers(-8000, 8001, size=rows) / 8.0
    w[5] = np.inf; w[77] = np.nan; w[78] = -np.inf; w[400] = np.inf; w[401] = -np.inf
    g = sdb.Segment(c, rows)
    try:                                                 # the segment must not outlive its context, even on failure
        for f, vals in {1: key, 2: v, 4: w}.items():
            g.stage_column(f, vals)
        scan = sdb.IResearchScan([g])
        preds = [sdb.pred(2, "GE", -900)]
        local = scan.groupby(preds, 1, sum_int_field=2, avg_f64_field=4)
        span = 97
        d_i64, d_f64 = _zeros(4 * span), _cuda(np.zeros(span))
        scan.groupby_partial(preds, 1, 0, span, 2, 4, d_i64.data_ptr(), d_f64.data_ptr())
        sel = (v >= -900) & np.isfinite(w)
        c.dist_groupby_merge(d_i64.data_ptr(), d_f64.data_ptr(), span, float(np.abs(w[sel]).sum()))
        got = scan.groupby_finalize(0, span, d_i64.data_ptr(), d_f64.data_ptr(), span)
    finally:
        g.close()
    for f in ("key", "count", "sum_lo", "sum_hi", "cnt_f64"):
        assert np.array_equal(got[f], local[f]), f
    assert np.array_equal(np.isnan(got["sum_f64"]), np.isnan(local["sum_f64"]))
    assert np.isnan(local["sum_f64"]).any() and np.isinf(local["sum_f64"]).any()
    fin = ~np.isnan(local["sum_f64"])
    assert np.array_equal(got["sum_f64"][fin].view(np.uint64), local["sum_f64"][fin].view(np.uint64))
