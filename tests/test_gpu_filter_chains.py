"""GPU: filter chains (sdbg.h SDBG_OP_AND_NEXT, `WHERE body @@ '...' AND a < x AND b = y`) on every full-text entry.

A chain must give exactly what the same call gives when filtered by one indicator column m = 1, where m is the chain's
pass mask from predicate_reference, staged as a nullable int32 column with every row valid (no zonemap: the per-doc
path). Two segments of different sizes (one past 65 536 docs, both with a partial last zone) carry raw, bit-packed,
int32, float64 and nullable columns, plus a doc-ordered column and a blocky one whose zones the chains judge dead,
pass or mixed. A chain of one must be bit-identical to the single predicate; errors come before anything is queued."""
import json
import math
import subprocess

import numpy as np
import pytest

import count_reference as cr
import orc
import predicate_reference as pr
import serenedb_b200 as sdb
from gpu_util import ctx, to_gpu
from serenedb_b200._native import SdbgError

pytestmark = pytest.mark.gpu

SIZES = (150_000, 41 * 2048 + 37)
TERMS = [0, 2, 5, 17, 40]
RAW, PACKED, I32, F64, NULLABLE, ORDERED, BLOCKY, M = 1, 2, 3, 4, 5, 6, 7, 99
NAN = float("nan")
QUERIES = {sdb.OR: [[1], [2, 3], [1, 2, 3, 4]], sdb.AND: [[0, 1], [0, 2, 4]]}
GROUPS = [[[1], [2, 3]], [[0, 2], [3, 4]]]
MIN_MATCH = [[1, 1], [1, 2]]
EXCLUDE = [[4], []]
K = 25

CHAINS = [
    [(ORDERED, "LT", 60000), (RAW, "GT", 0)],
    [(PACKED, "BETWEEN", 100, 700), (F64, "LT", 0.5), (BLOCKY, "NE", 3)],
    [(ORDERED, "GE", 30000.5), (I32, "LE", 2 ** 30), (NULLABLE, "IS_NOT_NULL"), (F64, "NE", NAN)],
    [(BLOCKY, "EQ", 2), (NULLABLE, "IS_NULL"), (PACKED, "GT", 10), (ORDERED, "LT", 1e18)],
    [(I32, "LT", 2.5e8), (ORDERED, "BETWEEN", 1000.5, 140000.25), (F64, "GE", -1.0)],
    [(NULLABLE, "LE", 0), (ORDERED, "GT", 5000), (BLOCKY, "GE", 1)],
    [(BLOCKY, "EQ", 9), (ORDERED, "GE", 0)],                    # dead everywhere
    [(F64, "EQ", NAN), (ORDERED, "GT", 5)],                     # NaN: no row
    [(ORDERED, "GE", 0), (BLOCKY, "LE", 4), (PACKED, "IS_NOT_NULL")],   # passes everywhere
    [(PACKED, "IS_NOT_NULL"), (F64, "NE", NAN)],                # passes everywhere without a zonemap read
]


def _columns(rng, n):
    f = rng.standard_normal(n)
    f[rng.random(n) < 0.01] = NAN
    valid = rng.random(n) < 0.8
    return {RAW: (rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64, endpoint=True), None),
            PACKED: (rng.integers(0, 1000, n, dtype=np.int64), None),
            I32: (rng.integers(-2 ** 31, 2 ** 31 - 1, n, dtype=np.int64).astype(np.int32), None),
            F64: (f, None),
            NULLABLE: (rng.integers(-5, 5, n, dtype=np.int64), valid),
            ORDERED: (np.arange(n, dtype=np.int64), None),
            BLOCKY: (((np.arange(n) // 2048) % 5).astype(np.int32), None)}


def _stage(seg, field, values, valid):
    seg.stage_column(field, values, None if valid is None else cr.validity_words(valid))


class Corpus:
    def __init__(self):
        rng = np.random.default_rng(20261017)
        self.cols, self.segs, dls, lists_all = [], [], 0, []
        for n in SIZES:
            oseg, dl, lists = orc.synth_segment(n, TERMS)
            cols = _columns(rng, n)
            seg = to_gpu(oseg)
            for f, (v, ok) in cols.items():
                _stage(seg, f, v, ok)
            assert seg.column_packed(PACKED, n) is not None and seg.column_packed(RAW, n) is None
            self.cols.append(cols)
            self.segs.append(seg)
            dls += int(dl.sum())
            lists_all.append([len(d) for d, _ in lists])
        docs_per_term = [sum(x[t] for x in lists_all) for t in range(len(TERMS))]
        self.reader = sdb.IndexReader(self.segs, sum(SIZES), dls, docs_per_term)
        self.scorer = sdb.BM25()

    def stage_indicator(self, chain):
        """m = 1 where every predicate of the chain holds, per segment; nullable with every row valid."""
        for seg, cols, n in zip(self.segs, self.cols, SIZES):
            m = pr.pass_mask_all(cols, chain).astype(np.int32)
            _stage(seg, M, m, np.ones(n, bool))


@pytest.fixture(scope="module")
def C():
    return Corpus()


def _preds(chain):
    return [sdb.pred(f, op, *b) for f, op, *b in chain]


IND = sdb.pred(M, "EQ", 1)


def _outputs(C, filt, totals=True):
    """Every full-text entry under `filt`, as comparable values. totals=False drops the top-k entries' total_matches,
    which block-max pruning (levels 1, 2) makes a lower bound that depends on the order the threshold rises in."""
    r, s = C.reader, C.scorer
    out = {}
    for kind, qs in QUERIES.items():
        out["topk", kind] = sdb.ExecuteTopKBatch(r, qs, kind, s, K, filt=filt)
        out["count", kind] = sdb.ExecuteCountBatch(r, qs, kind, filt=filt)
        out["facet", kind] = sdb.ExecuteFacetCountsBatch(r, qs, kind, BLOCKY, key_min=0, key_span=5, filt=filt)
        out["agg", kind] = sdb.ExecuteMatchAggregatesBatch(r, qs, kind, PACKED, key_field=BLOCKY, key_min=0, key_span=5, filt=filt)
        out["sorted", kind] = sdb.ExecuteTopKByColumnBatch(r, qs, kind, RAW, K, descending=True, filt=filt)
        out["scan", kind] = [sdb.StreamScoredDocs(r, si, q, kind, s, filt=filt) for si in range(len(SIZES)) for q in qs]
    qs = QUERIES[sdb.OR][:2]
    out["excl"] = sdb.ExecuteTopKBatch(r, qs, sdb.OR, s, K, filt=filt, exclude=EXCLUDE)
    out["excl_count"] = sdb.ExecuteCountBatch(r, qs, sdb.OR, filt=filt, exclude=EXCLUDE)
    out["groups"] = sdb.ExecuteTopKGroupsBatch(r, GROUPS, s, K, filt=filt)
    out["min_match"] = sdb.ExecuteTopKGroupsBatch(r, GROUPS, s, K, filt=filt, min_match=MIN_MATCH)
    out["groups_count"] = sdb.ExecuteCountGroupsBatch(r, GROUPS, filt=filt, min_match=MIN_MATCH)
    out["groups_facet"] = sdb.ExecuteFacetCountsGroupsBatch(r, GROUPS, BLOCKY, key_min=0, key_span=5, filt=filt, exclude=EXCLUDE)
    if not totals:
        for key in [("topk", kind) for kind in QUERIES] + ["excl", "groups", "min_match"]:
            out[key] = out[key][:2]
    return out


def _assert_same(a, b, what=""):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            _assert_same(a[k], b[k], f"{what}/{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, f"{what}[{i}]")
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape, what
        if a.dtype == object:                        # exact integers (128-bit sums)
            assert a.tolist() == b.tolist(), what
        else:
            assert a.tobytes() == b.tobytes(), what  # bit for bit (NaN payloads, float scores)
    else:
        assert a == b or (isinstance(a, float) and math.isnan(a) and math.isnan(b)), (what, a, b)


def _matches(out):
    return sum(int(np.sum(out["count", kind])) for kind in QUERIES)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_chain_equals_indicator_column(C, level):
    ctx().set_wand(level)
    try:
        for chain in CHAINS:
            C.stage_indicator(chain)
            _assert_same(_outputs(C, _preds(chain), level == 0), _outputs(C, IND, level == 0), repr(chain))
    finally:
        ctx().set_wand(False)


def test_verdicts_at_their_limits(C):
    """A chain dead everywhere finds nothing; one that passes everywhere is the unfiltered query, bit for bit."""
    dead = _outputs(C, _preds(CHAINS[6]))
    assert _matches(dead) == 0
    for kind in QUERIES:
        hits, n_out, total = dead["topk", kind]
        assert not n_out.any() and not total.any()
        assert all(len(d) == 0 for d, _ in dead["scan", kind])
    _assert_same(_outputs(C, _preds(CHAINS[8])), _outputs(C, None))
    _assert_same(_outputs(C, _preds(CHAINS[9])), _outputs(C, None))
    assert _matches(_outputs(C, None)) > 0


def test_chain_of_one_is_the_predicate(C):
    import torch
    for f, op, *b in [(ORDERED, "LT", 70000), (NULLABLE, "GE", 0), (F64, "BETWEEN", -0.5, 0.5), (PACKED, "NE", 7)]:
        p = sdb.pred(f, op, *b)
        _assert_same(_outputs(C, [p]), _outputs(C, p), repr((f, op)))
        _assert_same(_outputs(C, (p,)), _outputs(C, p), repr((f, op)))
        r, qs = C.reader, [[1, 2], [0, 3]]
        dist = [lambda filt: sdb.ExecuteDistCountGroupsBatch(r, GROUPS, filt=filt, min_match=MIN_MATCH),
                lambda filt: sdb.ExecuteDistFacetCountsGroupsBatch(r, GROUPS, BLOCKY, 0, 5, filt=filt),
                lambda filt: sdb.ExecuteDistMatchAggregatesGroupsBatch(r, GROUPS, PACKED, BLOCKY, 0, 5, filt=filt),
                lambda filt: sdb.ExecuteDistTopKByColumnGroupsBatch(r, GROUPS, RAW, K, filt=filt),
                lambda filt: sdb.PreparedBatch(r, qs, sdb.OR, C.scorer, K, filt=filt).run_dist()]
        for fn in dist:
            _assert_same(fn([p]), fn(p))
        keys = [torch.zeros(len(qs) * K, dtype=torch.int64, device="cuda") for _ in range(2)]
        totals = [torch.zeros(len(qs), dtype=torch.int64, device="cuda") for _ in range(2)]
        for i, filt in enumerate(([p], p)):
            sdb.PreparedBatch(r, qs, sdb.OR, C.scorer, K, filt=filt).run_device(0, keys[i].data_ptr(), totals[i].data_ptr())
        ctx().sync()
        assert torch.equal(keys[0], keys[1]) and torch.equal(totals[0], totals[1])
    _assert_same(_outputs(C, []), _outputs(C, None))


def test_verdicts_follow_writes_and_restaging(C):
    """The ordered column rewritten in place (sdbg_column_device_ptr) and restaged: the zonemaps and so the verdicts
    follow the new values."""
    import torch
    chain = [(ORDERED, "BETWEEN", 20000, 90000), (BLOCKY, "NE", 1)]
    C.stage_indicator(chain)
    _assert_same(_outputs(C, _preds(chain)), _outputs(C, IND))
    originals = [cols[ORDERED][0].copy() for cols in C.cols]
    try:
        for seg, cols, n in zip(C.segs, C.cols, SIZES):
            new = (n - 1 - np.arange(n)).astype(np.int64)          # reversed: other zones are dead and pass now
            ptr, rows = seg.column_device_ptr(ORDERED)
            assert rows == n
            ctx().sync()

            class _Mem:
                __cuda_array_interface__ = dict(shape=(n,), typestr="<i8", data=(int(ptr), False), version=3)
            torch.as_tensor(_Mem(), device="cuda").copy_(torch.from_numpy(new).cuda())
            torch.cuda.synchronize()
            cols[ORDERED] = (new, None)
        C.stage_indicator(chain)
        _assert_same(_outputs(C, _preds(chain)), _outputs(C, IND))
        for seg, cols, n in zip(C.segs, C.cols, SIZES):
            new = (np.arange(n) * 3 % 100_000).astype(np.int64)
            _stage(seg, ORDERED, new, None)
            cols[ORDERED] = (new, None)
        C.stage_indicator(chain)
        _assert_same(_outputs(C, _preds(chain)), _outputs(C, IND))
    finally:
        for seg, cols, old in zip(C.segs, C.cols, originals):
            _stage(seg, ORDERED, old, None)
            cols[ORDERED] = (old, None)


def _expect_rejected(code, fn):
    before = ctx().launches
    with pytest.raises(SdbgError, match="^" + code):
        fn()
    assert ctx().launches == before, "a rejected call queued work"


def test_errors_before_anything_is_queued(C):
    r, s, qs = C.reader, C.scorer, [[1, 2]]
    ok = sdb.pred(ORDERED, "LT", 100)
    garbage = sdb.pred(12345, "LT", 0)
    garbage.op = 77
    entries = [lambda f: sdb.ExecuteTopKBatch(r, qs, sdb.OR, s, K, filt=f),
               lambda f: sdb.ExecuteCountBatch(r, qs, sdb.OR, filt=f),
               lambda f: sdb.ExecuteFacetCountsBatch(r, qs, sdb.OR, BLOCKY, key_min=0, key_span=5, filt=f),
               lambda f: sdb.ExecuteTopKByColumnBatch(r, qs, sdb.OR, RAW, K, filt=f),
               lambda f: sdb.StreamScoredDocs(r, 0, qs[0], sdb.OR, s, filt=f),
               lambda f: sdb.ExecuteTopKGroupsBatch(r, GROUPS, s, K, filt=f)]
    short = 77
    for seg, n in zip(C.segs, SIZES):
        _stage(seg, short, np.zeros(n - 1, np.int32), None)
    sdb.ExecuteCountBatch(r, qs, sdb.OR, filt=ok)   # a packed column's raw view is decoded once, on first use
    for fn in entries:
        _expect_rejected("EUNSUPPORTED", lambda: fn([ok, ok, ok, ok, garbage]))   # the bit on the 4th; the 5th never read
        _expect_rejected("ENOTFOUND", lambda: fn([ok, sdb.pred(4242, "LT", 1), ok]))
        _expect_rejected("EINVAL", lambda: fn([ok, ok, sdb.pred(short, "LT", 1)]))
        bad = sdb.pred(ORDERED, "LT", 1)
        bad.op = 42
        _expect_rejected("EINVAL", lambda: fn([ok, ok, bad]))
    chained = sdb.pred(ORDERED, "LT", 100)
    chained.op |= sdb.engine.AND_NEXT
    with pytest.raises(SdbgError, match="^EINVAL"):
        sdb.resolve_pred(chained, np.int64)
    with pytest.raises(SdbgError, match="^EINVAL"):
        sdb.IResearchScan([C.segs[0]]).count_sum([chained, ok])


def test_adapter_chain_matches_indicator():
    from serenedb_b200 import build as b
    exe = b.build_adapters()
    res = subprocess.run([exe, "200000", "chain"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    chain, ind = [json.loads(line) for line in res.stdout.strip().splitlines()]
    assert chain["indicator"] == 0 and ind["indicator"] == 1
    for key in ("topk", "total", "stream_n", "stream_doc_sum", "count"):
        assert chain[key] == ind[key], key
    assert chain["count"] > 0 and len(chain["topk"]) == 100
