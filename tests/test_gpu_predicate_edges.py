"""GPU: pushed column predicates at special values and domain edges, through every consumer, compared exactly with
predicate_reference.

One table of 40 x 2048 + 37 rows (the last zonemap block is partial) holds NaN of both signs, +-0.0, +-inf, denormals,
+-DBL_MAX and the int64 / int32 extremes, in constant blocks and mixed among random values; the same rows carry
synthetic postings, so the text consumers filter on the same columns. Each predicate (every op; float, int, out-of-range,
NaN and infinite constants on every column type; conjunctions that mix always-true and always-false predicates with
ordinary ones) goes through the filter bitmap, COUNT / SUM, every GROUP BY path (TMA with zonemaps on and off, raw and
bit-packed columns, the register path, the hash path) and the hybrid filter of count, stream, top-k, facet counts and
the sorted scan."""
import math

import numpy as np
import pytest

import count_reference as cr
import facet_reference as fr
import orc
import predicate_reference as pr
import serenedb_b200 as sdb
import sort_reference as sr
from gpu_util import ctx, to_gpu

pytestmark = pytest.mark.gpu

ROWS = 40 * 2048 + 37
BLK = 2048
N_BLOCKS = (ROWS + BLK - 1) // BLK
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
NAN, INF = float("nan"), math.inf
NEG_NAN = -NAN
DENORM = 5e-324
DBL_MAX = float(np.finfo(np.float64).max)
ONE_UP, ONE_DOWN = float(np.nextafter(1.0, INF)), float(np.nextafter(1.0, -INF))

# predicate columns
F64, F64N = 1, 2                       # float64, and its nullable copy
I64, I64C, I64P, I64N = 3, 4, 5, 6     # int64: raw; blocks of every width (packed on the device); I64C's values staged
                                       # packed by stage_column_for; nullable copy of I64C
NARROW, I32 = 7, 8                     # bit-packed just below INT64_MAX; int32
# GROUP BY keys and aggregates
KEY, WKEY, SUMI, AVGF = 9, 10, 11, 12
NOT_NULL_COLS = (F64, I64, I64P, I64C, NARROW, I32)
TERMS = [0, 2, 5, 17, 40]
QUERIES = {sdb.OR: [[1], [2, 3], [1, 2, 3, 4]], sdb.AND: [[0, 1], [0, 2, 4], [0, 1, 2, 3]]}
K = 20

F_SPECIALS = [NAN, NEG_NAN, INF, -INF, -0.0, 0.0, DENORM]                    # one constant block each
I64_EDGES = [I64_MIN, I64_MIN + 1, -(1 << 62) - 1, -(1 << 53) - 1, -1, 0, 1, (1 << 53) + 1, 1 << 62, I64_MAX - 1, I64_MAX]
I32_EDGES = [I32_MIN, I32_MIN + 1, -1, 0, 1, I32_MAX - 1, I32_MAX]


def _build_columns(rng):
    cols = {}
    f = rng.standard_normal(ROWS)
    for b, v in enumerate(F_SPECIALS):
        f[b * BLK:(b + 1) * BLK] = v
    pool = np.array(F_SPECIALS + [DBL_MAX, -DBL_MAX, 1.0, -1.0, ONE_UP, ONE_DOWN, -DENORM, 0.625])
    rest = np.arange(len(F_SPECIALS) * BLK, ROWS)
    pick = rest[rng.random(len(rest)) < 0.3]
    f[pick] = pool[rng.integers(0, len(pool), len(pick))]
    cols[F64] = (f, None)

    # I64: every block holds INT64_MIN and INT64_MAX, so no block packs narrower than 64 bits and the column stays raw
    a = rng.integers(I64_MIN, I64_MAX, ROWS, dtype=np.int64, endpoint=True)
    pick = rng.random(ROWS) < 0.3
    a[pick] = np.array(I64_EDGES, np.int64)[rng.integers(0, len(I64_EDGES), int(pick.sum()))]
    small = rng.random(ROWS) < 0.2
    a[small] = rng.integers(-5, 6, int(small.sum()))
    a[0::BLK], a[1::BLK] = I64_MIN, I64_MAX
    cols[I64] = (a, None)

    # I64C: constant blocks of each edge, blocks of small values, full-range blocks: bit widths 0, 4 and 64; a 64-bit block's
    # base + delta wraps around in the unpacking
    c = rng.integers(I64_MIN, I64_MAX, ROWS, dtype=np.int64, endpoint=True)
    for b, v in enumerate(I64_EDGES):
        c[b * BLK:(b + 1) * BLK] = v
    c[11 * BLK:25 * BLK] = rng.integers(-5, 6, 14 * BLK)
    rest = np.arange(25 * BLK, ROWS)
    pick = rest[rng.random(len(rest)) < 0.2]
    c[pick] = np.array(I64_EDGES, np.int64)[rng.integers(0, len(I64_EDGES), len(pick))]
    cols[I64C] = (c, None)
    cols[I64P] = (c, None)

    cols[NARROW] = (I64_MAX - rng.integers(0, 1000, ROWS).astype(np.int64), None)
    i = rng.integers(I32_MIN, I32_MAX, ROWS, dtype=np.int64, endpoint=True)
    for b, v in enumerate([I32_MIN, I32_MAX, 0, -1, 1]):
        i[b * BLK:(b + 1) * BLK] = v
    i[5 * BLK:15 * BLK] = rng.integers(-5, 6, 10 * BLK)
    pick = rng.random(ROWS) < 0.2
    i[pick] = np.array(I32_EDGES)[rng.integers(0, len(I32_EDGES), int(pick.sum()))]
    cols[I32] = (i.astype(np.int32), None)

    cols[F64N] = (f.copy(), rng.random(ROWS) < 0.7)
    cols[I64N] = (c.copy(), rng.random(ROWS) < 0.7)
    cols[KEY] = (rng.integers(0, 64, ROWS).astype(np.int64), None)
    wide = rng.integers(I64_MIN, I64_MAX, 200, dtype=np.int64, endpoint=True)
    cols[WKEY] = (wide[rng.integers(0, len(wide), ROWS)], None)
    cols[SUMI] = (rng.integers(-2 ** 40, 2 ** 40, ROWS).astype(np.int64), None)
    cols[AVGF] = (rng.standard_normal(ROWS), None)
    return cols


class Table:
    def __init__(self):
        rng = np.random.default_rng(20261016)
        self.cols = _build_columns(rng)
        self._masks = {}
        self.oseg, dl, lists = orc.synth_segment(ROWS, TERMS)
        staged = {f: (v, None if ok is None else cr.validity_words(ok)) for f, (v, ok) in self.cols.items()
                  if f not in (I64P, NARROW)}
        self.seg = to_gpu(self.oseg, columns=staged)
        self.seg.stage_column_for(I64P, sdb.pack_for(self.cols[I64P][0]))
        self.seg.stage_column_for(NARROW, sdb.pack_for(self.cols[NARROW][0]))
        for f in (I64P, NARROW, I64C):
            assert self.seg.column_packed(f, ROWS) is not None, f
        assert self.seg.column_packed(I64, ROWS) is None
        self.reader = sdb.IndexReader([self.seg], ROWS, int(dl.sum()), [len(d) for d, _ in lists])
        self.scan = sdb.IResearchScan([self.seg])
        self.scorer = sdb.BM25()
        docs = [d for d, _ in lists]
        self.matches = {kind: [cr.match_docs(docs, kind, q) for q in qs] for kind, qs in QUERIES.items()}
        self.streams = {kind: [sdb.StreamScoredDocs(self.reader, 0, q, kind, self.scorer) for q in qs]
                        for kind, qs in QUERIES.items()}
        for kind in QUERIES:
            for m, (d, _) in zip(self.matches[kind], self.streams[kind]):
                assert np.array_equal(m, d)
        # the unfiltered matches in top-k order (score desc, doc asc) and in sorted-scan order (sort_reference)
        self.by_score = {kind: [np.lexsort((d, -sc)) for d, sc in self.streams[kind]] for kind in QUERIES}
        self.by_col = {kind: [sr.sorted_hits([[m]], sdb.OR, [0], [(self.cols[SUMI][0], None)]) for m in self.matches[kind]]
                       for kind in QUERIES}

    def mask(self, preds):
        key = repr(preds)      # only NaN and -NaN share a repr, and they select the same rows
        if key not in self._masks:
            self._masks[key] = pr.pass_mask_all(self.cols, preds)
        return self._masks[key]


@pytest.fixture(scope="module")
def T():
    return Table()


def _consts(field):
    if field in (F64, F64N):
        return [NAN, NEG_NAN, INF, -INF, 0.0, -0.0, DENORM, -DENORM, DBL_MAX, -DBL_MAX, 1.0, ONE_UP, ONE_DOWN, -1.0,
                0, (1 << 53) + 1, 0.625]
    return [I64_MIN, I64_MIN + 1, I64_MAX - 1, I64_MAX, 2 ** 63, -2 ** 63 - 2048, I32_MIN - 1, I32_MIN, I32_MIN + 1,
            I32_MAX - 1, I32_MAX, I32_MAX + 1, -1, 0, 1, 0.5, -0.5, 2.5, -2.5, float(1 << 53), float(1 << 62),
            float(2 ** 63), -float(2 ** 63), 1e300, -1e300, INF, -INF, NAN, np.float32(2.5), (1 << 53) + 1, I64_MAX - 500]


def _betweens(field):
    if field in (F64, F64N):
        return [(1.0, 1.0), (ONE_UP, 1.0), (-INF, 0.0), (0.0, INF), (NAN, INF), (-INF, NAN), (0.0, -0.0),
                (-DBL_MAX, DBL_MAX), (DENORM, DBL_MAX)]
    return [(0, 0), (1, 0), (0.5, INF), (-INF, 3.5), (NAN, 5.0), (-5.0, NAN), (I64_MIN, I64_MAX), (-2.5, 2.5),
            (I64_MAX - 5, I64_MAX), (float(1 << 62), INF), (-1e300, -1e299)]


def _singles(fields):
    out = []
    for f in fields:
        for c in _consts(f):
            out += [[(f, op, c)] for op in ("LT", "LE", "GT", "GE", "EQ", "NE")]
        out += [[(f, "BETWEEN", lo, hi)] for lo, hi in _betweens(f)]
        out += [[(f, "IS_NULL")], [(f, "IS_NOT_NULL")]]
    return out


ALL_FIELDS = (F64, F64N, I64, I64P, I64C, I64N, NARROW, I32)
CONJUNCTIONS = [
    [(I64, "NE", NAN), (F64, "GE", 0.0)],
    [(I64, "LE", INF), (I32, "GT", 0), (F64, "LT", 1.0)],
    [(F64, "NE", NAN), (I64, "LT", -INF)],
    [(I64, "GT", I64_MAX), (F64, "GE", 0.0)],
    [(I32, "GE", -0.5), (I64P, "LT", 2.5), (NARROW, "GT", 9.2e18), (F64, "NE", 1.0)],
    [(I64N, "NE", NAN), (F64N, "LE", INF)],
    [(I64C, "BETWEEN", -2.5, INF), (F64, "BETWEEN", -INF, 0.0), (I32, "NE", 0), (I64P, "GE", -1)],
    [(F64, "EQ", 0.0), (I64C, "LE", 1e300)],
    [(NARROW, "GE", I64_MAX - 10), (I64C, "BETWEEN", -1, 1), (F64, "GT", -INF)],
    [(F64, "LT", NAN), (I32, "GE", I32_MIN)],
    [(I64C, "EQ", 0), (I64P, "EQ", 0.0), (I32, "LT", 2 ** 63)],
    [(I32, "LT", 2 ** 63), (I64N, "GT", -1e19), (F64N, "NE", -0.0)],
]
CASES = _singles(ALL_FIELDS) + CONJUNCTIONS


def _g(preds):
    return [sdb.pred(*p) for p in preds]


def test_filter_bitmap_is_bit_identical(T):
    for preds in CASES:
        got = T.seg.filter_bitmap(_g(preds))
        assert np.array_equal(got, cr.validity_words(T.mask(preds))), preds


def test_count_sum_is_exact(T):
    sumi = T.cols[SUMI][0]
    for preds in CASES:
        m = T.mask(preds)
        cnt, si, _ = T.scan.count_sum(_g(preds), SUMI)
        assert (cnt, si) == (int(m.sum()), int(sumi[m].sum())), preds


def _groupby_ref(T, mask, key_field):
    k = T.cols[key_field][0][mask]
    keys, inv, counts = np.unique(k, return_inverse=True, return_counts=True)
    sums = np.zeros(len(keys), np.int64)
    np.add.at(sums, inv, T.cols[SUMI][0][mask])          # exact: |sum| < 2^17 rows * 2^40
    fs, fabs = np.zeros(len(keys)), np.zeros(len(keys))
    np.add.at(fs, inv, T.cols[AVGF][0][mask])
    np.add.at(fabs, inv, np.abs(T.cols[AVGF][0][mask]))
    return keys, counts, sums, fs, fabs


def _check_groups(got, ref, what):
    keys, counts, sums, fs, fabs = ref
    assert np.array_equal(got["key"], keys), what
    assert np.array_equal(got["count"], counts), what
    assert np.array_equal(got["cnt_f64"], counts), what
    assert sdb.sum_i128(got) == [int(s) for s in sums], what
    assert np.all(np.abs(got["sum_f64"] - fs) <= 1e-9 * fabs + 1e-300), what


def _groupby(T, preds, key_field):
    if key_field == KEY:
        return T.scan.groupby(_g(preds), KEY, sum_int_field=SUMI, avg_f64_field=AVGF, cap=64)
    return T.scan.groupby(_g(preds), WKEY, sum_int_field=SUMI, avg_f64_field=AVGF, cap=256, n_groups_hint=200)


def _dead_lower_bound(T, preds):
    """Blocks the zonemap verdict must skip: constant blocks (min == max) of a NOT NULL column whose value fails one of
    the set's predicates other than <> (a <> verdict needs the excluded value alone in the block's key range)."""
    n = 0
    for b in range(N_BLOCKS):
        for f, op, *bounds in preds:
            blk = T.cols[f][0][b * BLK:(b + 1) * BLK]
            bits = blk.view(np.int64) if blk.dtype == np.float64 else blk
            if f in NOT_NULL_COLS and op != "NE" and (bits == bits[0]).all() and not pr.pass_mask(blk[:1], None, op, *bounds)[0]:
                n += 1
                break
    return n


def test_groupby_tma_with_and_without_zonemaps(T, monkeypatch):
    """TMA path (raw, bit-packed and FOR-wrapping predicate columns; nullable ones fall back to the register path): exact
    against the NumPy GROUP BY of the masked rows; zonemaps on and off give the same rows, and with them on the constant
    blocks a predicate excludes are skipped, while no block holding a passing row is."""
    skip_checked = 0
    for preds in CASES:
        m = T.mask(preds)
        ref = _groupby_ref(T, m, KEY)
        monkeypatch.setenv("SDBG_ZONEMAP", "1")
        on = _groupby(T, preds, KEY)
        stats = ctx().scan_stats()
        _check_groups(on, ref, ("zonemap on", preds))
        monkeypatch.setenv("SDBG_ZONEMAP", "0")
        off = _groupby(T, preds, KEY)
        _check_groups(off, ref, ("zonemap off", preds))
        for f in ("key", "count", "sum_lo", "sum_hi", "cnt_f64"):
            assert np.array_equal(on[f], off[f]), (f, preds)
        nullable_or_null_op = any(f in (F64N, I64N) or op in ("IS_NULL", "IS_NOT_NULL") for f, op, *_ in preds)
        if nullable_or_null_op or m.all() or not m.any():
            continue   # register path, or a predicate set the host folds to always / never: no zonemap pass ran
        total, skipped = stats
        live = sum(bool(m[b * BLK:(b + 1) * BLK].any()) for b in range(N_BLOCKS))
        assert total == N_BLOCKS and skipped <= N_BLOCKS - live, (preds, stats, live)
        need = _dead_lower_bound(T, preds)
        assert skipped >= need, (preds, stats, need)
        skip_checked += need > 0
    assert skip_checked >= 50


@pytest.mark.parametrize("path", ["register", "hash"])
def test_groupby_register_and_hash_paths(T, monkeypatch, path):
    if path == "register":
        monkeypatch.setenv("SDBG_GROUPBY_TMA", "0")
    key = KEY if path == "register" else WKEY
    for preds in CASES:
        _check_groups(_groupby(T, preds, key), _groupby_ref(T, T.mask(preds), key), (path, preds))


def _hybrid_expected(T, mask):
    """Per kind and query: the filtered count, stream (docs, scores), top-k docs, facet counts and sorted-scan docs."""
    out = {}
    for kind in QUERIES:
        for qi in range(len(QUERIES[kind])):
            m = [T.matches[kind][qi]]
            sd, ss = T.streams[kind][qi]
            keep = mask[sd.astype(np.int64) - 1]
            by_score = T.by_score[kind][qi]
            by_col = T.by_col[kind][qi]
            out[kind, qi] = dict(
                count=cr.count([m], sdb.OR, [0], masks=[mask]), docs=sd[keep], scores=ss[keep],
                topk=by_score[keep[by_score]][:K],      # (score desc, doc asc) of the matches, filtered: the first K
                facets=fr.facet_counts([m], sdb.OR, [0], [(T.cols[KEY][0], None)], 0, 64, masks=[mask]),
                sorted=by_col["docs"][mask[by_col["docs"].astype(np.int64) - 1]][:K])
    return out


def test_hybrid_filter_every_text_consumer(T):
    """filt= on count, stream, top-k, facet counts and the sorted scan, OR and AND queries of 1-4 terms, pruning levels 0
    and 2: each equals the unfiltered matches restricted to the reference mask (the sorted scan: sort_reference's order
    of all matches, restricted to the mask, which is its order of the filtered matches)."""
    singles = _singles((F64, F64N, I64, I64C, I64N, NARROW, I32))
    try:
        for (pred_spec,) in singles:
            filt = sdb.pred(*pred_spec)
            exp = _hybrid_expected(T, T.mask([pred_spec]))
            for level in (0, 2):
                ctx().set_wand(level)
                for kind, qs in QUERIES.items():
                    what = (level, kind, pred_spec)
                    counts = sdb.ExecuteCountBatch(T.reader, qs, kind, filt=filt)
                    hits, n_out, total = sdb.ExecuteTopKBatch(T.reader, qs, kind, T.scorer, K, filt=filt)
                    facets = sdb.ExecuteFacetCountsBatch(T.reader, qs, kind, KEY, key_min=0, key_span=64, filt=filt)
                    by_col = sdb.ExecuteTopKByColumnBatch(T.reader, qs, kind, SUMI, K, filt=filt)
                    for qi, q in enumerate(qs):
                        e = exp[kind, qi]
                        assert counts[qi] == e["count"], what + (q,)
                        gd, gs = sdb.StreamScoredDocs(T.reader, 0, q, kind, T.scorer, filt=filt)
                        assert np.array_equal(gd, e["docs"]), what + (q,)
                        assert np.array_equal(gs.view(np.uint32), e["scores"].view(np.uint32)), what + (q,)
                        if level == 0:
                            assert total[qi] == e["count"], what + (q,)   # exact without pruning
                        h = hits[qi, :n_out[qi]]
                        sd, ss = T.streams[kind][qi]
                        assert np.array_equal(h["doc"], sd[e["topk"]]), what + (q,)
                        assert np.array_equal(h["score"].view(np.uint32), ss[e["topk"]].view(np.uint32)), what + (q,)
                        assert np.array_equal(facets["counts"][qi], e["facets"][0]), what + (q,)
                        assert facets["nulls"][qi] == e["facets"][1], what + (q,)
                        assert np.array_equal(by_col["docs"][qi], e["sorted"]), what + (q,)
                        assert np.array_equal(by_col["values"][qi], T.cols[SUMI][0][e["sorted"].astype(np.int64) - 1]), what + (q,)
    finally:
        ctx().set_wand(0)
