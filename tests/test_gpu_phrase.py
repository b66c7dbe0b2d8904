"""Exact phrase queries on the GPU (sdbg_stage_positions, sdbg_phrase_count_batch, sdbg_phrase_topk_batch) against the
NumPy statement (tests/phrase_reference.py): counts and top-k hits bit for bit (doc, segment, order, fp32 score bits)
over token-sequence segments (a term missing from one of them), every doc and frequency block encoding (the
shape_corpora.py shapes with positions added), doc ids past 2^31, deleted docs, filter chains of 1..4 predicates,
exclusions, BM25 / BM15 / BM1 / TFIDF, pruning levels 0..2, k above the match count, ties at the cut, a batch of
phrase lengths 1..16 with repeated terms, gaps, the error codes and the staging checks."""
import ctypes as C

import numpy as np
import pytest

import orc
import phrase_reference as pr
import serenedb_b200 as sdb
from serenedb_b200 import _native as N
from gpu_util import ctx, to_gpu
from shape_corpora import NORM_WIDTHS, companion, shape_segment

pytestmark = pytest.mark.gpu

V = 12   # vocabulary of the token corpora: term 11 never occurs in segment 1


def _token_segment(rng, n, vocab, missing=()):
    p = 1.0 / np.arange(1, vocab + 1)
    for t in missing:
        p[t] = 0
    p /= p.sum()
    docs = [rng.choice(vocab, size=int(rng.integers(1, 40)), p=p).tolist() for _ in range(n)]
    post = pr.postings(docs, vocab)
    oseg = orc.Segment(n, has_wand=True)
    norms = np.array([len(d) for d in docs], np.uint32)
    oseg.set_norms(norms)
    for d, f, _ in post:
        oseg.add_term(d, f)
    return docs, post, norms, oseg


@pytest.fixture(scope="module")
def tok():
    rng = np.random.default_rng(2024)
    sizes = (3000, 2500, 4000)
    segs, docs, posts, norms = [], [], [], []
    cols = []
    for i, n in enumerate(sizes):
        d, post, nm, oseg = _token_segment(rng, n, V, missing=(11,) if i == 1 else ())
        c = {1: (rng.integers(0, 1000, n).astype(np.int32), None), 2: (rng.integers(-10**9, 10**9, n).astype(np.int64), None),
             3: (rng.random(n) * 100.0, None), 4: (rng.integers(0, 50, n).astype(np.int32), None)}
        g = to_gpu(oseg, columns=c)
        g.stage_positions(*pr.staged_positions(post))
        segs.append(g); docs.append(d); posts.append(post); norms.append(nm); cols.append(c)
    deleted = [rng.choice(np.arange(1, sizes[0] + 1), 300, replace=False).astype(np.uint32), None, None]
    segs[0].stage_docs_mask(deleted[0])
    dwt = [sum(len(p[t][0]) for p in posts) for t in range(V)]
    reader = sdb.IndexReader(segs, sum(sizes), int(sum(int(n.sum()) for n in norms)), dwt)
    return dict(segs=segs, docs=docs, posts=posts, norms=norms, cols=cols, deleted=deleted, reader=reader, rng=rng)


def _phrases(t, rng, n, lengths):
    """Phrases cut from the corpus's own docs (so that they match), of the given lengths, plus a few random ones."""
    out = []
    for L in lengths:
        for _ in range(n):
            seq = t["docs"][int(rng.integers(0, 3))][int(rng.integers(0, 2500))]
            if len(seq) >= L:
                s = int(rng.integers(0, len(seq) - L + 1))
                out.append(seq[s:s + L])
            else:
                out.append(rng.integers(0, 4, L).tolist())
    return out


def _ref_matches(t, phrase, rel=None, excl=(), masks=None):
    masks = masks or [None] * 3
    return [pr.match(d, phrase, rel, excl, x, m) for d, x, m in zip(t["docs"], t["deleted"], masks)]


def _check(t, phrases, scorer=None, k=10, rels=None, filt=None, masks=None, excl=None, levels=(0,)):
    rels = rels or [None] * len(phrases)
    excl = excl or [[]] * len(phrases)
    want = [_ref_matches(t, p, r, x, masks) for p, r, x in zip(phrases, rels, excl)]
    counts = sdb.ExecutePhraseCountBatch(t["reader"], phrases, rel_pos=rels, filt=filt, exclude=excl)
    assert counts.tolist() == [sum(len(m[0]) for m in w) for w in want]
    if scorer is None:
        return counts
    for lv in levels:
        ctx().set_wand(lv)
        hits, n_out, total = sdb.ExecutePhraseTopKBatch(t["reader"], phrases, scorer, k, rel_pos=rels, filt=filt, exclude=excl)
        assert np.array_equal(total, counts)
        for q, (p, w) in enumerate(zip(phrases, want)):
            c = pr.consts(t["reader"].phrase_stats(scorer, p), scorer.k, scorer.b)
            ref, _ = pr.topk(w, t["norms"], c, k)
            got = hits[q, :n_out[q]]
            assert len(got) == len(ref), (p, lv)
            assert np.array_equal(got["doc"], ref["doc"]) and np.array_equal(got["seg"], ref["seg"]), (p, lv)
            assert np.array_equal(got["score"].view(np.uint32), ref["score"].view(np.uint32)), (p, lv)
    ctx().set_wand(False)
    return counts


def test_counts_and_topk_lengths_1_to_16(tok):
    rng = np.random.default_rng(5)
    phrases = _phrases(tok, rng, 3, range(1, 17)) + [[0, 0], [0, 0, 0], [1, 0, 1, 0], [0, 11], [11]]
    counts = _check(tok, phrases, sdb.BM25(), k=20, levels=(0, 1, 2))
    assert counts[:6].min() > 0 and counts[-2] >= 0


@pytest.mark.parametrize("scorer", [sdb.BM25(), sdb.BM25(1.2, 0.0), sdb.BM25(0.0, 0.75), sdb.TFIDF(False), sdb.TFIDF(True)],
                         ids=["bm25", "bm15", "bm1", "tfidf", "tfidf_norm"])
def test_every_scorer(tok, scorer):
    rng = np.random.default_rng(6)
    _check(tok, _phrases(tok, rng, 4, (1, 2, 3, 5)), scorer, k=7)


def test_one_slot_equals_term_query(tok):
    sc = sdb.BM25()
    ctx().set_wand(0)
    for term in range(V):
        h, n, tot = sdb.ExecutePhraseTopKBatch(tok["reader"], [[term]], sc, 50)
        h2, n2, tot2 = sdb.ExecuteTopKBatch(tok["reader"], [[term]], sdb.AND, sc, 50)
        assert tot[0] == tot2[0] and n[0] == n2[0]
        assert np.array_equal(h[0, :n[0]], h2[0, :n2[0]])
        assert sdb.ExecutePhraseCount(tok["reader"], [term]) == sdb.ExecuteCount(tok["reader"], [term], sdb.AND)
    ctx().set_wand(False)


def test_large_k_ties_and_threshold(tok):
    rng = np.random.default_rng(7)
    phrases = _phrases(tok, rng, 3, (2, 3))
    counts = _check(tok, phrases, sdb.BM25(), k=4096)
    hits, n_out, total = sdb.ExecutePhraseTopKBatch(tok["reader"], phrases, sdb.BM25(), 4096)
    assert n_out.tolist() == counts.tolist() == total.tolist()
    # ties at the cut: many docs share (phrase freq, length), so a small k cuts inside a run of equal scores
    for k in (1, 2, 3, 5, 9):
        _check(tok, phrases[:4], sdb.BM25(), k=k)
    # threshold_in: only scores above it
    h, n, _ = sdb.ExecutePhraseTopKBatch(tok["reader"], phrases[:1], sdb.BM25(), 4096)
    mid = float(h[0, n[0] // 2]["score"])
    h2, n2, _ = sdb.ExecutePhraseTopKBatch(tok["reader"], phrases[:1], sdb.BM25(), 4096, threshold=mid)
    assert np.array_equal(h2[0, :n2[0]], h[0, :n[0]][h[0, :n[0]]["score"] > np.float32(mid)])


def test_gaps(tok):
    rng = np.random.default_rng(8)
    phrases, rels = [], []
    for _ in range(12):
        seq = tok["docs"][0][int(rng.integers(0, 3000))]
        if len(seq) < 6:
            continue
        idx = sorted(rng.choice(len(seq), 3, replace=False).tolist())
        phrases.append([seq[i] for i in idx])
        rels.append([i - idx[0] for i in idx])
    phrases.append([0, 1]); rels.append(None)
    _check(tok, phrases, sdb.BM25(), k=10, rels=rels)


@pytest.mark.parametrize("n_preds", [1, 2, 3, 4])
def test_filter_chains_and_exclusions(tok, n_preds):
    rng = np.random.default_rng(9 + n_preds)
    chain = [(1, "LT", 700), (2, "GT", -5 * 10**8), (3, "LE", 80.0), (4, "NE", 3)][:n_preds]
    filt = [sdb.pred(f, op, v) for f, op, v in chain]
    masks = []
    for c in tok["cols"]:
        m = np.ones(len(c[1][0]), bool)
        for f, op, v in chain:
            x = c[f][0]
            m &= {"LT": x < v, "GT": x > v, "LE": x <= v, "NE": x != v}[op]
        masks.append(m)
    phrases = _phrases(tok, rng, 3, (1, 2, 3))
    excl = [[int(rng.integers(4, 11))] if i % 2 else [] for i in range(len(phrases))]
    _check(tok, phrases, sdb.BM25(), k=15, filt=filt, masks=masks, excl=excl)


def test_batch_4096(tok):
    rng = np.random.default_rng(10)
    phrases = _phrases(tok, rng, 1, (2,)) * 4096
    phrases = phrases[:4096]
    got = sdb.ExecutePhraseCountBatch(tok["reader"], phrases)
    assert got.tolist() == [sum(len(m[0]) for m in _ref_matches(tok, phrases[0]))] * 4096


# ---------------------------------------------------------------- encodings and high doc ids
def _positions_for(lists, rng):
    """Positions for shape lists: a list's posting of freq f gets 0, 2, .., 2(f - 1); its "+lead" companion (freq 1)
    one odd position, so "x x+lead" and "x+lead x" match some of their common docs."""
    posts = []
    for name, d, f in lists:
        if name.endswith("+lead"):
            pos = (2 * rng.integers(0, 4, len(d)) + 1).astype(np.uint32)
        else:
            pos = np.concatenate([np.arange(0, 2 * int(x), 2, dtype=np.uint32) for x in f]) if len(f) else np.zeros(0, np.uint32)
        posts.append((d, f, pos))
    return posts


@pytest.mark.parametrize("width", NORM_WIDTHS)
def test_every_block_encoding(width):
    """Every doc encoding (the shape_corpora.py shapes) and every frequency encoding whose positions fit a test, each list
    followed by its companion. The shapes with more than 200 000 positions are replaced by small lists that reach the same
    frequency encodings (with the 1-byte norm column): one 128-posting block bit-packed at 11..24 bits (its first posting,
    which the companion shares, holds the wide frequency), a block of all-same 16-bit frequencies, a 2-posting tail of
    all-same 32-bit frequencies and a 2-posting raw tail (a frequency of 2^24). Bit-packed widths 25..31 need more than
    2^24 positions in one posting and are left out."""
    _, norms, lists = shape_segment(width)
    pairs = [lists[i:i + 2] for i in range(0, len(lists), 2) if int(lists[i][2].astype(np.uint64).sum()) <= 200_000]
    lists = [x for p in pairs for x in p]
    if width == 1:
        rng = np.random.default_rng(77)
        span = len(norms)
        wide = []
        for w in range(11, 25):
            f = np.ones(128, np.uint32)
            f[0] = 2 ** (w - 1)
            wide.append((f"freq_bits{w}", f))
        wide += [("freq_same16", np.full(128, 300, np.uint32)), ("freq_same32", np.full(2, 70_000, np.uint32)),
                 ("freq_raw_tail", np.array([2 ** 24, 1], np.uint32))]
        for name, f in wide:
            d = np.sort(rng.choice(np.arange(1, span + 1), len(f), replace=False)).astype(np.uint32)
            lists.append((name, d, f))
            lists.append((name + "+lead",) + companion(d, rng, span))
    oseg = orc.Segment(len(norms) if norms is not None else 2 ** 30 + 2 ** 16, has_wand=True)
    if norms is not None:
        oseg.set_norms(norms)
    for _, d, f in lists:
        oseg.add_term(d, f)
    posts = _positions_for(lists, np.random.default_rng(31))
    g = to_gpu(oseg)
    g.stage_positions(*pr.staged_positions(posts))
    dwt = [len(d) for _, d, _ in lists]
    reader = sdb.IndexReader([g], oseg.n_docs, int(norms.astype(np.uint64).sum()) if norms is not None else oseg.n_docs, dwt)
    phrases = []
    for i in range(0, len(lists), 2):
        phrases += [[i, i + 1], [i + 1, i], [i, i], [i]]
    want = [pr.match_postings(posts, p) for p in phrases]
    assert sdb.ExecutePhraseCountBatch(reader, phrases).tolist() == [len(w[0]) for w in want]
    assert sum(len(w[0]) for w in want[0::4]) > 0
    sc = sdb.BM25()
    hits, n_out, total = sdb.ExecutePhraseTopKBatch(reader, phrases, sc, 30)
    assert total.tolist() == [len(w[0]) for w in want]
    for q, p in enumerate(phrases):
        ref, _ = pr.topk([want[q]], [norms], pr.consts(reader.phrase_stats(sc, p), sc.k, sc.b), 30)
        got = hits[q, :n_out[q]]
        assert np.array_equal(got["doc"], ref["doc"]), (lists[p[0]][0], p)
        assert np.array_equal(got["score"].view(np.uint32), ref["score"].view(np.uint32)), (lists[p[0]][0], p)


def test_doc_ids_past_2_31():
    n = (1 << 32) - 2
    rng = np.random.default_rng(41)
    top = np.sort(rng.choice(np.arange(n - 5_000_000, n + 1, dtype=np.int64), 3000, replace=False)).astype(np.uint32)
    low = np.sort(rng.choice(np.arange(1, 1 << 20), 500, replace=False)).astype(np.uint32)
    a = np.unique(np.concatenate([low, top, [1 << 31, (1 << 31) + 1, n]])).astype(np.uint32)
    b = a[rng.random(len(a)) < 0.6]
    b = np.unique(np.concatenate([b, [1 << 31, n]])).astype(np.uint32)
    fa = rng.integers(1, 4, len(a)).astype(np.uint32)
    fb = np.ones(len(b), np.uint32)
    posts = [(a, fa, np.concatenate([np.arange(0, 2 * int(x), 2, dtype=np.uint32) for x in fa])),
             (b, fb, (2 * rng.integers(0, 3, len(b)) + 1).astype(np.uint32))]
    oseg = orc.Segment(n, has_wand=True)
    for d, f, _ in posts:
        oseg.add_term(d, f)
    g = to_gpu(oseg)
    g.stage_positions(*pr.staged_positions(posts))
    g.stage_docs_mask(np.array([n, int(top[5])], np.uint32))
    reader = sdb.IndexReader([g], n, n, [len(a), len(b)])
    phrases = [[0, 1], [1, 0], [0], [0, 0]]
    dels = [n, int(top[5])]
    want = [pr.match_postings(posts, p, deleted=dels) for p in phrases]
    assert sdb.ExecutePhraseCountBatch(reader, phrases).tolist() == [len(w[0]) for w in want]
    sc = sdb.BM25()
    hits, n_out, _ = sdb.ExecutePhraseTopKBatch(reader, phrases, sc, 100)
    for q, p in enumerate(phrases):
        ref, _ = pr.topk([want[q]], [None], pr.consts(reader.phrase_stats(sc, p), sc.k, sc.b), 100)
        assert np.array_equal(hits[q, :n_out[q]]["doc"], ref["doc"])
        assert np.array_equal(hits[q, :n_out[q]]["score"].view(np.uint32), ref["score"].view(np.uint32))


# ---------------------------------------------------------------- errors
def _rc_count(t, terms, rel, off, excl=None, excl_off=None):
    terms = np.ascontiguousarray(terms, np.uint32) if terms is not None else None
    rel = np.ascontiguousarray(rel, np.uint32) if rel is not None else None
    off = np.ascontiguousarray(off, np.uint32)
    counts = np.zeros(len(off) - 1, np.uint64)
    segs = (C.c_void_p * len(t["segs"]))(*[s._h.value for s in t["segs"]])
    ptr = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    return N.lib().sdbg_phrase_count_batch(segs, len(t["segs"]), ptr(terms), ptr(rel), ptr(off), len(off) - 1,
                                           ptr(excl), ptr(excl_off), None, counts.ctypes.data_as(C.c_void_p))


def test_errors(tok):
    inval, unsup, notfound = -1, -7, -5
    launches = ctx().launches
    assert _rc_count(tok, [0, 1], None, [0, 0, 2]) == inval                # empty phrase
    assert _rc_count(tok, [0, 1], None, [0, 2, 1]) == inval                # decreasing offsets
    assert _rc_count(tok, [0, 1], [1, 2], [0, 2]) == inval                 # rel_pos not starting at 0
    assert _rc_count(tok, [0, 1], [0, 0], [0, 2]) == inval                 # not increasing
    assert _rc_count(tok, None, None, [0, 2]) == inval                     # NULL terms
    assert _rc_count(tok, list(range(17)), None, [0, 17]) == unsup         # 17 slots
    assert _rc_count(tok, [0], None, [0, 1], np.arange(17, dtype=np.uint32) % V, np.array([0, 17], np.uint32)) == unsup
    assert _rc_count(tok, [0, 99], None, [0, 2]) == inval                  # term id out of range
    assert ctx().launches == launches
    # a segment without positions
    oseg = orc.Segment(100, has_wand=True)
    oseg.add_term(np.array([1, 2], np.uint32), np.array([1, 1], np.uint32))
    g = to_gpu(oseg)
    r = sdb.IndexReader([g], 100, 100, [2])
    with pytest.raises(N.SdbgError, match="ENOTFOUND"):
        sdb.ExecutePhraseCountBatch(r, [[0]])
    with pytest.raises(N.SdbgError, match="ENOTFOUND"):
        sdb.ExecutePhraseTopKBatch(r, [[0]], sdb.BM25(), 5)
    with pytest.raises(N.SdbgError, match="EUNSUPPORTED"):
        sdb.ExecutePhraseTopKBatch(tok["reader"], [[0]], sdb.BM25(), 4097)


def test_staging_checks():
    oseg = orc.Segment(10, has_wand=True)
    oseg.add_term(np.array([1, 3], np.uint32), np.array([2, 1], np.uint32))
    oseg.add_term(np.array([2], np.uint32), np.array([1], np.uint32))
    g = to_gpu(oseg)
    good = (np.array([0, 4, 7, 2], np.uint32), np.array([0, 3, 4], np.uint64))
    g.stage_positions(*good)
    with pytest.raises(N.SdbgError, match="EFORMAT"):
        g.stage_positions(np.array([0, 4, 7], np.uint32), np.array([0, 2, 3], np.uint64))     # wrong count
    with pytest.raises(N.SdbgError, match="EFORMAT"):
        g.stage_positions(np.array([4, 4, 7, 2], np.uint32), np.array([0, 3, 4], np.uint64))  # not ascending
    with pytest.raises(N.SdbgError, match="EINVAL"):
        g.stage_positions(good[0], np.array([0, 3], np.uint64))                              # n_terms differs
    r = sdb.IndexReader([g], 10, 10, [2, 1])
    # the failed restagings kept the good positions: doc 1 holds term 0 at 0 and 4
    assert sdb.ExecutePhraseCount(r, [0]) == 2
    assert sdb.ExecutePhraseCount(r, [0, 0], rel_pos=[0, 4]) == 1
    s = sdb.Segment(ctx(), 10)
    with pytest.raises(N.SdbgError, match="EINVAL"):
        s.stage_positions(*good)                                                           # before the postings


def _selftest_corpus(n_docs):
    """The token corpus of adapter_selftest's "phrase" mode, rebuilt from its generator."""
    state, docs = 12345, []
    def nxt():
        nonlocal state
        state = (state * 1664525 + 1013904223) & 0xFFFFFFFF
        return state >> 16
    for _ in range(n_docs):
        n = 1 + nxt() % 16
        docs.append([nxt() % 6 for _ in range(n)])
    return docs


def test_adapters_phrase_mode():
    """GpuTopKIterator and GpuCountScan with phrase_positions against the NumPy statement, scored with the phrase's
    statistics computed here by hand: the slots' BM25 idfs summed in float32."""
    import json
    import subprocess
    from serenedb_b200 import build as b

    exe = b.build_adapters()
    n = 20_000
    res = subprocess.run([exe, str(n), "phrase"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = [json.loads(l) for l in res.stdout.strip().splitlines()]
    assert len(lines) == 2
    docs = _selftest_corpus(n)
    norms = np.array([len(d) for d in docs], np.uint32)
    post = pr.postings(docs, 6)
    sc = sdb.BM25()
    for x in lines:
        ds, fs = pr.match(docs, x["slots"], x["rel"], x["excl"])
        assert x["count"] == x["total"] == len(ds) > 0
        idf = np.float32(0)
        for t in x["slots"]:
            idf = np.float32(idf + np.float32(sc.collect(n, int(norms.sum()), len(post[t][0])).idf))
        st = sc.collect(n, int(norms.sum()), len(post[x["slots"][0]][0]))
        c0 = np.float32(np.float32(np.float32(1.0) * np.float32(np.float32(1.2) + np.float32(1))) * idf)
        ref, _ = pr.topk([(ds, fs)], [norms], (c0, np.float32(st.norm_const), np.float32(st.norm_length)), 50)
        got = np.array([h[0] for h in x["topk"]], np.uint32)
        scores = np.array([h[1] for h in x["topk"]], np.float32)
        assert np.array_equal(got, ref["doc"]), x["slots"]
        assert np.array_equal(scores.view(np.uint32), ref["score"].view(np.uint32)), x["slots"]
