"""NumPy statement of exact phrase queries (sdbg_phrase_count_batch / sdbg_phrase_topk_batch) over token-sequence
corpora: a doc is a sequence of term ids, a term's positions in it are the indexes where it occurs. A phrase is slots
(term t_i at relative position r_i, r_0 = 0, increasing); doc d matches when some anchor p has p + r_i among t_i's
positions for every slot, d is not deleted, passes the mask and holds no excluded term. The phrase frequency counts the
anchors (overlaps included); the score is bm25(phrase frequency, norm) in float32 with plain float32 operations in the
device's order. Restated from the semantics (no reference golden exists for phrases).

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np


def postings(docs, n_terms):
    """Token sequences (docs[i] is doc i + 1) -> per term (doc ids, freqs, positions in posting order)."""
    occ = [dict() for _ in range(n_terms)]
    for i, seq in enumerate(docs):
        for p, t in enumerate(seq):
            occ[t].setdefault(i + 1, []).append(p)
    out = []
    for t in range(n_terms):
        ds = sorted(occ[t])
        out.append((np.array(ds, np.uint32), np.array([len(occ[t][d]) for d in ds], np.uint32),
                    np.array([p for d in ds for p in occ[t][d]], np.uint32)))
    return out


def staged_positions(post):
    """The arguments of sdbg_stage_positions for postings(): (positions, term_pos_off)."""
    off = np.zeros(len(post) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for _, _, p in post])
    pos = np.concatenate([p for _, _, p in post]) if post else np.zeros(0, np.uint32)
    return pos.astype(np.uint32), off


def phrase_freq(seq, terms, rel=None):
    """Phrase frequency of one doc (a token sequence)."""
    rel = list(range(len(terms))) if rel is None else list(rel)
    seq = list(seq)
    return sum(1 for p in range(len(seq)) if all(p + r < len(seq) and seq[p + r] == t for t, r in zip(terms, rel)))


def match(docs, terms, rel=None, excl=(), deleted=None, mask=None):
    """(doc ids, phrase freqs) of one segment's matches, ascending by doc."""
    dels = set() if deleted is None else {int(d) for d in deleted}
    ex = {int(t) for t in excl}
    ds, fs = [], []
    for i, seq in enumerate(docs):
        d = i + 1
        if d in dels or (mask is not None and not mask[i]) or ex.intersection(seq):
            continue
        f = phrase_freq(seq, terms, rel)
        if f:
            ds.append(d)
            fs.append(f)
    return np.array(ds, np.uint32), np.array(fs, np.uint32)


def match_postings(post, terms, rel=None, excl=(), deleted=None, mask=None):
    """match() over postings() triples instead of token sequences: (doc ids, phrase freqs) of one segment."""
    rel = list(range(len(terms))) if rel is None else list(rel)
    by_term = {}
    for t in set(terms):
        docs, freqs, pos = post[t]
        ends = np.cumsum(freqs.astype(np.int64))
        by_term[t] = {int(d): pos[e - f:e].astype(np.int64) for d, f, e in zip(docs, freqs, ends)}
    cand = set.intersection(*(set(by_term[t]) for t in terms))
    for t in excl:
        if int(t) < len(post):
            cand -= set(post[int(t)][0].tolist())
    if deleted is not None:
        cand -= {int(d) for d in deleted}
    if mask is not None:
        cand = {d for d in cand if mask[d - 1]}
    ds, fs = [], []
    for d in sorted(cand):
        anchors = by_term[terms[0]][d]
        ok = np.ones(len(anchors), bool)
        for t, r in zip(terms, rel):
            ok &= np.isin(anchors + r, by_term[t][d])
        f = int(ok.sum())
        if f:
            ds.append(d)
            fs.append(f)
    return np.array(ds, np.uint32), np.array(fs, np.uint32)


def count(seg_docs, terms, rel=None, excl=(), deleted=None, masks=None):
    n = len(seg_docs)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    return sum(len(match(d, terms, rel, excl, x, m)[0]) for d, x, m in zip(seg_docs, deleted, masks))


def score(freq, norm, c0, nc, nl):
    """bm25() of bm25_kernels.cuh in float32 with its operation order, every form (NaN markers as fill_qterm sets them)."""
    f32 = np.float32
    freq, norm = f32(freq), f32(norm)
    if nc != nc:                                   # TFIDF
        r = f32(np.sqrt(freq)) * f32(c0)
        return f32(r / f32(np.sqrt(norm))) if nl != 0 else f32(r)
    if nl != nl:                                   # BM15
        return f32(f32(c0) - f32(c0) / f32(f32(1) + f32(freq / f32(nc))))
    c1 = f32(f32(nc) + f32(f32(nl) * norm))
    return f32(f32(c0) - f32(f32(f32(c0) * c1) / f32(c1 + freq)))


def consts(stats, k1, b):
    """(c0, norm_const, norm_length) of a phrase's statistics under the scorer (k1, b), as fill_qterm derives them."""
    f32 = np.float32
    if k1 == -1:
        return f32(f32(stats.boost) * f32(stats.idf)), float("nan"), (1.0 if b != 0 else 0.0)
    if k1 == 0:
        return f32(0), f32(stats.norm_const), f32(stats.norm_length)
    c0 = f32(f32(f32(stats.boost) * f32(f32(k1) + f32(1))) * f32(stats.idf))
    return c0, f32(stats.norm_const), (float("nan") if b == 0 else f32(stats.norm_length))


def topk(seg_matches, seg_norms, c, k, threshold=np.float32(1.1754944e-38)):
    """The k best (score desc, segment asc, doc asc) of the matches scoring > threshold, as a structured array, and the
    match count. seg_matches: per segment (doc ids, phrase freqs) from match() / match_postings(); seg_norms: per segment
    the norms by row (doc - 1), or None for norm 1."""
    rows, total = [], 0
    for si, ((ds, fs), norms) in enumerate(zip(seg_matches, seg_norms)):
        total += len(ds)
        for d, f in zip(ds, fs):
            s = score(f, 1 if norms is None else norms[d - 1], *c)
            if s > np.float32(threshold):
                rows.append((np.float32(s), int(d), si))
    rows.sort(key=lambda r: (-r[0], r[2], r[1]))
    out = np.zeros(min(k, len(rows)), [("score", "<f4"), ("doc", "<u4"), ("seg", "<u4")])
    for i, r in enumerate(rows[:k]):
        out[i] = r
    return out, total
