"""Reference results for queries with excluded terms (`a & b & !c`), built on the CPU oracle without changing it.

Excluding a term removes the docs of its list from the matches: they are neither collected nor counted, and the positive
terms' scores of the other docs are untouched. That is exactly what the oracle does with a segment's deleted docs
(MaskDocIterator semantics), so the reference masks, per segment, the union of the deleted docs and of the excluded
lists -- decoded through the oracle's own reader -- and runs the oracle's exhaustive evaluation. An excluded id that a
segment does not hold excludes nothing there. The masks are restored afterwards.

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np

import orc


def excluded_docs(oseg, exclude):
    """Union of the doc lists of the excluded term ids the segment holds (uint32, sorted)."""
    out = np.zeros(0, np.uint32)
    for t in exclude:
        if int(t) < oseg.num_terms():
            out = np.union1d(out, oseg.decode_term(int(t))[0])
    return out.astype(np.uint32)


def topk_excl(osegs, kind, terms, exclude, k, k1=1.2, b=0.75, filt=None, deleted=None, mode=1):
    """orc.bm25_topk of the positive terms minus the docs of `exclude` (term ids). deleted: per segment the deleted docs
    it carries (None: none). mode: 0 or 1, both exhaustive. Returns (hits, total_matches)."""
    assert mode in (0, 1), "mode 2 prunes regardless of the mask: not a reference for exclusions"
    deleted = deleted or [None] * len(osegs)
    try:
        for o, dele in zip(osegs, deleted):
            base = np.zeros(0, np.uint32) if dele is None else np.asarray(dele, np.uint32)
            o.set_docs_mask(np.union1d(base, excluded_docs(o, exclude)).astype(np.uint32))
        hits, total, _ = orc.bm25_topk(osegs, kind, terms, k, k1=k1, filt=filt, mode=mode, b=b)
    finally:
        for o, dele in zip(osegs, deleted):
            o.set_docs_mask(np.zeros(0, np.uint32) if dele is None else np.asarray(dele, np.uint32))
    return hits, total


def topk_batch_excl(osegs, kind, queries_terms, excludes, k, **kw):
    """One topk_excl per query: (hits [Q, k], n_out [Q], total [Q])."""
    nq = len(queries_terms)
    hits = np.zeros((nq, k), dtype=orc.HIT_DTYPE)
    n_out = np.zeros(nq, np.uint32)
    total = np.zeros(nq, np.uint64)
    for q, (terms, excl) in enumerate(zip(queries_terms, excludes)):
        h, t = topk_excl(osegs, kind, terms, excl, k, **kw)
        hits[q, :len(h)] = h
        n_out[q], total[q] = len(h), t
    return hits, n_out, total
