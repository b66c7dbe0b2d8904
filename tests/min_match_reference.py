"""Reference results for OR groups with a minimum match count (`2 of (a | b | c) & d`), built on the CPU oracle without
changing it, the way tests/groups_reference.py builds them for plain OR groups.

Group g of such a query holds a doc when at least mins[g] of its posting lists hold it (None: 1 for every group, which
is exactly the groups_reference statement). A query matches the docs of the flat OR of its positive terms that every
group holds and no excluded list holds, and scores each of them as that flat OR does. So the reference decodes the
positive and excluded lists through the oracle's own reader, masks per segment every doc of the OR that fails a group or
hits an exclusion -- together with the segment's deleted docs -- and runs the oracle's exhaustive evaluation of the flat
OR. The masks are restored afterwards. `match_docs` is the plain NumPy statement of the matching doc set, for counts.

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np

import orc
from excl_reference import excluded_docs


def _docs(oseg, t):
    return oseg.decode_term(int(t))[0].astype(np.uint32) if int(t) < oseg.num_terms() else np.zeros(0, np.uint32)


def _group_docs(lists_of_group, m):
    """Docs that at least m of the group's doc lists (each without repeats) hold."""
    docs, hits = np.unique(np.concatenate([np.asarray(d, np.uint32) for d in lists_of_group]), return_counts=True)
    return docs[hits >= m]


def rejected_docs(oseg, group_ids, exclude, mins=None):
    """Docs of the flat OR of the groups' term ids that fail a group or occur in an excluded list (uint32, sorted)."""
    mins = mins or [1] * len(group_ids)
    glists = [[_docs(oseg, t) for t in g] for g in group_ids]
    gdocs = [_group_docs(l, m) for l, m in zip(glists, mins)]
    union = np.unique(np.concatenate([d for l in glists for d in l])) if glists else np.zeros(0, np.uint32)
    keep = union
    for d in gdocs:
        keep = np.intersect1d(keep, d)
    return np.union1d(np.setdiff1d(union, keep), excluded_docs(oseg, exclude)).astype(np.uint32)


def topk_groups(osegs, groups, exclude, k, k1=1.2, b=0.75, filt=None, deleted=None, mode=1, mins=None):
    """orc.bm25_topk of the flat OR of `groups` (lists of orc.BM25Term) restricted to the docs every group holds (at least
    mins[g] of its lists, default 1), minus the docs of `exclude` (term ids). deleted: per segment the deleted docs it
    carries (None: none). mode: 0 or 1, both exhaustive. Returns (hits, total_matches)."""
    assert mode in (0, 1), "mode 2 prunes regardless of the mask: not a reference for per-doc checks"
    deleted = deleted or [None] * len(osegs)
    group_ids = [[t.term for t in g] for g in groups]
    flat = [t for g in groups for t in g]
    try:
        for o, dele in zip(osegs, deleted):
            base = np.zeros(0, np.uint32) if dele is None else np.asarray(dele, np.uint32)
            o.set_docs_mask(np.union1d(base, rejected_docs(o, group_ids, exclude, mins)).astype(np.uint32))
        hits, total, _ = orc.bm25_topk(osegs, "OR", flat, k, k1=k1, filt=filt, mode=mode, b=b)
    finally:
        for o, dele in zip(osegs, deleted):
            o.set_docs_mask(np.zeros(0, np.uint32) if dele is None else np.asarray(dele, np.uint32))
    return hits, total


def topk_batch_groups(osegs, queries, excludes, k, min_match=None, **kw):
    """One topk_groups per query (min_match: per query its groups' minimums, or None): (hits [Q, k], n_out [Q], total [Q])."""
    nq = len(queries)
    hits = np.zeros((nq, k), dtype=orc.HIT_DTYPE)
    n_out = np.zeros(nq, np.uint32)
    total = np.zeros(nq, np.uint64)
    min_match = min_match or [None] * nq
    for q, (groups, excl) in enumerate(zip(queries, excludes)):
        h, t = topk_groups(osegs, groups, excl or [], k, mins=min_match[q], **kw)
        hits[q, :len(h)] = h
        n_out[q], total[q] = len(h), t
    return hits, n_out, total


def match_docs(lists, groups, excl=(), deleted=None, mask=None, mins=None):
    """NumPy statement: docs of one segment that a query of OR groups matches. lists: doc arrays by term id (the segment's
    terms); groups: lists of term ids; mask: bool per row (row = doc - 1) of the filter, or None; mins: per group the
    number of its lists that must hold a doc (None: 1)."""
    docs = None
    for g, m in zip(groups, mins or [1] * len(groups)):
        gd = _group_docs([np.unique(np.asarray(lists[t], np.uint32)) if t < len(lists) else np.zeros(0, np.uint32) for t in g], m)
        docs = gd if docs is None else np.intersect1d(docs, gd)
    for t in excl:
        if int(t) < len(lists):                 # an id the segment does not hold excludes nothing
            docs = np.setdiff1d(docs, lists[int(t)])
    if deleted is not None and len(deleted):
        docs = np.setdiff1d(docs, np.asarray(deleted, np.uint32))
    if mask is not None:
        docs = docs[mask[docs.astype(np.int64) - 1]]
    return docs.astype(np.uint32)


def count(seg_lists, groups, excl=(), deleted=None, masks=None, mins=None):
    """Count summed over segments; seg_lists / deleted / masks are per segment (None entries: none)."""
    n = len(seg_lists)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    return sum(len(match_docs(l, groups, excl, d, m, mins)) for l, d, m in zip(seg_lists, deleted, masks))
