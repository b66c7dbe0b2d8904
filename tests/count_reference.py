"""NumPy statement of what the Count mode of the search scan counts, built from the raw doc lists: the positive part's
matches (union for OR, intersection for AND), minus the segment's deleted docs, minus the docs of the excluded term ids
the segment holds, restricted to the docs whose row passes the pushed column predicate (a NULL fails every comparison;
IS_NULL passes exactly the NULLs). Counts are summed over the segments.

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np

OPS = dict(LT=0, LE=1, GT=2, GE=3, EQ=4, NE=5, BETWEEN=6, IS_NULL=7, IS_NOT_NULL=8)


def pred_mask(values, valid, op, lo=0, hi=0):
    """Boolean pass mask per row (row = doc - 1). valid: bool per row, or None for a NOT NULL column."""
    values = np.asarray(values)
    valid = np.ones(len(values), bool) if valid is None else np.asarray(valid, bool)
    if op == "IS_NULL":
        return ~valid
    if op == "IS_NOT_NULL":
        return valid
    cmp = {"LT": values < lo, "LE": values <= lo, "GT": values > lo, "GE": values >= lo, "EQ": values == lo,
           "NE": values != lo, "BETWEEN": (values >= lo) & (values <= hi)}[op]
    return valid & cmp


def validity_words(valid):
    """Bool per row -> the staged validity bitmap (uint64 words, bit r = row r is not NULL)."""
    valid = np.asarray(valid, bool)
    b = np.zeros((len(valid) + 63) // 64 * 8, np.uint8)
    packed = np.packbits(valid, bitorder="little")
    b[:len(packed)] = packed
    return b.view("<u8").astype(np.uint64)


def match_docs(lists, kind, pos, excl=(), deleted=None, mask=None):
    """Docs of one segment that the query counts. lists: doc arrays by term id (the segment's terms)."""
    sets = [np.asarray(lists[t], np.uint32) for t in pos]
    docs = sets[0]
    for s in sets[1:]:
        docs = np.union1d(docs, s) if kind in ("OR", 0) else np.intersect1d(docs, s)
    for t in excl:
        if int(t) < len(lists):                 # an id the segment does not hold excludes nothing
            docs = np.setdiff1d(docs, lists[int(t)])
    if deleted is not None and len(deleted):
        docs = np.setdiff1d(docs, np.asarray(deleted, np.uint32))
    if mask is not None:
        docs = docs[mask[docs.astype(np.int64) - 1]]
    return docs.astype(np.uint32)


def count(seg_lists, kind, pos, excl=(), deleted=None, masks=None):
    """Count summed over segments; seg_lists / deleted / masks are per segment (None entries: none)."""
    n = len(seg_lists)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    return sum(len(match_docs(l, kind, pos, excl, d, m)) for l, d, m in zip(seg_lists, deleted, masks))
