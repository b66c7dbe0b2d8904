"""NumPy statement of the sorted scan (sdbg_match_topk_by_column_batch, `WHERE body @@ '...' ORDER BY col LIMIT k`): the
docs count_reference.match_docs gives per segment, ordered by (NULL placement, normalised value, direction, segment,
doc). Row = doc - 1; a doc past the column's rows is NULL. Values ascend or descend; NULLs all come first or all last;
ties, NULLs included, go by (segment asc, doc asc) in both directions. float64: -0.0 equals +0.0, every NaN equals
every NaN and sorts above +inf. The value returned is the stored one, bit for bit.

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np

import count_reference as cr

SIGN = np.uint64(1 << 63)


def value_order(values):
    """Stored values -> uint64 whose ascending order is the sort's ascending order (equal values map to one key)."""
    values = np.asarray(values)
    if values.dtype == np.float64:
        bits = values.view(np.uint64).copy()
        bits[np.isnan(values)] = np.uint64(0x7FF8000000000000)
        bits[bits == SIGN] = np.uint64(0)
        return np.where(bits & SIGN, ~bits, bits | SIGN)
    return values.astype(np.int64).view(np.uint64) ^ SIGN


def sorted_hits(seg_lists, kind, pos, columns, descending=False, nulls_first=False, k=None, excl=(), deleted=None,
                masks=None):
    """All matches (or the first k) in sort order. columns: per segment (values, valid bool per row or None).
    Returns dict of arrays: values (stored dtype; 0 for NULL), docs, segs, nulls."""
    n = len(seg_lists)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    dtype = np.asarray(columns[0][0]).dtype
    parts = []
    for si, (lists, dele, mask, (vals, valid)) in enumerate(zip(seg_lists, deleted, masks, columns)):
        docs = cr.match_docs(lists, kind, pos, excl, dele, mask)
        vals = np.asarray(vals)
        r = docs.astype(np.int64) - 1
        inside = r < len(vals)
        ok = inside.copy()
        if valid is not None:
            ok[inside] &= np.asarray(valid, bool)[r[inside]]
        v = np.zeros(len(docs), dtype)
        v[ok] = vals[r[ok]]
        parts.append((v, docs, np.full(len(docs), si, np.uint32), ~ok))
    values = np.concatenate([p[0] for p in parts])
    docs = np.concatenate([p[1] for p in parts])
    segs = np.concatenate([p[2] for p in parts])
    nulls = np.concatenate([p[3] for p in parts])
    vkey = value_order(values)
    if descending:
        vkey = ~vkey
    vkey[nulls] = 0
    group = np.where(nulls, 0 if nulls_first else 1, 1 if nulls_first else 0)
    o = np.lexsort((docs, segs, vkey, group))[:k]
    return dict(values=values[o], docs=docs[o], segs=segs[o], nulls=nulls[o])
