"""NumPy statement of the facet counts (sdbg_match_facet_counts_batch, `SELECT col, count(*) ... WHERE body @@ '...' GROUP BY
col`): the docs count_reference.match_docs gives per segment, counted per value of the key column. Row = doc - 1; a doc
past the column's rows, or whose row is NULL, has a NULL key, and all NULL keys form one group. Counts are summed over
the segments, so sum(counts) + nulls equals count_reference.count.

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np

import count_reference as cr


def keys_of(docs, values, valid=None):
    """Key per doc: (int64 values, bool is_null). values / valid are per row (valid None: NOT NULL)."""
    values = np.asarray(values)
    r = np.asarray(docs, np.int64) - 1
    ok = r < len(values)
    if valid is not None:
        ok[ok] &= np.asarray(valid, bool)[r[ok]]
    v = np.zeros(len(r), np.int64)
    v[ok] = values[r[ok]].astype(np.int64)
    return v, ~ok


def facet_counts(seg_lists, kind, pos, columns, key_min, key_span, excl=(), deleted=None, masks=None):
    """(counts uint64[key_span], nulls) of one query. columns: per segment (values, valid bool per row or None).
    Raises ValueError when a counted doc's non-NULL key lies outside [key_min, key_min + key_span)."""
    n = len(seg_lists)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    counts = np.zeros(key_span, np.uint64)
    nulls = 0
    for lists, dele, mask, (vals, valid) in zip(seg_lists, deleted, masks, columns):
        docs = cr.match_docs(lists, kind, pos, excl, dele, mask)
        v, is_null = keys_of(docs, vals, valid)
        nulls += int(is_null.sum())
        bins = v[~is_null].astype(object) - int(key_min)   # exact for every int64 key and key_min
        if any(b < 0 or b >= key_span for b in set(bins.tolist())):
            raise ValueError("key outside the range")
        counts += np.bincount(np.asarray(bins, np.int64), minlength=key_span).astype(np.uint64)
    return counts, nulls


def facet_dict(seg_lists, kind, pos, columns, excl=(), deleted=None, masks=None):
    """{key: count} of the keys with matches, plus {None: n} when n > 0 matches have a NULL key."""
    n = len(seg_lists)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    out = {}
    for lists, dele, mask, (vals, valid) in zip(seg_lists, deleted, masks, columns):
        v, is_null = keys_of(cr.match_docs(lists, kind, pos, excl, dele, mask), vals, valid)
        for key, c in zip(*np.unique(v[~is_null], return_counts=True)):
            out[int(key)] = out.get(int(key), 0) + int(c)
        if is_null.any():
            out[None] = out.get(None, 0) + int(is_null.sum())
    return out
