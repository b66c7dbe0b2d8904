"""Python statement of the aggregates over a full-text query's matches (sdbg_match_aggregate_batch(_groups_min), `SELECT
col, count(*), count(v), sum(v), avg(v), min(v), max(v) ... WHERE body @@ '...' GROUP BY col`): the docs
count_reference.match_docs / min_match_reference.match_docs give per segment, grouped by the keys facet_reference.keys_of
gives (or all in one group), and the value of each doc's row (row = doc - 1; a doc past the value column's rows, or whose
row is NULL, has a NULL value).

A cell is dict(count, count_value, sum, min, max), and for float64 columns abs: the exact sum of |v| over the finite
values, which bounds the rounding error of a float64 sum in any order (count_value * 2^-52 * abs). Integer sums are exact Python ints; float64 sums follow IEEE rules (NaN
if any value is NaN or both infinities occur, else the infinity that occurs, else math.fsum of the values). MIN / MAX of
float64 values use the sorted scan's order: -0.0 equals +0.0 and comes back as +0.0, every NaN equals every NaN, sorts
above +inf and comes back as NaN. A cell without values has sum, min and max 0.

TEST INFRASTRUCTURE: imported by tests only."""
import math

import numpy as np

import count_reference as cr
import facet_reference as fr
import min_match_reference as mr


def empty_cell(is_float):
    if is_float:
        return dict(count=0, count_value=0, sum=0.0, min=0.0, max=0.0, abs=0.0)
    return dict(count=0, count_value=0, sum=0, min=0, max=0)


def float_sum(vals):
    """IEEE sum of float64 values, exact in the finite part."""
    if any(math.isnan(v) for v in vals):
        return math.nan
    pinf, ninf = math.inf in vals, -math.inf in vals
    if pinf and ninf:
        return math.nan
    if pinf or ninf:
        return math.inf if pinf else -math.inf
    return math.fsum(vals)


def _order(v):
    """The sorted scan's order of a float64: NaN above +inf; -0.0 == +0.0 compares equal already."""
    return (1, 0.0) if math.isnan(v) else (0, v)


def _canon(v):
    return math.nan if math.isnan(v) else (0.0 if v == 0.0 else v)


def cell_of(values, is_float, n_null=0):
    """The cell of a group: `values` its non-NULL values, n_null its docs with a NULL value."""
    vals = np.asarray(values, np.float64 if is_float else np.int64)
    c = empty_cell(is_float)
    c["count"] = len(vals) + int(n_null)
    c["count_value"] = len(vals)
    if len(vals):
        if is_float:
            c["sum"] = float_sum(vals.tolist())
            c["abs"] = math.fsum(np.abs(vals[np.isfinite(vals)]).tolist())
            nan = np.isnan(vals)
            c["max"] = math.nan if nan.any() else _canon(float(vals.max()))
            c["min"] = math.nan if nan.all() else _canon(float(vals[~nan].min()))
        else:   # exact: two int64 limbs that cannot overflow for fewer than 2^31 values
            c["sum"] = int((vals >> 32).sum()) * 2 ** 32 + int((vals & 0xFFFFFFFF).sum())
            c["min"], c["max"] = int(vals.min()), int(vals.max())
    return c


def merge(a, b, is_float):
    """The cell of the union of two groups' docs."""
    if not b["count_value"]:
        return dict(a, count=a["count"] + b["count"])
    if not a["count_value"]:
        return dict(b, count=a["count"] + b["count"])
    c = dict(count=a["count"] + b["count"], count_value=a["count_value"] + b["count_value"])
    if is_float:
        c["sum"] = float_sum([a["sum"], b["sum"]])
        c["abs"] = a["abs"] + b["abs"]
        c["min"] = min(a["min"], b["min"], key=_order)
        c["max"] = max(a["max"], b["max"], key=_order)
    else:
        c["sum"], c["min"], c["max"] = a["sum"] + b["sum"], min(a["min"], b["min"]), max(a["max"], b["max"])
    return c


def values_of(docs, values, valid=None):
    """Value per doc: (values, is_null), the values typed as the column (0 where NULL)."""
    values = np.asarray(values)
    r = np.asarray(docs, np.int64) - 1
    ok = r < len(values)
    if valid is not None:
        ok[ok] &= np.asarray(valid, bool)[r[ok]]
    v = np.zeros(len(r), values.dtype)
    v[ok] = values[r[ok]]
    return v, ~ok


def cells_of_docs(seg_docs, key_columns, val_columns, key_min, key_span):
    """(cells [key_span], NULL-key cell) of per-segment matching docs. key_columns None: ungrouped (key_span must be 1 and
    the NULL-key cell stays empty); else per segment (values, valid or None). val_columns: per segment (values, valid or
    None). Raises ValueError when a matching doc's non-NULL key lies outside [key_min, key_min + key_span)."""
    is_float = np.asarray(val_columns[0][0]).dtype == np.float64
    bins, vals, vnull = [], [], []
    for si, docs in enumerate(seg_docs):
        v, v_null = values_of(docs, *val_columns[si])
        if key_columns is None:
            b = np.zeros(len(docs), np.int64)
        else:
            k, k_null = fr.keys_of(docs, *key_columns[si])
            rel = k[~k_null].astype(object) - int(key_min)   # exact for every int64 key and key_min
            if any(x < 0 or x >= key_span for x in set(rel.tolist())):
                raise ValueError("key outside the range")
            b = np.full(len(docs), key_span, np.int64)
            b[~k_null] = np.asarray(rel, np.int64)
        bins.append(b)
        vals.append(v.astype(np.float64 if is_float else np.int64))
        vnull.append(v_null)
    b, v, vn = np.concatenate(bins), np.concatenate(vals), np.concatenate(vnull)
    order = np.argsort(b, kind="stable")
    b, v, vn = b[order], v[order], vn[order]
    bounds = np.searchsorted(b, np.arange(key_span + 2))
    cells = []
    for key in range(key_span + 1):
        lo, hi = bounds[key], bounds[key + 1]
        cells.append(cell_of(v[lo:hi][~vn[lo:hi]], is_float, int(vn[lo:hi].sum())))
    return cells[:key_span], cells[key_span]


def aggregate(seg_lists, kind, pos, key_columns, val_columns, key_min=0, key_span=1, excl=(), deleted=None, masks=None):
    """(cells [key_span], NULL-key cell) of one flat query (count_reference.match_docs)."""
    n = len(seg_lists)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    docs = [cr.match_docs(l, kind, pos, excl, d, m) for l, d, m in zip(seg_lists, deleted, masks)]
    return cells_of_docs(docs, key_columns, val_columns, key_min, key_span)


def aggregate_groups(seg_lists, groups, key_columns, val_columns, key_min=0, key_span=1, excl=(), deleted=None, masks=None,
                     mins=None):
    """(cells [key_span], NULL-key cell) of one query of OR groups (min_match_reference.match_docs)."""
    n = len(seg_lists)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    docs = [mr.match_docs(l, groups, excl, d, m, mins) for l, d, m in zip(seg_lists, deleted, masks)]
    return cells_of_docs(docs, key_columns, val_columns, key_min, key_span)
