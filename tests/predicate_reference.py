"""Exact statement of what one pushed column predicate (sdbg_col_pred, built by engine.pred) selects, for every column type
and constant, in plain Python arithmetic.

- NULL never passes, except under IS_NULL; IS_NOT_NULL passes exactly the valid rows.
- Integer columns (int32, int64, int64 staged bit-packed): the exact mathematical comparison of the integer with the
  constant, whether the constant is an int or a float. The values are compared as Python ints with the constant as a
  Python int or float, which Python does exactly (never through float64). So a NaN constant is false for every op
  except NE, where it is true; v < inf and v < 2**63 always hold; v == 1e30 never does.
- Double columns: IEEE comparison with the constant converted to the nearest double first, as DuckDB casts the constant
  to the column type (an int constant above 2**53 is rounded; one beyond the double range becomes +-inf). NaN compares
  false, except NE, where it is true; -0.0 == +0.0.
- BETWEEN lo, hi is v >= lo AND v <= hi, so lo > hi selects nothing.

TEST INFRASTRUCTURE: imported by tests only."""
import math

import numpy as np

OPS = ("LT", "LE", "GT", "GE", "EQ", "NE", "BETWEEN", "IS_NULL", "IS_NOT_NULL")


def constant(x):
    """A predicate constant as an exact Python number: a float stays a float (NumPy floats widen exactly), an integer
    becomes a Python int."""
    if isinstance(x, (float, np.floating)):
        return float(x)
    return int(x)


def as_double(x):
    """The constant converted to the double a double column is compared with (nearest; +-inf beyond the range)."""
    x = constant(x)
    try:
        return float(x)
    except OverflowError:
        return math.inf if x > 0 else -math.inf


def _compare(v, op, lo, hi):
    if op == "LT":
        return v < lo
    if op == "LE":
        return v <= lo
    if op == "GT":
        return v > lo
    if op == "GE":
        return v >= lo
    if op == "EQ":
        return v == lo
    if op == "NE":
        return v != lo
    if op == "BETWEEN":
        return (v >= lo) & (v <= hi)
    raise ValueError(op)


def pass_mask(values, valid, op, lo=0, hi=0):
    """Bool per row: does the row pass `column op lo` (BETWEEN: lo <= column <= hi)? values: int32 / int64 / float64
    array; valid: bool per row, or None for a NOT NULL column."""
    values = np.asarray(values)
    valid = np.ones(len(values), bool) if valid is None else np.asarray(valid, bool)
    if op == "IS_NULL":
        return ~valid
    if op == "IS_NOT_NULL":
        return valid.copy()
    with np.errstate(invalid="ignore"):      # comparisons with NaN are false (NE: true) without a warning
        if values.dtype == np.float64:
            out = _compare(values, op, np.float64(as_double(lo)), np.float64(as_double(hi)))
        elif values.dtype in (np.int64, np.int32):
            obj = values.astype(object)      # Python ints: int-vs-int and int-vs-float comparisons are exact
            out = np.asarray(_compare(obj, op, constant(lo), constant(hi)), bool)
        else:
            raise TypeError(values.dtype)
    return valid & np.asarray(out, bool)


def pass_mask_all(columns, preds):
    """Conjunction of predicates. columns: {field: (values, valid or None)}; preds: (field, op[, lo[, hi]]) tuples.
    No predicate: every row passes."""
    rows = len(next(iter(columns.values()))[0])
    out = np.ones(rows, bool)
    for field, op, *bounds in preds:
        values, valid = columns[field]
        out &= pass_mask(values, valid, op, *bounds)
    return out
