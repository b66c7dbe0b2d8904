"""CPU checks of the pushed-predicate contract: predicate_reference.pass_mask against hand-checked truth sets at the
special values and domain edges, against the oracle on ordinary columns, and the predicate the kernels evaluate
(engine.pred, then sdbg_col_pred_resolve, a host-only call of libsdbg) against pass_mask for every op and constant kind."""
import math

import numpy as np
import pytest

import count_reference as cr
import orc
import predicate_reference as pr
import serenedb_b200 as sdb

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
DENORM = 5e-324
DBL_MAX = np.finfo(np.float64).max
NAN = float("nan")
NEG_NAN = -NAN
INF = math.inf
CMP_OPS = ("LT", "LE", "GT", "GE", "EQ", "NE", "BETWEEN")

I64_PROBES = np.array([I64_MIN, I64_MIN + 1, -(1 << 62) - 1, -(1 << 62), -(1 << 53) - 1, -4, -3, -2, -1, 0, 1, 2, 3, 4,
                       (1 << 53), (1 << 53) + 1, (1 << 62), (1 << 62) + 1, I64_MAX - 1, I64_MAX], np.int64)


def _kernel_mask(values, valid, p):
    """What the kernels compute for pred() `p`: its resolved form (sdbg_col_pred_resolve) compared as cmp_i64 / cmp_f64
    do, i.e. integer against integer or double against double, which pass_mask states exactly."""
    r = sdb.resolve_pred(p, values.dtype)
    op = pr.OPS[r.op]
    if values.dtype == np.float64:
        assert r.is_float == 1
        return pr.pass_mask(values, valid, op, r.lo_f, r.hi_f)
    assert r.is_float == 0
    return pr.pass_mask(values, valid, op, r.lo_i, r.hi_i)


def _rows(values, mask):
    return [int(v) for v in np.asarray(values)[mask]]


# Float (and out-of-range) constants on an integer column: (op, lo, hi, the rows of I64_PROBES that pass).
BUG_TABLE = [
    ("BETWEEN", 0.5, INF, lambda v: v >= 1),
    ("BETWEEN", -INF, 3.5, lambda v: v <= 3),
    ("LT", 1e300, 0, lambda v: True),
    ("LT", INF, 0, lambda v: True),
    ("LE", 9.3e18, 0, lambda v: True),
    ("GT", -INF, 0, lambda v: True),
    ("GE", -1e19, 0, lambda v: True),
    ("EQ", 1e30, 0, lambda v: False),
    ("LT", NAN, 0, lambda v: False),
    ("NE", NAN, 0, lambda v: True),
    ("LT", np.float32(2.5), 0, lambda v: v <= 2),
    ("LT", 2 ** 63, 0, lambda v: True),
]


@pytest.mark.parametrize("op,lo,hi,truth", BUG_TABLE, ids=[f"{o}-{lo!r}-{hi!r}" for o, lo, hi, _ in BUG_TABLE])
def test_float_and_wide_constants_on_integer_columns(op, lo, hi, truth):
    """Each case selects exactly its truth set, in the reference and in the predicate the kernels evaluate; on int32 too,
    and NULL rows never pass."""
    exp = np.array([truth(int(v)) for v in I64_PROBES])
    p = sdb.pred(0, op, lo, hi)
    assert np.array_equal(pr.pass_mask(I64_PROBES, None, op, lo, hi), exp)
    assert np.array_equal(_kernel_mask(I64_PROBES, None, p), exp)
    i32 = np.array([I32_MIN, I32_MIN + 1, -4, -1, 0, 1, 2, 3, 4, I32_MAX - 1, I32_MAX], np.int32)
    assert np.array_equal(_kernel_mask(i32, None, p), np.array([truth(int(v)) for v in i32]))
    valid = np.arange(len(I64_PROBES)) % 3 != 0
    assert np.array_equal(_kernel_mask(I64_PROBES, valid, p), exp & valid)


def test_integer_edges_by_hand():
    v = I64_PROBES
    assert _rows(v, pr.pass_mask(v, None, "LT", I64_MIN)) == []
    assert _rows(v, pr.pass_mask(v, None, "LE", I64_MIN)) == [I64_MIN]
    assert _rows(v, pr.pass_mask(v, None, "GT", I64_MAX)) == []
    assert _rows(v, pr.pass_mask(v, None, "GE", I64_MAX)) == [I64_MAX]
    assert _rows(v, pr.pass_mask(v, None, "NE", I64_MAX)) == [int(x) for x in v[:-1]]
    assert _rows(v, pr.pass_mask(v, None, "GT", float(-2 ** 63))) == [int(x) for x in v[1:]]   # -2^63 is INT64_MIN exactly
    assert _rows(v, pr.pass_mask(v, None, "GE", float(-2 ** 63))) == [int(x) for x in v]
    assert _rows(v, pr.pass_mask(v, None, "LE", float(I64_MAX))) == [int(x) for x in v]     # float(INT64_MAX) is 2^63
    assert _rows(v, pr.pass_mask(v, None, "LT", float(2 ** 63))) == [int(x) for x in v]
    assert _rows(v, pr.pass_mask(v, None, "EQ", (1 << 53) + 1)) == [(1 << 53) + 1]            # an int constant: exact
    assert _rows(v, pr.pass_mask(v, None, "EQ", float((1 << 53) + 1))) == [1 << 53]           # the float rounds first
    assert _rows(v, pr.pass_mask(v, None, "EQ", float(1 << 62))) == [1 << 62]
    assert _rows(v, pr.pass_mask(v, None, "BETWEEN", -2.5, 2.5)) == [-2, -1, 0, 1, 2]
    assert _rows(v, pr.pass_mask(v, None, "BETWEEN", 2, 1)) == []
    assert _rows(v, pr.pass_mask(v, None, "BETWEEN", 3, 3)) == [3]
    assert _rows(v, pr.pass_mask(v, None, "BETWEEN", NAN, INF)) == []
    assert _rows(v, pr.pass_mask(v, None, "EQ", 2.5)) == []
    assert _rows(v, pr.pass_mask(v, None, "NE", 2.5)) == [int(x) for x in v]
    i32 = np.array([I32_MIN, I32_MIN + 1, -1, 0, 1, I32_MAX - 1, I32_MAX], np.int32)
    assert _rows(i32, pr.pass_mask(i32, None, "LT", I32_MIN)) == []
    assert _rows(i32, pr.pass_mask(i32, None, "LE", I32_MIN - 1)) == []
    assert _rows(i32, pr.pass_mask(i32, None, "GE", I32_MAX + 1)) == []
    assert _rows(i32, pr.pass_mask(i32, None, "GT", I32_MAX - 1)) == [I32_MAX]
    assert _rows(i32, pr.pass_mask(i32, None, "LT", -0.5)) == [I32_MIN, I32_MIN + 1, -1]
    assert _rows(i32, pr.pass_mask(i32, None, "GE", -0.0)) == [0, 1, I32_MAX - 1, I32_MAX]
    assert _rows(i32, pr.pass_mask(i32, None, "NE", I32_MAX + 1)) == [int(x) for x in i32]


def test_double_edges_by_hand():
    one_up, one_down = np.nextafter(1.0, INF), np.nextafter(1.0, -INF)
    v = np.array([NAN, NEG_NAN, INF, -INF, -0.0, 0.0, DENORM, -DENORM, 1.0, one_up, one_down, DBL_MAX, -DBL_MAX,
                  float(1 << 53), float((1 << 53) + 2)])
    assert math.copysign(1.0, v[1]) < 0 and math.copysign(1.0, v[4]) < 0   # NaN with the sign bit, and -0.0

    def idx(op, lo=0, hi=0, valid=None):
        return np.nonzero(pr.pass_mask(v, valid, op, lo, hi))[0].tolist()

    non_nan = list(range(2, len(v)))
    assert idx("EQ", 0.0) == [4, 5] and idx("EQ", -0.0) == [4, 5]
    assert idx("LT", 0.0) == [3, 7, 12] and idx("LT", -0.0) == [3, 7, 12]
    assert idx("LE", -0.0) == [3, 4, 5, 7, 12]
    assert idx("GT", 0.0) == [2, 6, 8, 9, 10, 11, 13, 14]
    assert idx("GT", DENORM) == [2, 8, 9, 10, 11, 13, 14]
    assert idx("LT", -DENORM) == [3, 12]
    for op in ("LT", "LE", "GT", "GE", "EQ"):
        assert idx(op, NAN) == [] and idx(op, NEG_NAN) == []
    assert idx("NE", NAN) == list(range(len(v))) and idx("NE", NEG_NAN) == list(range(len(v)))
    assert idx("NE", 0.0) == [0, 1, 2, 3] + list(range(6, len(v)))
    assert idx("EQ", 1.0) == [8] and idx("GT", 1.0) == [2, 9, 11, 13, 14] and idx("LT", one_up) == [3, 4, 5, 6, 7, 8, 10, 12]
    assert idx("GE", DBL_MAX) == [2, 11] and idx("GT", DBL_MAX) == [2] and idx("LE", -DBL_MAX) == [3, 12]
    assert idx("LT", INF) == [i for i in non_nan if i != 2] and idx("LE", INF) == non_nan and idx("GT", INF) == []
    assert idx("BETWEEN", 1.0, 1.0) == [8] and idx("BETWEEN", one_up, 1.0) == []
    assert idx("BETWEEN", -INF, INF) == non_nan and idx("BETWEEN", NAN, INF) == [] and idx("BETWEEN", -INF, NAN) == []
    assert idx("BETWEEN", 0.0, -0.0) == [4, 5]
    assert idx("EQ", (1 << 53) + 1) == [13]               # an int constant is rounded to the double 2^53 first
    assert idx("GE", 10 ** 400) == [2]                     # beyond the double range: +inf
    valid = np.arange(len(v)) % 2 == 0
    assert idx("NE", NAN, valid=valid) == list(range(0, len(v), 2))
    assert idx("IS_NULL", valid=valid) == list(range(1, len(v), 2))
    assert idx("IS_NOT_NULL", valid=valid) == list(range(0, len(v), 2))


def test_pass_mask_all_is_the_conjunction():
    cols = {1: (I64_PROBES, None), 2: (np.arange(len(I64_PROBES), dtype=np.float64), np.arange(len(I64_PROBES)) % 4 != 1)}
    got = pr.pass_mask_all(cols, [(1, "GE", -2.5), (2, "LT", 15.0), (1, "NE", NAN)])
    exp = (I64_PROBES >= -2) & (np.arange(len(I64_PROBES)) < 15) & cols[2][1]
    assert np.array_equal(got, exp)
    assert pr.pass_mask_all(cols, []).all()
    assert not pr.pass_mask_all(cols, [(1, "LT", -INF)]).any()


def test_reference_agrees_with_oracle_on_ordinary_columns():
    rng = np.random.default_rng(3)
    rows = 5000
    cols = {1: rng.integers(0, 1000, rows).astype(np.int64), 2: rng.random(rows) * 1000.0,
            3: rng.integers(-500, 500, rows).astype(np.int32)}
    valid = {1: rng.random(rows) < 0.8, 2: None, 3: None}
    oseg = orc.Segment(rows, has_wand=False)
    for f, vals in cols.items():
        oseg.add_column(f, vals, None if valid[f] is None else cr.validity_words(valid[f]))
    cases = [(1, "LT", 250), (1, "GE", 999), (1, "EQ", 7), (1, "NE", 7), (1, "BETWEEN", 100, 200), (1, "IS_NULL"),
             (1, "IS_NOT_NULL"), (2, "LT", 250.5), (2, "GE", 999.0), (2, "BETWEEN", 10.0, 20.0), (2, "NE", 3.0),
             (3, "LE", -1), (3, "GT", 0), (3, "BETWEEN", -10, 10)]
    for case in cases:
        f, op, *b = case
        is_float = cols[f].dtype == np.float64
        om = orc.filter_bitmap(oseg, [orc.make_pred(f, op, *b, is_float=is_float)], rows)
        exp = pr.pass_mask(cols[f], valid[f], op, *b)
        assert np.array_equal(om, cr.validity_words(exp)), case


def _constants(b):
    """A bound in every constant kind that holds it exactly."""
    out = [float(b), np.float64(b)]
    if math.isfinite(b) and float(b) == int(b) and abs(b) < 2 ** 63:
        out += [int(b), np.int64(int(b))]
    if abs(b) <= float(np.finfo(np.float32).max) and float(np.float32(b)) == b:
        out.append(np.float32(b))
    return out


BOUNDS = [0.0, 2.0, -3.0, 2.5, -2.5, 0.5, -0.5, float(2 ** 53), float(2 ** 62), -float(2 ** 62), float(2 ** 63),
          -float(2 ** 63), float(2 ** 63 - 1024), 1e300, -1e300, INF, -INF, NAN, float(I32_MAX), float(I32_MIN),
          I32_MAX + 0.5, I32_MIN - 0.5]


@pytest.mark.parametrize("op", CMP_OPS)
def test_engine_pred_resolves_exactly_around_each_bound(op):
    """engine.pred + sdbg_col_pred_resolve against pass_mask, for every constant kind (float, int, np.float32,
    np.float64, np.int64), on probes at bound - 1, bound, bound + 1 and the int64 extremes (int64, int32), and on the
    double neighbours of the bound (float64). BETWEEN pairs each bound with itself and with +-inf."""
    for b in BOUNDS:
        probes = {I64_MIN, I64_MIN + 1, I64_MAX - 1, I64_MAX, 0}
        if math.isfinite(b):
            for c in (math.floor(b), math.ceil(b)):
                probes |= {c - 1, c, c + 1}
        probes = np.array(sorted(x for x in probes if I64_MIN <= x <= I64_MAX), np.int64)
        i32 = probes[(probes >= I32_MIN) & (probes <= I32_MAX)].astype(np.int32)
        f64 = np.array([b, np.nextafter(b, INF), np.nextafter(b, -INF), 0.0, -0.0, INF, -INF, NAN, DBL_MAX, -DBL_MAX])
        his = [b, INF, -INF, 0.0] if op == "BETWEEN" else [0]
        for c in _constants(b):
            for hi in his:
                p = sdb.pred(0, op, c, hi)
                for vals in (probes, i32, f64):
                    exp = pr.pass_mask(vals, None, op, c, hi)
                    assert np.array_equal(_kernel_mask(vals, None, p), exp), (op, repr(c), hi, vals.dtype)


def test_engine_pred_constant_kinds():
    assert sdb.pred(0, "LT", np.int64(5)).is_float == 0 and sdb.pred(0, "LT", np.float32(2.5)).is_float == 1
    assert sdb.pred(0, "LT", np.float64(2.0)).is_float == 1 and sdb.pred(0, "LT", 2).is_float == 0
    # an int outside int64 is never wrapped: it goes as the nearest double, exact on both column types
    f64 = np.array([0.0, DBL_MAX, -DBL_MAX, INF, -INF, NAN, -2.0 ** 63, 2.0 ** 63, -2.0 ** 63 - 2048, 2.0 ** 64])
    for c in (2 ** 63, 2 ** 63 + 1, -2 ** 63 - 2048, -2 ** 63 - 3000, 2 ** 64 + 5, -2 ** 64, 10 ** 400, -10 ** 400):
        for op in CMP_OPS:
            p = sdb.pred(0, op, c, c)
            assert p.is_float == 1 and p.lo_f == pr.as_double(c)
            for vals in (I64_PROBES, f64):
                assert np.array_equal(_kernel_mask(vals, None, p), pr.pass_mask(vals, None, op, c, c)), (op, c, vals.dtype)
    # ... except within 1024 below INT64_MIN, whose nearest double is INT64_MIN itself
    for c in (-2 ** 63 - 1, -2 ** 63 - 1024):
        with pytest.raises(ValueError):
            sdb.pred(0, "LE", c)
    # BETWEEN mixing an int and a float bound: the int goes as a double, so it must be one exactly
    p = sdb.pred(0, "BETWEEN", -2, 2.5)
    assert p.is_float == 1 and (p.lo_f, p.hi_f) == (-2.0, 2.5)
    p = sdb.pred(0, "BETWEEN", I64_MIN, 2.5)
    assert p.is_float == 1 and (p.lo_f, p.hi_f) == (-2.0 ** 63, 2.5)
    assert np.array_equal(_kernel_mask(I64_PROBES, None, p), pr.pass_mask(I64_PROBES, None, "BETWEEN", I64_MIN, 2.5))
    with pytest.raises(ValueError):
        sdb.pred(0, "BETWEEN", (1 << 53) + 1, INF)
    with pytest.raises(TypeError):
        sdb.pred(0, "LT", "3")


def test_resolve_rejects_bad_ops_and_types():
    from serenedb_b200 import _native
    p = sdb.pred(0, "LT", 1.5)
    p.op = 9
    with pytest.raises(_native.SdbgError, match="EINVAL"):
        sdb.resolve_pred(p, np.int64)
    with pytest.raises(_native.SdbgError, match="EINVAL"):
        _native.check(_native.lib().sdbg_col_pred_resolve(sdb.pred(0, "LT", 1.5), 3, _native.ColPred()))
    # IS_NULL / IS_NOT_NULL pass through untouched whatever the constants
    r = sdb.resolve_pred(sdb.pred(0, "IS_NULL", NAN), np.int64)
    assert pr.OPS[r.op] == "IS_NULL"
