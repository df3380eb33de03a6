"""Exact reference for scan quals (`col op const`, ANDed), CPU only, with PostgreSQL's semantics:

  - float8 compares as float8_cmp_internal (float.c), never by subtraction: NaN equals NaN (either sign) and sorts
    above +inf, +-inf equal themselves, -0 = +0;
  - "char" compares as uint8 (charlt etc., char.c), the constant taken mod 256;
  - int4 / date values are widened and compared with the int64 constant by value (int48lt etc.), so x = 2^32 + 5
    never holds for an int4 x;
  - a NULL fails every qual (a strict operator returns NULL, which ExecQual treats as false).

Pinned to the oracle's ExecQual restatement by tests/test_qual_ref_cpu.py.  The value sets below are shared with the
GPU tests (tests/test_gpu_quals_exprs.py): each type's edge values and their neighbours, used both as column values
and as constants."""
import numpy as np

import opentenbase_b200 as g

I32, I64 = np.iinfo(np.int32), np.iinfo(np.int64)
DBL_MAX, DBL_TRUE_MIN = np.finfo(np.float64).max, np.float64(5e-324)
NAN = np.float64(np.nan)
NEG_NAN = np.copysign(NAN, -1.0)
OPS = [g.GX_LT, g.GX_LE, g.GX_EQ, g.GX_GE, g.GX_GT, g.GX_NE]
TYPES = [g.GX_INT4, g.GX_INT8, g.GX_DATE, g.GX_CHAR, g.GX_FLOAT8]

EDGES = {
    g.GX_INT4: [I32.min, I32.min + 1, -2, -1, 0, 1, 5, I32.max - 1, I32.max],
    g.GX_INT8: [I64.min, I64.min + 1, -2**32 - 1, -2**32, -2**32 + 1, -2**31 - 1, -2**31, -2**31 + 1, -1, 0, 1, 5,
                2**31 - 1, 2**31, 2**31 + 1, 2**32 - 1, 2**32, 2**32 + 1, 2**32 + 5, I64.max - 1, I64.max],
    g.GX_DATE: [I32.min, I32.min + 1, -2_451_545, -36_525, -2, -1, 0, 1, 5, 2_147_483_646, I32.max],
    g.GX_CHAR: [0, 1, 126, 127, 128, 129, 199, 200, 201, 254, 255],
    g.GX_FLOAT8: [NAN, NEG_NAN, -np.inf, np.inf, -0.0, 0.0, DBL_TRUE_MIN, -DBL_TRUE_MIN, 2 * DBL_TRUE_MIN, -2 * DBL_TRUE_MIN,
                  DBL_MAX, -DBL_MAX, np.nextafter(DBL_MAX, 0), -np.nextafter(DBL_MAX, 0), 1.0, -1.0],
}
# constants outside int32 against int4 / date columns: a kernel that narrows the constant to 32 bits would take
# x = 2^32 + 5 for x = 5, and x < 2^31 for x < INT32_MIN
WIDE_CONSTS = [2**31, -2**31 - 1, 2**32, 2**32 + 5, -2**32 + 5, I64.min, I64.max]


def consts(t):
    """the constants a qual on a column of type t is tested with"""
    return EDGES[t] + (WIDE_CONSTS if t in (g.GX_INT4, g.GX_DATE) else [])


def column(rng, t, n, null_frac=0.0):
    """n values of type t: every edge value (in random order, repeated), with NULLs where null_frac asks
    (None: no NULL array).  Returns (values in the library's numpy dtype, uint8 NULL flags or None)."""
    e = EDGES[t]
    idx = np.concatenate([np.arange(len(e)), rng.integers(0, len(e), max(n - len(e), 0))])[:n]
    idx = rng.permutation(idx)
    if t == g.GX_FLOAT8:
        v = np.array(e, np.float64)[idx]
    elif t == g.GX_CHAR:
        v = np.array(e, np.uint8)[idx].view(np.int8)
    else:
        v = np.array(e, np.int64)[idx].astype(g.NP_DTYPES[t])
    nl = (rng.random(n) < null_frac).astype(np.uint8) if null_frac else None
    return v, nl


def _type_of(v):
    if v.dtype.kind == "f":
        return g.GX_FLOAT8
    return g.GX_CHAR if v.dtype.itemsize == 1 else g.GX_INT8


def cmp(v, k, t):
    """-1 / 0 / +1 per value: v compared with the constant k under type t's comparison"""
    if t == g.GX_FLOAT8:
        x, k = np.asarray(v, np.float64), float(k)
        xn = np.isnan(x)
        with np.errstate(invalid="ignore"):
            ord_ = np.where(x > k, 1, np.where(x < k, -1, 0))
        if np.isnan(k):
            return np.where(xn, 0, -1)
        return np.where(xn, 1, ord_)
    if t == g.GX_CHAR:
        x, k = np.asarray(v).astype(np.int8).view(np.uint8).astype(np.int64), int(k) & 0xFF
    else:
        x, k = np.asarray(v).astype(np.int64), int(k)
    return np.where(x > k, 1, np.where(x < k, -1, 0))


HOLDS = {g.GX_LT: lambda c: c < 0, g.GX_LE: lambda c: c <= 0, g.GX_EQ: lambda c: c == 0,
         g.GX_GE: lambda c: c >= 0, g.GX_GT: lambda c: c > 0, g.GX_NE: lambda c: c != 0}


def quals(cols, nulls, preds, n, types=None):
    """rows passing every qual (col, op, const[, is_float]) of preds.  types: the columns' GX_* types; without them a
    column's type is read off its dtype (float64 float8, int8 "char", any other integer by value)."""
    keep = np.ones(n, bool)
    for p in preds:
        col, op, k = p[0], p[1], p[2]
        v = np.asarray(cols[col])
        t = types[col] if types is not None else _type_of(v)
        keep &= HOLDS[op](cmp(v, k, t))
        if nulls is not None and nulls[col] is not None:
            keep &= ~np.asarray(nulls[col]).astype(bool)
    return keep
