"""tests/qual_ref.py pinned to the oracle's ExecQual restatement, without a GPU.

The oracle evaluates the quals of a sequential scan tuple by tuple (orc_exec.c: float8_cmp, cmp_char, cmp_int on the
widened value).  A unique row-id column grouped with count(*) under the quals shows which rows it keeps: the groups
present are exactly the rows that passed.  Every type, every operator, every edge value of the shared value sets as a
constant, NULLs in the column, and four ANDed quals over mixed types."""
import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import join_ref as J
import qual_ref as Q

CNT = (g.GX_AGG_COUNT_STAR, [])


def oracle_kept(types, cols, nulls, preds):
    """row ids (column 0) of the rows the oracle's scan keeps under preds"""
    plan = O.make_plan(preds=preds, group_cols=[(0, 0)], aggs=[CNT], est_groups=len(cols[0]))
    r = O.exec_agg(O.Rel(types, cols, nulls), plan)
    assert (r.aggs[:, 0].view(np.int64) == 1).all()
    return np.sort(r.keys[:, 0])


def pred(col, op, k, t):
    return (col, op, k, True) if t == g.GX_FLOAT8 else (col, op, k)


@pytest.mark.parametrize("t", Q.TYPES)
def test_every_operator_and_constant_matches_the_oracle(t):
    rng = np.random.default_rng(t)
    n = 160
    v, nl = Q.column(rng, t, n, null_frac=0.1)
    rowid = np.arange(n, dtype=np.int64)
    types, cols, nulls = [g.GX_INT8, t], [rowid, v], [None, nl]
    for op in Q.OPS:
        for k in Q.consts(t):
            p = pred(1, op, k, t)
            want = np.flatnonzero(Q.quals(cols, nulls, [p], n, types))
            np.testing.assert_array_equal(oracle_kept(types, cols, nulls, [p]), want, err_msg=f"type {t} op {op} const {k!r}")
            # the reference infers the type from the dtype when none is given (join_ref.quals' callers)
            np.testing.assert_array_equal(np.flatnonzero(J.quals(cols, nulls, [p], n)), want)


def test_four_anded_quals_over_mixed_types():
    rng = np.random.default_rng(99)
    n = 3000
    types = [g.GX_INT8] + Q.TYPES
    cols, nulls = [np.arange(n, dtype=np.int64)], [None]
    for t in Q.TYPES:
        v, nl = Q.column(rng, t, n, null_frac=0.05)
        cols.append(v); nulls.append(nl)
    cases = [
        [(1, g.GX_GE, -1), (4, g.GX_GT, 100), (5, g.GX_LT, np.inf, True), (2, g.GX_NE, 2**32)],
        [(3, g.GX_LE, 0), (5, g.GX_GE, -0.0, True), (4, g.GX_NE, 200), (1, g.GX_LT, 2**31)],
        [(2, g.GX_GT, -2**31), (2, g.GX_LE, 2**32), (5, g.GX_EQ, np.nan, True), (4, g.GX_GE, 128)],
        [(5, g.GX_GT, -np.inf, True), (5, g.GX_LT, np.nan, True), (3, g.GX_GE, int(Q.I32.min)), (1, g.GX_LE, 2**32 + 5)],
    ]
    for preds in cases:
        want = np.flatnonzero(Q.quals(cols, nulls, preds, n, types))
        assert 0 < len(want) < n, preds
        np.testing.assert_array_equal(oracle_kept(types, cols, nulls, preds), want, err_msg=str(preds))


def test_the_cases_a_subtracting_reference_got_wrong():
    """+inf = +inf and -inf <= -inf hold (inf - inf is NaN, not 0); "char" 200 > 100 holds (uint8, not int8)"""
    f = [np.array([np.inf, -np.inf, 1.0])]
    assert Q.quals(f, None, [(0, g.GX_EQ, np.inf, True)], 3).tolist() == [True, False, False]
    assert Q.quals(f, None, [(0, g.GX_LE, -np.inf, True)], 3).tolist() == [False, True, False]
    assert J.quals(f, None, [(0, g.GX_EQ, np.inf, True)], 3).tolist() == [True, False, False]
    assert J.quals(f, None, [(0, g.GX_LE, -np.inf, True)], 3).tolist() == [False, True, False]
    c = [np.array([200, 100, 50], np.uint8).view(np.int8)]
    assert Q.quals(c, None, [(0, g.GX_GT, 100)], 3).tolist() == [True, False, False]
    assert J.quals(c, None, [(0, g.GX_GT, 100)], 3).tolist() == [True, False, False]
    # and the oracle agrees on all three
    rid = np.arange(3, dtype=np.int64)
    assert oracle_kept([g.GX_INT8, g.GX_FLOAT8], [rid, f[0]], None, [(1, g.GX_EQ, np.inf, True)]).tolist() == [0]
    assert oracle_kept([g.GX_INT8, g.GX_FLOAT8], [rid, f[0]], None, [(1, g.GX_LE, -np.inf, True)]).tolist() == [1]
    assert oracle_kept([g.GX_INT8, g.GX_CHAR], [rid, c[0]], None, [(1, g.GX_GT, 100)]).tolist() == [0]


def test_nan_minus_zero_and_wide_constants():
    """NaN of either sign equals NaN and sorts above +inf; -0 = +0; an int4 5 is not 2^32 + 5"""
    x = [np.array([np.nan, Q.NEG_NAN, np.inf, -0.0, 0.0])]
    assert Q.quals(x, None, [(0, g.GX_EQ, Q.NEG_NAN, True)], 5).tolist() == [True, True, False, False, False]
    assert Q.quals(x, None, [(0, g.GX_GT, np.inf, True)], 5).tolist() == [True, True, False, False, False]
    assert Q.quals(x, None, [(0, g.GX_EQ, 0.0, True)], 5).tolist() == [False, False, False, True, True]
    i = [np.array([5, -1, Q.I32.min], np.int32)]
    assert Q.quals(i, None, [(0, g.GX_EQ, 2**32 + 5)], 3, [g.GX_INT4]).tolist() == [False, False, False]
    assert Q.quals(i, None, [(0, g.GX_LT, 2**31)], 3, [g.GX_INT4]).tolist() == [True, True, True]
    assert Q.quals(i, None, [(0, g.GX_GT, Q.I64.min)], 3, [g.GX_INT4]).tolist() == [True, True, True]
    assert Q.quals(i, [np.array([1, 0, 0], np.uint8)], [(0, g.GX_NE, 7)], 3).tolist() == [False, True, True]
