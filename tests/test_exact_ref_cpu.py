"""tests/exact_ref.py pinned to the oracle (the reference's executor restated) before any GPU result is judged
by it: on finite data both agree within the summation bound, on every special value the error class, NaN,
infinity and the sign of zero agree exactly."""
import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import fp_edge_data as D

C, K, MUL = g.GX_OP_COL, g.GX_OP_CONST, g.GX_OP_MUL
TYPES = [g.GX_INT4, g.GX_FLOAT8, g.GX_FLOAT8]
ALL_AGGS = [(g.GX_AGG_SUM_F8, [(C, 1, 0)]), (g.GX_AGG_AVG_F8, [(C, 1, 0)]), (g.GX_AGG_MIN_F8, [(C, 1, 0)]),
            (g.GX_AGG_MAX_F8, [(C, 1, 0)]), (g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(C, 1, 0), (C, 2, 0), (MUL, 0, 0)])]


def _cols(gi, x, y):
    return [(gi * 7 - 3).astype(np.int32), x, y]


def _agree(plan, cols, types=TYPES, nulls=None):
    want = X.expect_groups(plan, cols, nulls, types)
    try:
        got = O.exec_agg(O.Rel(types, cols, nulls), plan)
    except RuntimeError as e:
        assert "status 6" in str(e), e
        assert want == "overflow", f"the oracle errors, the exact reference says {want}"
        return "overflow"
    assert want != "overflow", "the exact reference errors, the oracle does not"
    X.check(plan, want, (got.keys, got.aggs, got.nulls), [types[plan.group_cols[c].col] for c in range(plan.n_group_cols)])
    return want


@pytest.mark.parametrize("name", ["cancel", "subnormal", "special"])
def test_exact_reference_agrees_with_the_oracle(name):
    rng = np.random.default_rng(7)
    data = {"cancel": lambda: D.cancel(rng, D.CANCEL_SIZES[:-1], top=100), "subnormal": lambda: D.subnormal(rng, 6),
            "special": lambda: D.special(rng)}[name]()
    plan = O.make_plan(group_cols=[(0, 0)], aggs=ALL_AGGS, est_groups=16)
    want = _agree(plan, _cols(*data))
    assert len(want) == len(set(data[0].tolist()))
    if name == "special":
        w = {k[0]: v for k, v in want.items()}
        assert w[-3][0].value == np.inf and w[-3][1].value == np.inf           # inf input: not an overflow
        assert np.isnan(w[11][0].value)                                        # +inf + -inf
        assert np.signbit(w[25][0].value) and w[25][0].value == 0              # sum of only -0.0
        assert not np.signbit(w[32][0].value)                                  # mixed zeros: +0
        assert np.isnan(w[46][3].value) and w[46][2].value == -3.0             # max sorts NaN last, min skips it
    if name == "cancel":                                                       # sums up to 1e300 without avg()
        plan = O.make_plan(group_cols=[(0, 0)], aggs=[a for a in ALL_AGGS if a[0] != g.GX_AGG_AVG_F8], est_groups=16)
        assert _agree(plan, _cols(*D.cancel(rng, D.CANCEL_SIZES[:-1]))) != "overflow"


@pytest.mark.parametrize("case", ["sum_finite", "max_xx", "sum_xx", "avg_sxx", "mul_underflow", "sum_int8", "avg_inf"])
def test_error_classes_agree_with_the_oracle(case):
    x = {"sum_finite": [1e308, 1e308, 5.0], "max_xx": [1e200, 2.0, 3.0], "sum_xx": [1e200, 2.0, 3.0],
         "avg_sxx": [1e200, -1e200, 1e200, -1e200], "mul_underflow": [1e-200, 2.0, 3.0], "sum_int8": [1.0, 2.0, 3.0],
         "avg_inf": [1.0, np.inf, 2.0]}[case]
    n = len(x)
    cols = [np.zeros(n, np.int32), np.array(x), np.full(n, 1e-200), np.array([2**62, 2**62, 5], np.int64)[:n] if n == 3 else np.zeros(n, np.int64)]
    types = TYPES + [g.GX_INT8]
    xx = [(C, 1, 0), (C, 1, 0), (MUL, 0, 0)]
    agg = {"sum_finite": (g.GX_AGG_SUM_F8, [(C, 1, 0)]), "max_xx": (g.GX_AGG_MAX_F8, xx), "sum_xx": (g.GX_AGG_SUM_F8, xx),
           "avg_sxx": (g.GX_AGG_AVG_F8, [(C, 1, 0)]), "mul_underflow": (g.GX_AGG_SUM_F8, [(C, 1, 0), (C, 2, 0), (MUL, 0, 0)]),
           "sum_int8": (g.GX_AGG_SUM_I8, [(C, 3, 0)]), "avg_inf": (g.GX_AGG_AVG_F8, [(C, 1, 0)])}[case]
    plan = O.make_plan(group_cols=[(0, 0)], aggs=[agg], est_groups=4)
    assert (_agree(plan, cols, types) == "overflow") == (case != "avg_inf")


def test_float8_group_keys_agree_with_the_oracle():
    """+-0 fold into one group; NaN and a NaN of the other sign stay apart (hashfloat8 hashes the bits)"""
    nan, nnan = np.float64(np.nan), -np.float64(np.nan)
    assert np.signbit(nnan)
    k = np.array([0.0, -0.0, nan, nnan, nan, 1.5, -0.0, nnan])
    x = np.arange(len(k), dtype=np.float64)
    types = [g.GX_FLOAT8, g.GX_FLOAT8]
    plan = O.make_plan(group_cols=[(0, 0)], aggs=[(g.GX_AGG_SUM_F8, [(C, 1, 0)]), (g.GX_AGG_COUNT_STAR, [])], est_groups=8)
    want = _agree(plan, [k, x], types)
    assert len(want) == 4
