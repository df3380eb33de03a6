"""tests/distinct_ref.py against a row-by-row count of Python sets, with no GPU: NULL arguments skipped, all-NULL groups
counting 0, NULL group keys, INT64_MIN / INT32_MIN as ordinary values, repeated rows (a join's fan-out), no GROUP BY
and no rows."""
import numpy as np
import pytest

import opentenbase_b200 as g
import distinct_ref as D

I64, I32 = np.iinfo(np.int64), np.iinfo(np.int32)
TYPES = [g.GX_INT4, g.GX_INT8, g.GX_INT4, g.GX_DATE, g.GX_CHAR, g.GX_FLOAT8]


def data(rng, n):
    grp = rng.integers(0, 6, n).astype(np.int32)
    a8 = rng.choice(np.array([I64.min, I64.max, 0, -1, 5, 2**40], np.int64), n)
    a4 = rng.choice(np.array([I32.min, I32.max, 0, 7], np.int64), n).astype(np.int32)
    ad = rng.integers(-3, 3, n).astype(np.int32)
    ac = rng.integers(-128, 128, n).astype(np.int8)
    x = rng.standard_normal(n)
    nl = lambda f: (rng.random(n) < f).astype(np.uint8)
    nulls = [nl(0.1), nl(0.2), nl(0.2), nl(0.2), nl(0.2), None]
    for c in (1, 2, 3, 4):
        nulls[c][grp == 5] = 1                                  # group 5: every argument NULL
    return [grp, a8, a4, ad, ac, x], nulls


def brute(o, cols, nulls, gcol, arg):
    seen = {}
    for r in o.tolist():
        k = () if gcol is None else ((None if nulls[gcol][r] else int(cols[gcol][r])),)
        s = seen.setdefault(k, set())
        if not nulls[arg][r]:
            s.add(int(cols[arg][r]))
    return {k: len(v) for k, v in seen.items()}


@pytest.mark.parametrize("arg", [1, 2, 3, 4])
@pytest.mark.parametrize("grouped", [True, False])
def test_distinct_counts_match_python_sets(arg, grouped):
    rng = np.random.default_rng(arg)
    cols, nulls = data(rng, 3000)
    o = np.concatenate([np.arange(3000), rng.integers(0, 3000, 1000)])        # some rows twice, as a join repeats them
    plan = g.make_plan(group_cols=[(0, 0)] if grouped else [],
                       aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_COUNT_DISTINCT, [(g.GX_OP_COL, arg, 0)]),
                             (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 5, 0)])])
    want = D.expect_groups(plan, cols, TYPES, o, nulls)
    bf = brute(o, cols, nulls, 0 if grouped else None, arg)
    assert set(want) == set(bf)
    for k, n in bf.items():
        assert want[k][1].value == n
    if grouped:
        assert want[(5,)][1].value == 0 and want[(None,)][0].value > 0


def test_no_rows():
    rng = np.random.default_rng(0)
    cols, nulls = data(rng, 10)
    plan = g.make_plan(aggs=[(g.GX_AGG_COUNT_DISTINCT, [(g.GX_OP_COL, 1, 0)]), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 5, 0)])])
    want = D.expect_groups(plan, cols, TYPES, np.zeros(0, np.int64), nulls)
    assert list(want) == [()] and want[()][0].value == 0 and want[()][1].kind == "null"
    grouped = g.make_plan(group_cols=[(0, 0)], aggs=[(g.GX_AGG_COUNT_DISTINCT, [(g.GX_OP_COL, 1, 0)])])
    assert D.expect_groups(grouped, cols, TYPES, np.zeros(0, np.int64), nulls) == {}
