"""The provider's SQL:2003 binary aggregates over (float8, float8): what gpuexec_match_plan takes and declines, the
scan tuple of a two-phase plan, plan shipping, the host logic against the ABI double, and one Begin/Exec/End run on the
GPU.

Taken: regr_count (2818) .. corr (2829) over two float8 expressions of the outer relation, Y's program, GX_OP_ARG2 and
X's program in one descriptor argument.  Declined: DISTINCT, FILTER, ORDER BY, a program longer than GX_MAX_EXPR_OPS,
and a second (Y, X) pair (two regression states do not fit the library's state words)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import regr_ref as R
from test_provider_harness import HARNESS, write_case
from test_provider_planner_cpu import LINEITEM, parse_desc, plan
from test_provider_host_logic_cpu import DOUBLE, LTYPES, canned, run as run_double
from test_provider_ship_cpu import ship

needs_harness = pytest.mark.skipif(not os.path.exists(HARNESS), reason="harness binary not built (needs /root/reference at build time)")
needs_double = pytest.mark.skipif(not os.path.exists(DOUBLE), reason="harness binary not built (needs /root/reference at build time)")
FLOAT8OID, INT8OID, F8ARRAY = 701, 20, 1022
NAMES = ["regr_count", "regr_sxx", "regr_syy", "regr_sxy", "regr_avgx", "regr_avgy", "regr_r2", "regr_slope", "regr_intercept",
         "covar_pop", "covar_samp", "corr"]
TAKEN = [(n, 2818 + i, g.GX_AGG_REGR_COUNT + i) for i, n in enumerate(NAMES)]


def by_shipdate(*targets, dist="dist none"):
    return plan(LINEITEM, "scan 1", "group 1.6", "target var 1.6", *targets, dist, "groups 2526")


def col_of(d, attno):
    return [c for c, (a, t) in enumerate(d["outer"]["cols"]) if a == attno and t == g.GX_FLOAT8][0]


@needs_harness
@pytest.mark.parametrize("name, oid, fn", TAKEN)
def test_each_aggregate_is_taken(name, oid, fn):
    """SELECT l_shipdate, <agg>(l_extendedprice, l_discount) FROM lineitem GROUP BY l_shipdate"""
    r = by_shipdate(f"target agg {name} v1.3 , v1.4")
    assert r is not None and r["path"] == "path pushdown: CustomScan"
    d = parse_desc(r["desc"])
    y, x = col_of(d, 2), col_of(d, 3)
    assert d["aggs"] == [(fn, [(g.GX_OP_COL, y, 0), (g.GX_OP_ARG2, 0, 0), (g.GX_OP_COL, x, 0)])]


@needs_harness
def test_expression_argument_and_twins_are_taken():
    """corr(l_extendedprice * (1 - l_discount), l_quantity) next to regr_slope and regr_intercept of the same pair: 7 ops,
    one state"""
    pair = "v1.3 k1 v1.4 - * , v1.2"
    r = by_shipdate(f"target agg corr {pair}", f"target agg regr_slope {pair}", f"target agg regr_intercept {pair}",
                    "target agg sum_f8 v1.3")
    assert r is not None
    d = parse_desc(r["desc"])
    assert [a[0] for a in d["aggs"]] == [g.GX_AGG_CORR_F8, g.GX_AGG_REGR_SLOPE_F8, g.GX_AGG_REGR_INTERCEPT_F8, g.GX_AGG_SUM_F8]
    assert len(d["aggs"][0][1]) == 7 and d["aggs"][0][1] == d["aggs"][1][1] == d["aggs"][2][1]


@needs_harness
@pytest.mark.parametrize("targets, why", [
    (["target agg corr v1.3 , v1.4 distinct"], "DISTINCT"),
    (["target agg corr v1.3 , v1.4 filter"], "FILTER"),
    (["target agg regr_slope v1.3 , v1.4 order"], "ORDER BY inside the call"),
    (["target agg corr v1.3 k1 + k2 * k3 + k4 * , v1.4 k1 + k2 * k3 +"], "13 ops: longer than GX_MAX_EXPR_OPS"),
    (["target agg corr v1.3 , v1.4", "target agg regr_slope v1.4 , v1.3"], "a second (Y, X) pair"),
])
def test_declines(targets, why):
    assert by_shipdate(*targets) is None, why


@needs_harness
def test_two_phase_scan_types():
    """float8[6] for float8_regr_combine, int8 for regr_count's int8pl"""
    r = by_shipdate("target agg corr v1.3 , v1.4", "target agg regr_count v1.3 , v1.4", dist="dist shard 1.1 nodes 4")
    assert r["path"].startswith("path partial: Finalize Agg") and parse_desc(r["desc"])["partial"] == 1
    assert r["scan"][1:] == [("agg", "2829", "type", str(F8ARRAY), "split", "6"), ("agg", "2818", "type", str(INT8OID), "split", "6")]


PAIR = [(g.GX_OP_COL, 0, 0), (g.GX_OP_ARG2, 0, 0), (g.GX_OP_COL, 1, 0)]     # (l_extendedprice, l_discount)


def lineitem_case(d, partial, fns, n=400):
    l = O.gen_lineitem(1, 0, n)
    lrel = O.Rel(LTYPES, l)
    p = g.make_plan(group_cols=[(0, 2)], aggs=[(fn, PAIR) for fn in fns], est_groups=2526)
    case = os.path.join(d, "r.case")
    types = [INT8OID if fn == g.GX_AGG_REGR_COUNT else (F8ARRAY if partial else FLOAT8OID) for fn in fns]
    write_case(case, [(LTYPES, lrel)], {"rti": 1, "attnums": [2, 3, 5]}, None, p, partial, [1082] + types)
    return case, l, p


@needs_harness
def test_descriptor_survives_plan_shipping():
    with tempfile.TemporaryDirectory() as d:
        case, _, _ = lineitem_case(d, True, [g.GX_AGG_CORR_F8, g.GX_AGG_REGR_COUNT, g.GX_AGG_REGR_SLOPE_F8])
        assert ship(case)


@needs_double
def test_host_logic_partial_states_carry_the_six_values():
    """two-phase: {N, Sx, Sxx, Sy, Syy, Sxy} from gx_result_fetch_regr; regr_count is the int8 count"""
    fns = [g.GX_AGG_CORR_F8, g.GX_AGG_REGR_COUNT]
    keys = np.array([[17], [-3]], np.int64)
    vals = np.array([[10.5, 0.0], [0.0, 0.0]])
    cnts = np.array([[4, 4], [0, 0]], np.int64)
    regr = np.zeros((2, 2, 6))
    regr[0, 0] = [4, 10.5, 2.25, 0.5, 1.0, -0.75]
    with tempfile.TemporaryDirectory() as d:
        case, _, _ = lineitem_case(d, True, fns)
        res = os.path.join(d, "r.res")
        canned(res, keys, vals, cnts, np.zeros((2, 3), np.uint8))
        with open(res, "ab") as f:
            f.write(np.zeros((2, 2)).tobytes())           # no variance: Sxx words unused
            f.write(regr.tobytes())
        rows, err = run_double(case, res)
    assert sorted(rows) == sorted([["17", "{4,10.5,2.25,0.5,1,-0.75}", "4"], ["-3", "{0,0,0,0,0,0}", "0"]]), rows
    assert "result_fetch_states" in err and "result_fetch_regr" in err and "result_fetch_sxx" not in err


@needs_double
def test_host_logic_final_values_and_nulls():
    fns = [g.GX_AGG_CORR_F8, g.GX_AGG_REGR_COUNT]
    keys = np.array([[17], [-3]], np.int64)
    aggs = np.array([[-0.5, np.array([4], np.int64).view(np.float64)[0]], [0.0, 0.0]])
    nulls = np.array([[0, 0, 0], [0, 1, 0]], np.uint8)                 # corr of no pair is NULL, regr_count 0
    with tempfile.TemporaryDirectory() as d:
        case, _, _ = lineitem_case(d, False, fns)
        res = os.path.join(d, "r.res")
        canned(res, keys, aggs, np.zeros((2, 2), np.int64), nulls)
        rows, err = run_double(case, res)
    assert sorted(rows) == sorted([["17", "-0.5", "4"], ["-3", "\\N", "0"]]), rows
    assert "result_fetch (final values)" in err and "result_fetch_regr" not in err


@pytest.mark.gpu
@needs_harness
def test_harness_regression_on_the_gpu():
    """SELECT l_shipdate, corr(l_extendedprice, l_discount), regr_slope(..), regr_count(..) FROM lineitem GROUP BY
    l_shipdate through Begin/Exec/End"""
    fns = [g.GX_AGG_CORR_F8, g.GX_AGG_REGR_SLOPE_F8, g.GX_AGG_REGR_COUNT]
    with tempfile.TemporaryDirectory() as d:
        case, l, p = lineitem_case(d, False, fns, n=60000)
        r = subprocess.run([HARNESS, case], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    rows = [line.split("\t") for line in r.stdout.splitlines() if line]
    price, disc, ship_date = np.asarray(l[2]), np.asarray(l[3]), np.asarray(l[5])
    assert len(rows) == len(np.unique(ship_date))
    for row in rows:
        sel = ship_date == int(row[0])
        for a, fn in enumerate(fns):
            want = R.expect(fn, disc[sel], price[sel])
            null = row[1 + a] == "\\N"
            if fn == g.GX_AGG_REGR_COUNT:
                assert not null and int(row[1 + a]) == want[1], (row, want)
            else:
                assert R.matches(want, 0.0 if null else float(row[1 + a]), null), (row, want)
