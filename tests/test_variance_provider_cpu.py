"""The provider's variance and standard deviation aggregates over float8: what gpuexec_match_plan takes and declines, the
scan tuple of a two-phase plan, plan shipping, the host logic against the ABI double, and one Begin/Exec/End run on the
GPU.

Taken: var_pop (2722), var_samp (2645), variance (2152), stddev_pop (2728), stddev_samp (2716) and stddev (2158) over a
float8 expression of the outer relation.  Declined: the float4 overloads (no float4 column on the device), the integer
and numeric ones (they return numeric), and any plan whose state words would exceed the library's limit."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import var_ref as V
from test_provider_harness import HARNESS, write_case
from test_provider_planner_cpu import LINEITEM, parse_desc, plan
from test_provider_host_logic_cpu import DOUBLE, LTYPES, canned, run as run_double
from test_provider_ship_cpu import ship

needs_harness = pytest.mark.skipif(not os.path.exists(HARNESS), reason="harness binary not built (needs /root/reference at build time)")
needs_double = pytest.mark.skipif(not os.path.exists(DOUBLE), reason="harness binary not built (needs /root/reference at build time)")
FLOAT8OID, F8ARRAY = 701, 1022
TAKEN = [("var_pop_f8", 2722, g.GX_AGG_VAR_POP_F8), ("var_samp_f8", 2645, g.GX_AGG_VAR_SAMP_F8),
         ("variance_f8", 2152, g.GX_AGG_VAR_SAMP_F8), ("stddev_pop_f8", 2728, g.GX_AGG_STDDEV_POP_F8),
         ("stddev_samp_f8", 2716, g.GX_AGG_STDDEV_SAMP_F8), ("stddev_f8", 2158, g.GX_AGG_STDDEV_SAMP_F8)]


def by_shipdate(*targets, dist="dist none"):
    return plan(LINEITEM, "scan 1", "group 1.6", "target var 1.6", *targets, dist, "groups 2526")


def price_col(d):
    return [c for c, (a, t) in enumerate(d["outer"]["cols"]) if a == 2 and t == g.GX_FLOAT8][0]


@needs_harness
@pytest.mark.parametrize("name, oid, fn", TAKEN + [("min_f8", 2136, g.GX_AGG_MIN_F8), ("max_f8", 2120, g.GX_AGG_MAX_F8)])
def test_each_aggregate_is_taken(name, oid, fn):
    """SELECT l_shipdate, avg(l_extendedprice), <agg>(l_extendedprice) FROM lineitem GROUP BY l_shipdate"""
    r = by_shipdate("target agg avg_f8 v1.3", f"target agg {name} v1.3")
    assert r is not None and r["path"] == "path pushdown: CustomScan"
    d = parse_desc(r["desc"])
    col = price_col(d)
    assert d["aggs"] == [(g.GX_AGG_AVG_F8, [(g.GX_OP_COL, col, 0)]), (fn, [(g.GX_OP_COL, col, 0)])]


@needs_harness
def test_expression_argument_is_taken():
    r = by_shipdate("target agg stddev_f8 v1.3 k1 v1.4 - *")
    assert r is not None and parse_desc(r["desc"])["aggs"][0][0] == g.GX_AGG_STDDEV_SAMP_F8


@needs_harness
@pytest.mark.parametrize("target, why", [
    ("target agg stddev_f4 v1.3", "stddev(float4): no float4 column on the device"),
    ("target agg stddev_i8 v1.1", "stddev(int8) returns numeric"),
    ("target agg stddev_f8 v1.3 distinct", "DISTINCT"),
])
def test_declines(target, why):
    assert by_shipdate(target) is None, why


@needs_harness
def test_state_words_over_the_library_limit_decline_at_plan_time():
    """four variances of four nullable arguments need 1 + 4 x 5 words, more than the library's 18; three fit, and so do
    four sums (two words each at most: eight aggregates without a variance or regression always fit)"""
    args = ["v1.3", "v1.3 k1 +", "v1.3 k2 *", "v1.3 v1.4 +"]
    assert by_shipdate(*[f"target agg var_pop_f8 {a}" for a in args]) is None
    assert by_shipdate(*[f"target agg var_pop_f8 {a}" for a in args[:3]]) is not None
    assert by_shipdate(*[f"target agg sum_f8 {a}" for a in args]) is not None
    # variances of one argument share their words: six of them are one state
    assert by_shipdate(*[f"target agg {n} v1.3" for n, _, _ in TAKEN]) is not None


@needs_harness
def test_two_phase_scan_types_are_float8_arrays():
    r = by_shipdate("target agg stddev_f8 v1.3", "target agg var_pop_f8 v1.3", "target agg avg_f8 v1.3", dist="dist shard 1.1 nodes 4")
    assert r["path"].startswith("path partial: Finalize Agg") and parse_desc(r["desc"])["partial"] == 1
    assert r["scan"][1:] == [("agg", "2158", "type", str(F8ARRAY), "split", "6"), ("agg", "2722", "type", str(F8ARRAY), "split", "6"),
                             ("agg", "2105", "type", str(F8ARRAY), "split", "6")]


def lineitem_case(d, partial, fns, n=400):
    l = O.gen_lineitem(1, 0, n)
    lrel = O.Rel(LTYPES, l)
    p = g.make_plan(group_cols=[(0, 2)], aggs=[(fn, [(g.GX_OP_COL, 0, 0)]) for fn in fns], est_groups=2526)
    case = os.path.join(d, "v.case")
    write_case(case, [(LTYPES, lrel)], {"rti": 1, "attnums": [2, 3, 5]}, None, p, partial,
               [1082] + [F8ARRAY if partial else FLOAT8OID] * len(fns))
    return case, l, p


@needs_harness
def test_descriptor_survives_plan_shipping():
    with tempfile.TemporaryDirectory() as d:
        case, _, _ = lineitem_case(d, True, [g.GX_AGG_STDDEV_SAMP_F8, g.GX_AGG_VAR_POP_F8, g.GX_AGG_AVG_F8])
        assert ship(case)


@needs_double
def test_host_logic_partial_states_carry_sxx():
    """two-phase: {N, Sx, Sxx} with Sxx from gx_result_fetch_sxx; avg's Sxx stays 0"""
    fns = [g.GX_AGG_STDDEV_SAMP_F8, g.GX_AGG_AVG_F8, g.GX_AGG_VAR_POP_F8]
    keys = np.array([[17], [-3]], np.int64)
    vals = np.array([[10.5, 10.5, 10.5], [0.0, 0.0, 0.0]])
    cnts = np.array([[4, 4, 4], [0, 0, 0]], np.int64)
    sxx = np.array([[2.25, 0.0, 2.25], [0.0, 0.0, 0.0]])
    with tempfile.TemporaryDirectory() as d:
        case, _, _ = lineitem_case(d, True, fns)
        res = os.path.join(d, "v.res")
        canned(res, keys, vals, cnts, np.zeros((2, 4), np.uint8))
        with open(res, "ab") as f:
            f.write(sxx.tobytes())
        rows, err = run_double(case, res)
    assert sorted(rows) == sorted([["17", "{4,10.5,2.25}", "{4,10.5,0}", "{4,10.5,2.25}"], ["-3", "{0,0,0}", "{0,0,0}", "{0,0,0}"]]), rows
    assert "result_fetch_states" in err and "result_fetch_sxx" in err


@needs_double
def test_host_logic_final_values_and_nulls():
    fns = [g.GX_AGG_STDDEV_SAMP_F8, g.GX_AGG_VAR_POP_F8]
    keys = np.array([[17], [-3]], np.int64)
    aggs = np.array([[1.5, 0.25], [0.0, 0.0]])
    nulls = np.array([[0, 0, 0], [0, 1, 0]], np.uint8)                 # stddev_samp of one value is NULL, var_pop is 0
    with tempfile.TemporaryDirectory() as d:
        case, _, _ = lineitem_case(d, False, fns)
        res = os.path.join(d, "v.res")
        canned(res, keys, aggs, np.zeros((2, 2), np.int64), nulls)
        rows, err = run_double(case, res)
    assert sorted(rows) == sorted([["17", "1.5", "0.25"], ["-3", "\\N", "0"]]), rows
    assert "result_fetch (final values)" in err and "result_fetch_sxx" not in err


@pytest.mark.gpu
@needs_harness
def test_harness_variance_on_the_gpu():
    """SELECT l_shipdate, stddev(l_extendedprice), var_pop(l_extendedprice) FROM lineitem GROUP BY l_shipdate through
    Begin/Exec/End"""
    fns = [g.GX_AGG_STDDEV_SAMP_F8, g.GX_AGG_VAR_POP_F8]
    with tempfile.TemporaryDirectory() as d:
        case, l, p = lineitem_case(d, False, fns, n=60000)
        r = subprocess.run([HARNESS, case], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    rows = [line.split("\t") for line in r.stdout.splitlines() if line]
    price, ship_date = np.asarray(l[2]), np.asarray(l[5])
    assert len(rows) == len(np.unique(ship_date))
    for row in rows:
        x = price[ship_date == int(row[0])]
        for a, fn in enumerate(fns):
            want = V.expect(fn, x)
            null = row[1 + a] == "\\N"
            assert V.matches(fn, want, 0.0 if null else float(row[1 + a]), null), (row, want)
