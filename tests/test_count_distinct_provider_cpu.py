"""The provider's count(DISTINCT col): what gpuexec_match_plan takes and declines, the descriptor it ships, its cost, its
host logic against the ABI double, and one run through Begin/Exec/End on the GPU.

Taken: count(DISTINCT v) over an int4 / int8 / date column of the outer relation, with no ORDER BY or FILTER, every
DISTINCT aggregate on that column, the group key plus the column within 16 bytes, in a plan pushed down whole or on a
single node.  est_groups becomes the estimate of distinct (group, value) pairs (the harness's "pairs N" line stands in
for estimate_num_groups), bounded by the input rows."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
from test_provider_harness import HARNESS, write_case
from test_provider_planner_cpu import LINEITEM, ORDERS, parse_desc, plan
from test_provider_host_logic_cpu import DOUBLE, canned, run as run_double
from test_provider_ship_cpu import ship
from test_star_agg_cpu import CUSTOMER, parse_chain_desc

needs_harness = pytest.mark.skipif(not os.path.exists(HARNESS), reason="harness binary not built (needs /root/reference at build time)")
CD = g.GX_AGG_COUNT_DISTINCT
INT8OID, DATEOID = 20, 1082
OTYPES = [O.GX_INT8, O.GX_INT4, O.GX_DATE, O.GX_INT4]


def one_scan(*extra, dist="dist none", pairs="pairs 400000"):
    return plan(ORDERS, "scan 2", "group 2.3", "target var 2.3", *extra, dist, "groups 2406", pairs)


@needs_harness
@pytest.mark.parametrize("att, gx_type", [("2.2", g.GX_INT4), ("2.1", g.GX_INT8), ("2.3", g.GX_DATE)])
def test_single_relation_is_taken_with_the_pair_estimate(att, gx_type):
    """SELECT o_orderdate, count(DISTINCT <col>), count(*) FROM orders GROUP BY o_orderdate"""
    r = one_scan(f"target agg count v{att} distinct", "target agg count_star")
    assert r is not None and r["path"] == "path pushdown: CustomScan"
    d = parse_desc(r["desc"])
    cols = d["outer"]["cols"]
    col = [c for c, (a, t) in enumerate(cols) if a == int(att.split(".")[1]) - 1 and t == gx_type][0]
    assert d["aggs"] == [(CD, [(g.GX_OP_COL, col, 0)]), (g.GX_AGG_COUNT_STAR, [])]
    assert d["est_groups"] == 400000 and r["rows"] == 2406
    # the pair estimate is bounded by the input rows
    assert parse_desc(one_scan("target agg count v2.2 distinct", pairs="pairs 1e12")["desc"])["est_groups"] == 1500000


@needs_harness
def test_join_and_chain_plans_are_taken():
    r = plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1", "group 2.3", "target var 2.3", "target agg count v1.1 distinct",
             "dist none", "groups 2406", "pairs 6000000")
    d = parse_desc(r["desc"])
    assert d["has_join"] and d["aggs"][0][0] == CD and d["est_groups"] == 6000000
    for jt in ("semi", "anti"):
        r = plan(LINEITEM, ORDERS, f"join 1.1 2.1 unique 0 {jt}", "group 1.6", "target var 1.6", "target agg count v1.1 distinct",
                 "dist none", "groups 2526", "pairs 100000")
        assert r is not None and parse_desc(r["desc"])["aggs"][0][0] == CD, jt
    r = plan(LINEITEM, ORDERS, CUSTOMER, "join 1.1 2.1 unique 1", "join 2.2 3.1 unique 1", "group 3.2", "target var 3.2",
             "target agg count v1.1 distinct", "dist none", "groups 5", "pairs 1000")
    assert r is not None and parse_chain_desc(r["desc"])["aggs"][0][0] == CD


@needs_harness
@pytest.mark.parametrize("extra, why", [
    (["target agg count v2.5 distinct"], "a float8 argument"),
    (["target agg count v2.2 distinct", "target agg count v2.4 distinct"], "two DISTINCT columns"),
    (["target agg sum_f8 v2.5 distinct"], "DISTINCT on sum(float8)"),
    (["target agg count v2.2 k1 + distinct"], "an expression argument"),
])
def test_declines_on_one_relation(extra, why):
    assert one_scan(*extra) is None, why


@needs_harness
def test_declines_elsewhere():
    tail = ["dist none", "groups 100", "pairs 1000"]
    # a build-side column
    assert plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1", "group 2.3", "target var 2.3", "target agg count v2.2 distinct", *tail) is None
    # count(bpchar), DISTINCT or not
    assert plan(LINEITEM, "scan 1", "group 1.6", "target var 1.6", "target agg count v1.7 distinct", *tail) is None
    assert plan(LINEITEM, "scan 1", "group 1.6", "target var 1.6", "target agg count v1.7", *tail) is None
    # int8 + date + bpchar(1) group key and a date argument: 17 bytes; without the bpchar column 16 bytes fit
    assert plan(LINEITEM, "scan 1", "group 1.1", "group 1.6", "group 1.7", "target agg count v1.6 distinct", *tail) is None
    assert plan(LINEITEM, "scan 1", "group 1.1", "group 1.6", "target agg count v1.6 distinct", *tail) is not None
    # a two-phase plan: GROUP BY does not cover the distribution key (the same plan with count(col) is taken two-phase)
    two = [LINEITEM, "scan 1", "group 1.6", "target var 1.6"]
    assert plan(*two, "target agg count v1.1", "dist shard 1.1 nodes 4", "groups 2526") is not None
    assert plan(*two, "target agg count v1.1 distinct", "dist shard 1.1 nodes 4", "groups 2526", "pairs 1000") is None
    assert plan(*two, "target agg count v1.1 distinct", "dist replicated", "groups 2526", "pairs 1000") is not None


@needs_harness
def test_cost_has_a_term_for_the_pairs_and_none_without_distinct():
    plain = one_scan("target agg count v2.2", pairs="pairs 400000")
    assert plain == one_scan("target agg count v2.2", pairs="pairs 1")       # no DISTINCT: the pair estimate is not read
    few, many = one_scan("target agg count v2.2 distinct", pairs="pairs 10"), one_scan("target agg count v2.2 distinct", pairs="pairs 1500000")
    assert plain["total"] <= few["total"] < many["total"]


@needs_harness
def test_descriptor_survives_plan_shipping():
    o = O.gen_orders(1, 0, 200)
    orel = O.Rel(OTYPES, o)
    p = g.make_plan(group_cols=[(0, 1)], aggs=[(CD, [(g.GX_OP_COL, 0, 0)]), (g.GX_AGG_COUNT_STAR, [])], est_groups=2**33 + 7)
    with tempfile.TemporaryDirectory() as d:
        case = os.path.join(d, "cd.case")
        write_case(case, [(OTYPES, orel)], {"rti": 1, "attnums": [1, 2]}, None, p, False, [DATEOID, INT8OID, INT8OID])
        wire = ship(case)
    assert wire


@pytest.mark.skipif(not os.path.exists(DOUBLE), reason="harness binary not built (needs /root/reference at build time)")
def test_host_logic_emits_the_count_as_int8():
    o = O.gen_orders(1, 0, 300)
    orel = O.Rel(OTYPES, o)
    p = g.make_plan(group_cols=[(0, 1)], aggs=[(CD, [(g.GX_OP_COL, 0, 0)]), (g.GX_AGG_COUNT_STAR, [])], est_groups=100)
    keys = np.array([[-3000], [17]], np.int64)
    aggs = np.array([[5, 9], [0, 2]], np.int64).view(np.float64)
    with tempfile.TemporaryDirectory() as d:
        case, res = os.path.join(d, "cd.case"), os.path.join(d, "cd.res")
        write_case(case, [(OTYPES, orel)], {"rti": 1, "attnums": [1, 2]}, None, p, False, [DATEOID, INT8OID, INT8OID])
        canned(res, keys, aggs, np.zeros((2, 2), np.int64), np.zeros((2, 3), np.uint8))
        rows, err = run_double(case, res)
    assert sorted(rows) == sorted([["-3000", "5", "9"], ["17", "0", "2"]]), rows
    assert "GPU Distinct Column" in err


@pytest.mark.gpu
@needs_harness
def test_harness_count_distinct_on_the_gpu():
    """SELECT o_orderdate, count(DISTINCT o_custkey), count(*) FROM orders GROUP BY o_orderdate through Begin/Exec/End"""
    o = O.gen_orders(1, 0, 60000)
    orel = O.Rel(OTYPES, o)
    p = g.make_plan(group_cols=[(0, 1)], aggs=[(CD, [(g.GX_OP_COL, 0, 0)]), (g.GX_AGG_COUNT_STAR, [])], est_groups=60000)
    with tempfile.TemporaryDirectory() as d:
        case = os.path.join(d, "cd.case")
        write_case(case, [(OTYPES, orel)], {"rti": 1, "attnums": [1, 2]}, None, p, False, [DATEOID, INT8OID, INT8OID])
        r = subprocess.run([HARNESS, case], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    got = {int(a): (int(b), int(c)) for a, b, c in (l.split("\t") for l in r.stdout.splitlines() if l)}
    cust, date = np.asarray(o[1]), np.asarray(o[2])
    want = {}
    for dt in np.unique(date):
        m = date == dt
        want[int(dt)] = (len(np.unique(cust[m])), int(m.sum()))
    assert got == want
    assert "GPU Distinct Column" in r.stderr
