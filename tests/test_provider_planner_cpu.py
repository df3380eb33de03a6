"""The provider's PLANNER side executed without a GPU and without a backend.

`provider/harness/gpuexec_harness --plan <scenario>` builds the PlannerInfo / Query / RelOptInfo / Path / Var / Aggref /
RestrictInfo nodes a query would arrive with at create_upper_paths_hook (hand-built from a small scenario file), calls
gpuexec_upper_paths_hook and PlanCustomPath, and prints what came out: the path shape (pushed down whole, or Partial ->
redistribute -> Finalize), its costs, the plan descriptor as it travels to the datanodes, and the scan tuple
(custom_scan_tlist).  The planner-side helpers the hook calls (get_sortgroupclause_tle, add_column_to_pathtarget,
mark_partial_aggref, makeTargetEntry, add_path, ...) are small restatements of the reference's, cited in the harness.

What is pinned here: which plans are accepted and which decline (planner.c:10026 push-down rule, the qual / join /
aggregate shapes of gpuexec_match_plan), the column numbering of the descriptor against the order columns are first
referenced, flipped `Const op Var` quals, inner-side GROUP BY columns riding in the join payload, and — the round-1
advisor finding — that the scan tuple is (GROUP BY columns in groupClause order, aggregates in target-list order) whatever
order the SELECT list has, with resjunk GROUP BY columns included."""
import os
import struct
import subprocess
import tempfile

import pytest

import opentenbase_b200 as g
from test_provider_harness import HARNESS

pytestmark = pytest.mark.skipif(not os.path.exists(HARNESS), reason="harness binary not built (needs /root/reference at build time)")

LINEITEM = "rel 1 tuples 6000000 pages 110000 cols int8 float8 float8 float8 float8 date bpchar1 bpchar1"   # orderkey qty price disc tax shipdate flag status
ORDERS = "rel 2 tuples 1500000 pages 26000 cols int8! int4! date! int4! float8! int8"                       # orderkey custkey orderdate shippriority totalprice (all NOT NULL), a nullable int8
INT8, FLOAT8, DATE, BPCHAR = 20, 701, 1082, 1042
F8ARRAY = 1022


def plan(*lines):
    with tempfile.NamedTemporaryFile("w", suffix=".scn", delete=False) as f:
        f.write("\n".join(lines) + "\n")
    try:
        r = subprocess.run([HARNESS, "--plan", f.name], capture_output=True, text=True, timeout=60)
    finally:
        os.unlink(f.name)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = r.stdout.splitlines()
    if out[0] == "declined":
        return None
    res = {"path": out[0], "scan": []}
    for l in out[1:]:
        w = l.split()
        if w[0] == "cost":
            res["startup"], res["total"], res["rows"] = float(w[2]), float(w[4]), float(w[6])
        elif w[0] == "desc":
            res["desc"] = [int(t) for t in l[5:].strip("()").split(" ")]
        elif w[0] == "scan":
            res["scan"].append(tuple(w[2:]))
        elif w[0] == "plan_tlist":
            res["plan_tlist"], res["scanrelid"] = int(w[1]), int(w[3])
    return res


def f8bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def parse_desc(d):
    """The wire layout of gpuexec_serialise (provider/gpuexec_provider.c)."""
    it = iter(d)
    nx = lambda: next(it)
    out = {"abi": nx(), "has_join": nx()}

    def rel():
        rti, n = nx(), nx()
        return {"rti": rti, "cols": [(nx(), nx()) for _ in range(n)]}
    out["outer"] = rel()
    if out["has_join"]:
        out["inner"] = rel()
        out["inner_key_col"] = nx()
        out["payload"] = [nx() for _ in range(nx())]
        out["inner_unique"] = nx()
        out["inner_preds"] = [(nx(), nx(), nx(), nx()) for _ in range(nx())]
    out["partial"] = nx()
    npred = nx()
    out["outer_key_col"] = nx()
    out["preds"] = [(nx(), nx(), nx(), nx()) for _ in range(npred)]
    out["group_cols"] = [(nx(), nx()) for _ in range(nx())]
    aggs = []
    for _ in range(nx()):
        fn, nops = nx(), nx()
        aggs.append((fn, [(nx(), nx(), nx()) for _ in range(nops)]))
    out["aggs"] = aggs
    out["est_groups"] = nx()
    assert next(it, None) is None
    return out


def test_config1_is_pushed_down_whole_and_the_scan_tuple_ignores_select_order():
    """SELECT count(*), l_returnflag FROM lineitem GROUP BY l_returnflag — aggregate first in the SELECT list."""
    r = plan(LINEITEM, "scan 1", "group 1.7", "target agg count_star", "target var 1.7", "dist none", "groups 3")
    assert r["path"] == "path pushdown: CustomScan" and r["scanrelid"] == 0 and r["plan_tlist"] == 2
    assert r["scan"] == [("var", "1.7", "type", str(BPCHAR)), ("agg", "2803", "type", str(INT8), "split", "0")]
    d = parse_desc(r["desc"])
    assert d["abi"] == 1 and not d["has_join"] and not d["partial"]
    assert d["outer"] == {"rti": 1, "cols": [(6, g.GX_CHAR)]}          # attnum 7 -> 0-based 6, bpchar(1) staged as one byte
    assert d["group_cols"] == [(0, 0)] and d["aggs"] == [(g.GX_AGG_COUNT_STAR, [])] and d["est_groups"] == 3


def test_group_by_column_that_is_not_selected_is_a_junk_entry_and_still_in_the_scan_tuple():
    """SELECT sum(l_extendedprice) FROM lineitem GROUP BY l_shipdate (config 2 without the key in the SELECT list)."""
    r = plan(LINEITEM, "scan 1", "group 1.6", "target agg sum_f8 v1.3", "dist replicated", "groups 2526")
    assert r["path"].startswith("path pushdown") and r["plan_tlist"] == 2            # the junk GROUP BY entry is in the plan's tlist
    assert r["scan"] == [("var", "1.6", "type", str(DATE)), ("agg", "2111", "type", str(FLOAT8), "split", "0")]
    d = parse_desc(r["desc"])
    # columns are numbered in the order the matcher first meets them: GROUP BY before the aggregate arguments
    assert d["outer"]["cols"] == [(5, g.GX_DATE), (2, g.GX_FLOAT8)]
    assert d["group_cols"] == [(0, 0)] and d["aggs"] == [(g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])]


def test_q1_expressions_quals_and_two_group_columns():
    r = plan(LINEITEM, "scan 1", "qual 1 6 date_le date -607",
             "group 1.7", "group 1.8",
             "target var 1.7", "target var 1.8", "target agg sum_f8 v1.2", "target agg sum_f8 v1.3 k1 v1.4 - *",
             "target agg sum_f8 v1.3 k1 v1.4 - * k1 v1.5 + *", "target agg avg_f8 v1.4", "target agg count_star", "dist none", "groups 6")
    assert r["path"].startswith("path pushdown")
    assert [s[0] for s in r["scan"]] == ["var", "var", "agg", "agg", "agg", "agg", "agg"]
    d = parse_desc(r["desc"])
    cols = [c for c, _ in d["outer"]["cols"]]
    assert cols[0] == 5                                               # the qual column is met first
    assert d["preds"] == [(0, g.GX_LE, -607, 0)]
    col = {att: i for i, att in enumerate(cols)}
    C, K, S, M, A = g.GX_OP_COL, g.GX_OP_CONST, g.GX_OP_SUB, g.GX_OP_MUL, g.GX_OP_ADD
    one = f8bits(1.0)
    assert d["group_cols"] == [(0, col[6]), (0, col[7])]
    assert d["aggs"][0] == (g.GX_AGG_SUM_F8, [(C, col[1], 0)])
    assert d["aggs"][1] == (g.GX_AGG_SUM_F8, [(C, col[2], 0), (K, 0, one), (C, col[3], 0), (S, 0, 0), (M, 0, 0)])
    assert d["aggs"][2][1][-4:] == [(K, 0, one), (C, col[4], 0), (A, 0, 0), (M, 0, 0)]
    assert d["aggs"][3][0] == g.GX_AGG_AVG_F8 and d["aggs"][4] == (g.GX_AGG_COUNT_STAR, [])


def test_config3_join_inner_group_column_rides_in_the_payload_and_quals_go_to_their_side():
    r = plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1",
             "qual 2 3 date_lt date -1752", "qual 1 6 date_gt date -1752 flip", "qual 2 1 int8ge int8 4611686018427400249",
             "group 2.3", "target var 2.3", "target agg count_star", "target agg sum_f8 v1.3", "dist none", "groups 2406")
    assert r["path"].startswith("path pushdown")
    assert r["scan"][0] == ("var", "2.3", "type", str(DATE))
    d = parse_desc(r["desc"])
    assert d["has_join"] and d["inner_unique"] == 1
    assert d["outer"]["rti"] == 1 and d["inner"]["rti"] == 2
    ocols = [c for c, _ in d["outer"]["cols"]]
    icols = [c for c, _ in d["inner"]["cols"]]
    assert ocols[d["outer_key_col"]] == 0 and icols[d["inner_key_col"]] == 0          # l_orderkey = o_orderkey
    assert d["group_cols"] == [(1, 0)] and [icols[c] for c in d["payload"]] == [2]    # o_orderdate is payload slot 0
    # `const > var` was written flipped: -1752 > l_shipdate  ==  l_shipdate < -1752
    assert d["preds"] == [(ocols.index(5), g.GX_LT, -1752, 0)]
    assert sorted(d["inner_preds"]) == sorted([(icols.index(2), g.GX_LT, -1752, 0), (icols.index(0), g.GX_GE, 4611686018427400249, 0)])


def test_join_written_inner_side_first_is_normalised():
    a = plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1", "group 2.3", "target var 2.3", "target agg count_star", "dist none")
    b = plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1 swapped", "group 2.3", "target var 2.3", "target agg count_star", "dist none")
    assert a["desc"] == b["desc"]


def test_distribution_decides_between_push_down_and_two_phase():
    """planner.c:10026 can_push_down_grouping: GROUP BY covers the distribution key -> the whole aggregate below the
    RemoteSubplan; otherwise Partial -> Distribute -> Finalize (xc_groupby.out:193-205) with transition-typed columns."""
    base = [LINEITEM, "scan 1", "group 1.1", "target var 1.1", "target agg count_star", "target agg avg_f8 v1.3", "groups 1000"]
    covered = plan(*base, "dist shard 1.1 nodes 4")
    assert covered["path"] == "path pushdown: CustomScan" and not parse_desc(covered["desc"])["partial"]
    other = [LINEITEM, "scan 1", "group 1.6", "target var 1.6", "target agg count_star", "target agg avg_f8 v1.3", "target agg sum_f8 v1.3", "groups 2526"]
    two = plan(*other, "dist shard 1.1 nodes 4")
    assert two["path"].startswith("path partial: Finalize Agg") and "RemoteSubplan" in two["path"]
    assert parse_desc(two["desc"])["partial"] == 1
    # the partial node returns transition values: int8 for count, float8[] for avg(float8), float8 for sum(float8); split = INITIAL_SERIAL
    assert two["scan"] == [("var", "1.6", "type", str(DATE)), ("agg", "2803", "type", str(INT8), "split", "6"),
                           ("agg", "2105", "type", str(F8ARRAY), "split", "6"), ("agg", "2111", "type", str(FLOAT8), "split", "6")]
    # costs are per datanode: four nodes read a quarter of the pages each
    one = plan(*other, "dist none")
    assert two["total"] < one["total"] / 3


@pytest.mark.parametrize("extra,why", [
    (["having"], "HAVING"),
    (["groupingsets"], "grouping sets"),
    (["target agg sum_numeric v1.2"], "an aggregate without a device counterpart"),
    (["target agg sum_f8 v1.3 distinct"], "DISTINCT aggregates"),
    (["target agg sum_f8 v1.3 k2 /"], "an operator outside + - *"),
    (["target var 1.2"], "a selected column that is not grouped"),
    (["qual 1 1 int84lt int4 5"], "a cross-type comparison"),
    (["qual 1 6 date_lt date null"], "a NULL constant"),
    (["protected"], "a relation under CLS / data masking / FGA"),
])
def test_declines(extra, why):
    assert plan(LINEITEM, "scan 1", "group 1.7", "target var 1.7", "target agg count_star", *extra, "dist none") is None, why


def test_join_shapes_that_decline():
    tail = ["group 2.3", "target var 2.3", "target agg count_star", "dist none"]
    assert plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1 left", *tail) is None                      # outer joins
    assert plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1 remote_inner", *tail) is None              # a redistribute below the join
    assert plan(LINEITEM, ORDERS, "join 1.6 2.3 unique 0", *tail) is None                           # date = date: only int4/int8 keys
    assert plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1", "group 2.3", "target var 2.3", "target agg sum_f8 v2.2", "dist none") is None   # aggregate over an inner column


def test_costs_follow_the_cost_model():
    """The path's numbers are gpuexec_cost.h's (tests/test_provider_cost_cpu.py): disk + (feed + device + start-up) / unit."""
    r = plan(LINEITEM, "scan 1", "group 1.6", "target var 1.6", "target agg sum_f8 v1.3", "dist none", "groups 2526")
    pages, tuples = 110000.0, 6000000.0
    staged = tuples * (4 + 8) * 1.25
    feed = max(1.5 * pages, pages * 8192 / 50e3)
    want = pages + (feed + 3 * staged / 3000e3 + 1500.0) / 10.0
    assert r["startup"] == pytest.approx(want, rel=1e-6)
    assert r["total"] == pytest.approx(want + 0.01 * 2526, rel=1e-6) and r["rows"] == 2526


def test_limits_of_the_library_decline_at_plan_time_instead_of_failing_at_run_time():
    """gx_hash_build carries the inner GROUP BY columns in ONE 8-byte payload word without NULL flags, gx_hash_agg packs the
    group key first-fit into two 8-byte words: what does not fit would be GX_ERR_ARG (an ERROR) at execution."""
    head = [LINEITEM, ORDERS, "join 1.1 2.1 unique 1"]
    tail = ["target agg count_star", "dist none"]
    ok = plan(*head, "group 2.3", "group 2.4", "target var 2.3", "target var 2.4", *tail)          # date + int4 = 8 bytes of payload
    assert ok is not None and parse_desc(ok["desc"])["group_cols"] == [(1, 0), (1, 1)]
    assert plan(*head, "group 2.2", "group 2.5", "target var 2.2", "target var 2.5", *tail) is None   # int4 + float8 = 12 bytes of payload
    assert plan(*head, "group 2.6", "target var 2.6", *tail) is None                                  # a nullable inner column
    three = plan(*head, "group 2.2", "group 2.3", "group 2.4", "target var 2.2", *tail)              # more than GX_MAX_PAYLOAD columns
    assert three is None
    # outer-side keys: int8 + int8 + date does not fit 8 + 8 first-fit; date + date + int8 does
    wide = "rel 1 tuples 1000 pages 10 cols int8 int8 date date float8"
    assert plan(wide, "scan 1", "group 1.1", "group 1.2", "group 1.3", "target agg sum_f8 v1.5", "dist none") is None
    assert plan(wide, "scan 1", "group 1.3", "group 1.4", "group 1.1", "target agg sum_f8 v1.5", "dist none") is not None


@pytest.mark.parametrize("att,typ", [(3, g.GX_DATE), (5, g.GX_FLOAT8)], ids=["date", "float8"])
def test_an_inner_column_grouped_twice_takes_one_payload_slot(att, typ):
    """GROUP BY o_orderdate, o_orderdate (or o_totalprice twice): both group columns read one payload slot, so a float8
    column fits the 8-byte payload word; the group key is the column twice"""
    r = plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1", f"group 2.{att}", f"group 2.{att}", "target agg count_star", "dist none")
    assert r is not None
    d = parse_desc(r["desc"])
    assert [d["inner"]["cols"][c] for c in d["payload"]] == [(att - 1, typ)]
    assert d["group_cols"] == [(1, 0), (1, 0)]


@pytest.mark.parametrize("name,lines,accepted", [
    ("8 aggregates", [LINEITEM, "scan 1", "group 1.7", "target var 1.7"] + ["target agg sum_f8 v1.2"] * 8 + ["dist none"], True),
    ("9 aggregates", [LINEITEM, "scan 1", "group 1.7", "target var 1.7"] + ["target agg sum_f8 v1.2"] * 9 + ["dist none"], False),
    ("5 group columns", [LINEITEM, "scan 1"] + [f"group 1.{i}" for i in (6, 7, 8, 1, 2)] + ["target agg count_star", "dist none"], False),
    ("an argument of 11 operations", [LINEITEM, "scan 1", "group 1.7", "target agg sum_f8 v1.2 v1.3 + v1.4 + v1.5 + v1.2 + v1.3 +", "dist none"], True),
    ("an argument of 15 operations", [LINEITEM, "scan 1", "group 1.7", "target agg sum_f8 v1.2 v1.3 + v1.4 + v1.5 + v1.2 + v1.3 + v1.4 + v1.5 +", "dist none"], False),
    ("4 quals", [LINEITEM, "scan 1"] + ["qual 1 6 date_lt date 5"] * 4 + ["group 1.7", "target agg count_star", "dist none"], True),
    ("5 quals", [LINEITEM, "scan 1"] + ["qual 1 6 date_lt date 5"] * 5 + ["group 1.7", "target agg count_star", "dist none"], False),
    ("no aggregate, no GROUP BY", [LINEITEM, "scan 1", "target var 1.1", "dist none"], False),
    ("aggregates without GROUP BY", [LINEITEM, "scan 1", "target agg count_star", "target agg sum_f8 v1.3", "dist none"], True),
    ("GROUP BY a relation that is not scanned", [LINEITEM, ORDERS, "scan 1", "group 2.3", "target agg count_star", "dist none"], False),
    ("count(bpchar)", [LINEITEM, "scan 1", "group 1.6", "target agg count v1.7", "dist none"], False),
    ("GROUP BY bpchar(3)", ["rel 1 tuples 10 pages 1 cols bpchar3 float8", "scan 1", "group 1.1", "target agg sum_f8 v1.2", "dist none"], False),
    ("GROUP BY text", ["rel 1 tuples 10 pages 1 cols text float8", "scan 1", "group 1.1", "target agg sum_f8 v1.2", "dist none"], False),
    ("bpchar(1) = 'R'", [LINEITEM, "scan 1", "qual 1 7 bpchareq bpchar1 R", "group 1.8", "target agg count_star", "dist none"], True),
    ("bpchar(1) = 'RX'", [LINEITEM, "scan 1", "qual 1 7 bpchareq bpchar1 RX", "group 1.8", "target agg count_star", "dist none"], False),
    ("sum(int4)", [ORDERS, "scan 2", "group 2.3", "target agg sum_i4 v2.2", "dist none"], True),
], ids=lambda x: x if isinstance(x, str) else None)
def test_capacity_edges_decline_cleanly(name, lines, accepted):
    """The descriptor's fixed capacities (GX_MAX_AGGS 8, GX_MAX_GROUP_COLS 4, GX_MAX_PREDS 4, GX_MAX_EXPR_OPS 12) and type limits:
    at the edge the plan is taken, one past it the hook declines — it never overruns the descriptor and never raises."""
    assert (plan(*lines) is not None) == accepted, name


def test_plain_aggregate_on_a_sharded_table_is_two_phase():
    """No GROUP BY, shard-distributed input: every datanode holds part of the one group -> Partial + Finalize (AGG_PLAIN)."""
    r = plan(LINEITEM, "scan 1", "target agg count_star", "target agg avg_f8 v1.3", "dist shard 1.1 nodes 2")
    assert r["path"].startswith("path partial: Finalize Agg (split 9, strategy 0)")          # AGGSPLIT_FINAL_DESERIAL, AGG_PLAIN
    assert [s[:4] for s in r["scan"]] == [("agg", "2803", "type", str(INT8)), ("agg", "2105", "type", str(F8ARRAY))]
