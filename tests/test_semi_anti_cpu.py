"""Aggregates over SEMI and ANTI hash joins, without a GPU: the provider's planner accepts them under the conditions an
INNER join has and carries the join type in its descriptor, the descriptor survives coordinator -> datanode shipping
through the reference's own nodes/read.c, and tests/exists_ref.py's per-group expectations for SEMI / ANTI equal the
oracle's aggregate over ExecHashJoinImpl's SEMI and ANTI arms."""
import os
import tempfile

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import join_ref as J
import exists_ref as E
from test_provider_harness import HARNESS, write_case
from test_provider_planner_cpu import LINEITEM, ORDERS, parse_desc, plan
from test_provider_ship_cpu import LTYPES, OTYPES, ship

needs_harness = pytest.mark.skipif(not os.path.exists(HARNESS), reason="harness binary not built (needs /root/reference at build time)")
TAIL = ["group 1.6", "target var 1.6", "target agg count_star", "target agg sum_f8 v1.3", "dist none", "groups 2526"]


@needs_harness
@pytest.mark.parametrize("word,jt", [("semi", g.GX_JOIN_SEMI), ("anti", g.GX_JOIN_ANTI)])
def test_planner_takes_semi_and_anti_and_the_descriptor_carries_the_join_type(word, jt):
    r = plan(LINEITEM, ORDERS, f"join 1.1 2.1 unique 0 {word}", "qual 2 3 date_lt date -1752", *TAIL)
    assert r is not None and r["path"].startswith("path pushdown")
    d = r["desc"]
    assert d[1] == 1 + jt                      # the word after the version: 0 no join, else 1 + GX_JOIN_*
    d = parse_desc([d[0], 1] + d[2:])         # otherwise the INNER layout, word for word
    ocols = [c for c, _ in d["outer"]["cols"]]
    icols = [c for c, _ in d["inner"]["cols"]]
    assert d["inner_unique"] == 0 and d["payload"] == [] and d["group_cols"] == [(0, ocols.index(5))]
    assert ocols[d["outer_key_col"]] == 0 and icols[d["inner_key_col"]] == 0
    assert d["inner_preds"] == [(icols.index(2), g.GX_LT, -1752, 0)]


@needs_harness
def test_inner_descriptor_is_unchanged():
    r = plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1", *TAIL)
    assert r["desc"][1] == 1 and parse_desc(r["desc"])["has_join"] == 1


@needs_harness
@pytest.mark.parametrize("word", ["semi", "anti"])
def test_semi_and_anti_decline_inner_side_columns(word):
    head = [LINEITEM, ORDERS, f"join 1.1 2.1 unique 0 {word}"]
    assert plan(*head, "group 2.3", "target var 2.3", "target agg count_star", "dist none") is None              # GROUP BY an inner column
    assert plan(*head, "group 1.6", "target var 1.6", "target agg sum_f8 v2.5", "dist none") is None             # aggregate over an inner column
    assert plan(*head, "group 1.6", "target var 1.6", "target agg count_star", "dist none") is not None


@needs_harness
@pytest.mark.parametrize("word", ["right", "full", "left"])
def test_other_join_types_decline(word):
    assert plan(LINEITEM, ORDERS, f"join 1.1 2.1 unique 1 {word}", *TAIL) is None


@needs_harness
@pytest.mark.parametrize("jt", [g.GX_JOIN_SEMI, g.GX_JOIN_ANTI])
def test_semi_anti_descriptor_survives_plan_shipping(jt):
    orel, lrel = O.Rel(OTYPES, O.gen_orders(1, 0, 200)), O.Rel(LTYPES, O.gen_lineitem(1, 0, 200))
    p = g.make_plan(preds=[(1, g.GX_GT, -1000)], outer_key_col=0, group_cols=[(0, 1)], aggs=[(g.GX_AGG_COUNT_STAR, [])],
                    est_groups=2**33 + 1, join_type=jt)
    with tempfile.TemporaryDirectory() as d:
        case = os.path.join(d, "semi.case")
        write_case(case, [(LTYPES, lrel), (OTYPES, orel)], {"rti": 1, "attnums": [0, 5]},
                   {"rti": 2, "attnums": [0, 2], "key_col": 0, "payload_cols": [], "unique": False, "preds": [(1, g.GX_LT, -1752)]},
                   p, False, [1082, 20])
        wire = ship(case)
    toks = wire.strip("()").split(" ")
    assert toks[1] == str(1 + jt) and toks[-1] == str(2**33 + 1)


def _data(rng, n_outer, n_build):
    """int8 outer keys against a build side with duplicates, NULL keys on both sides, INT64_MIN on both sides"""
    I64 = np.iinfo(np.int64)
    bk = np.concatenate([rng.integers(-50, 50, n_build - 4), [I64.min, I64.min, I64.max, 2**32]])
    bk = np.concatenate([bk, bk[rng.integers(0, len(bk), n_build // 2)]])       # duplicates
    bnull = (rng.random(len(bk)) < 0.08).astype(np.uint8)
    bq = rng.integers(0, 10, len(bk)).astype(np.int32)
    ok = np.concatenate([rng.integers(-80, 80, n_outer - 4), [I64.min, I64.max, 2**32, 2**32 + 1]])
    onull = (rng.random(n_outer) < 0.08).astype(np.uint8)
    og = rng.integers(0, 7, n_outer).astype(np.int32)
    ox = rng.standard_normal(n_outer) * 10.0 ** rng.integers(-3, 4, n_outer)
    return (bk, bnull, bq), (ok, onull, og, ox)


@pytest.mark.parametrize("jt", [g.GX_JOIN_SEMI, g.GX_JOIN_ANTI])
@pytest.mark.parametrize("grouped", [True, False])
def test_exists_groups_match_the_oracle(jt, grouped):
    """exists_ref.expect_exists_groups against orc_exec_agg over the SEMI / ANTI arm (make_join jointype 4 / 5), with quals on both
    sides, duplicate build keys, NULL keys on both sides and INT64_MIN keys"""
    rng = np.random.default_rng(31 + jt + 2 * grouped)
    (bk, bnull, bq), (ok, onull, og, ox) = _data(rng, 900, 120)
    ot, it = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8], [g.GX_INT8, g.GX_INT4]
    ocols, onulls = [ok, og, ox], [onull, None, None]
    ipreds = [(1, g.GX_GE, 2)]
    aggs = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 1, 0)]), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)]),
            (g.GX_AGG_MAX_F8, [(g.GX_OP_COL, 2, 0)])]
    plan_ = g.make_plan(preds=[(2, g.GX_LT, 5.0, True)], outer_key_col=0, group_cols=[(0, 1)] if grouped else [], aggs=aggs,
                        est_groups=10, join_type=jt)
    oplan = O.GxAggPlan.from_buffer_copy(bytes(plan_))          # the oracle reads the join type from make_join
    join = O.make_join(0, inner_unique=0, inner_preds=ipreds, jointype=jt)
    r = O.exec_agg(O.Rel(ot, ocols, onulls), oplan, O.Rel(it, [bk, bq], [bnull, None]), join)
    want = E.expect_exists_groups(plan_, jt, ocols, ot, bk, outer_nulls=onulls, inull=bnull,
                                  ikeep=J.quals([bk, bq], None, ipreds, len(bk)))
    X.check(plan_, want, (r.keys, r.aggs, r.nulls), [g.GX_INT4] if grouped else [])
    assert sum(e[0].value for e in want.values()) > 50


def test_semi_counts_a_row_once_and_anti_keeps_null_keys():
    """the two rules the helper exists for, on a hand-sized case"""
    ok = np.array([1, 1, 2, 3, 0], np.int64)
    onull = np.array([0, 0, 0, 0, 1], np.uint8)
    og = np.array([10, 10, 20, 30, 40], np.int32)
    bk = np.array([1, 1, 1, 3, 0], np.int64)
    bnull = np.array([0, 0, 0, 0, 1], np.uint8)
    p = g.make_plan(outer_key_col=0, group_cols=[(0, 1)], aggs=[(g.GX_AGG_COUNT_STAR, [])])
    cols, ot = [ok, og], [g.GX_INT8, g.GX_INT4]
    semi = E.expect_exists_groups(p, g.GX_JOIN_SEMI, cols, ot, bk, outer_nulls=[onull, None], inull=bnull)
    anti = E.expect_exists_groups(p, g.GX_JOIN_ANTI, cols, ot, bk, outer_nulls=[onull, None], inull=bnull)
    assert {k: v[0].value for k, v in semi.items()} == {(10,): 2, (30,): 1}
    assert {k: v[0].value for k, v in anti.items()} == {(20,): 1, (40,): 1}
