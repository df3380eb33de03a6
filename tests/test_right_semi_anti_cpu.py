"""Aggregates over right semi and right anti hash joins, without a GPU: tests/right_ref.py's per-group expectations equal
the oracle's aggregate over ExecHashJoinImpl's SEMI and ANTI arms with the build side as the outer relation, and the
constants and entry point of the C ABI are what the library and its Python binding use."""
import os
import re

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import join_ref as J
import right_ref as R

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gpuexec.h")


def _data(rng, n_build, n_probe):
    """a build side with duplicate keys, NULL keys and INT64_MIN; a probe side with the same kinds of keys"""
    I64 = np.iinfo(np.int64)
    bk = np.concatenate([rng.integers(-50, 50, n_build - 4), [I64.min, I64.min, I64.max, 2**32]])
    bk = np.concatenate([bk, bk[rng.integers(0, len(bk), n_build // 2)]])
    n = len(bk)
    bnull = (rng.random(n) < 0.08).astype(np.uint8)
    bg = rng.integers(0, 7, n).astype(np.int32)
    bx = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)
    pk = np.concatenate([rng.integers(-80, 80, n_probe - 4), [I64.min, I64.max, 2**32, 2**32 + 1]])
    pnull = (rng.random(n_probe) < 0.08).astype(np.uint8)
    pq = rng.integers(0, 10, n_probe).astype(np.int32)
    return (bk, bnull, bg, bx), (pk, pnull, pq)


@pytest.mark.parametrize("jt", [g.GX_JOIN_SEMI_RIGHT, g.GX_JOIN_ANTI_RIGHT])
@pytest.mark.parametrize("grouped", [True, False])
def test_right_groups_match_the_oracle(jt, grouped):
    """right_ref.expect_right_groups(P, B) against orc_exec_agg with B as the outer relation and P as the inner one over
    the SEMI / ANTI arm: quals on both sides and in the plan, duplicate keys, NULL and INT64_MIN keys on both sides"""
    rng = np.random.default_rng(7 + jt + 2 * grouped)
    (bk, bnull, bg, bx), (pk, pnull, pq) = _data(rng, 150, 700)
    bt, pt = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8], [g.GX_INT8, g.GX_INT4]
    bcols, bnulls = [bk, bg, bx], [bnull, None, None]
    bpreds, ppreds = [(1, g.GX_NE, 3)], [(1, g.GX_GE, 2)]
    aggs = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 1, 0)]), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)]),
            (g.GX_AGG_MAX_F8, [(g.GX_OP_COL, 2, 0)])]
    plan = g.make_plan(preds=[(2, g.GX_LT, 5.0, True)], group_cols=[(0, 1)] if grouped else [], aggs=aggs, est_groups=10)
    # the oracle: B outer, P inner, the left arm of the same name; B's quals are its scan quals
    oplan = O.make_plan(preds=[(2, g.GX_LT, 5.0, True)] + bpreds, outer_key_col=0, group_cols=[(0, 1)] if grouped else [],
                        aggs=aggs, est_groups=10)
    join = O.make_join(0, inner_unique=0, inner_preds=ppreds, jointype=R.AS_LEFT[jt])
    r = O.exec_agg(O.Rel(bt, bcols, bnulls), oplan, O.Rel(pt, [pk, pq], [pnull, None]), join)
    want = R.expect_right_groups(plan, jt, bcols, bt, 0, pk, bnulls, pnull, J.quals([pk, pq], None, ppreds, len(pk)), bpreds)
    X.check(plan, want, (r.keys, r.aggs, r.nulls), [g.GX_INT4] if grouped else [])
    assert sum(e[0].value for e in want.values()) > 10


def test_each_build_row_once_and_anti_keeps_null_keys():
    """the rules of the right forms on a hand-sized case: a build row is consumed once however many probe rows match it,
    every build row of a matched key is consumed, ANTI_RIGHT keeps a NULL-key build row, a NULL probe key matches nothing"""
    bk = np.array([1, 1, 2, 3, 0, 4], np.int64)
    bnull = np.array([0, 0, 0, 0, 1, 0], np.uint8)
    bg = np.array([10, 11, 20, 30, 40, 50], np.int32)
    pk = np.array([1, 1, 1, 3, 4, 0], np.int64)
    pnull = np.array([0, 0, 0, 0, 1, 1], np.uint8)
    p = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_COUNT_STAR, [])])
    cols, types = [bk, bg], [g.GX_INT8, g.GX_INT4]
    semi = R.expect_right_groups(p, g.GX_JOIN_SEMI_RIGHT, cols, types, 0, pk, [bnull, None], pnull)
    anti = R.expect_right_groups(p, g.GX_JOIN_ANTI_RIGHT, cols, types, 0, pk, [bnull, None], pnull)
    assert {k: v[0].value for k, v in semi.items()} == {(10,): 1, (11,): 1, (30,): 1}
    assert {k: v[0].value for k, v in anti.items()} == {(20,): 1, (40,): 1, (50,): 1}
    # an empty probe side: SEMI_RIGHT nothing, ANTI_RIGHT every build row
    none = np.zeros(0, np.int64)
    assert R.expect_right_groups(p, g.GX_JOIN_SEMI_RIGHT, cols, types, 0, none, [bnull, None]) == {}
    assert len(R.expect_right_groups(p, g.GX_JOIN_ANTI_RIGHT, cols, types, 0, none, [bnull, None])) == len(bk)


def test_abi_constants_and_entry_point():
    """the right join types carry the reference's JoinType values (nodes.h: JOIN_SEMI_RIGHT 8, JOIN_ANTI_RIGHT 9), the
    header declares gx_hash_agg_right and the binding knows it"""
    txt = open(HEADER).read()
    assert re.search(r"GX_JOIN_SEMI_RIGHT\s*=\s*8\b", txt) and re.search(r"GX_JOIN_ANTI_RIGHT\s*=\s*9\b", txt)
    assert (g.GX_JOIN_SEMI_RIGHT, g.GX_JOIN_ANTI_RIGHT) == (8, 9)
    assert "gx_hash_agg_right" in g.declared_symbols()
    assert re.search(r"#define GX_ABI_VERSION 1\b", txt)
