"""Exact per-group expectations of an aggregate over a right semi or right anti hash join, CPU only, built on
tests/join_ref.py and tests/exact_ref.py.

Semantics (gx_hash_agg_right, nodeHashjoin.c's JOIN_SEMI_RIGHT / JOIN_ANTI_RIGHT arms): the build side B is the
preserved relation and the probe side P only decides which of B's rows survive.  SEMI_RIGHT consumes once every B row
that passes the build quals and the plan's quals and whose non-NULL key equals the non-NULL key of a P row passing P's
quals; ANTI_RIGHT consumes the B rows passing those quals that have no such partner, NULL keys included.  That is
join_ref's SEMI / ANTI with B as the outer side and P as the inner one.  The aggregate reads B's columns only."""
import numpy as np

import opentenbase_b200 as g
import exact_ref as X
import join_ref as J
import distinct_ref as D

AS_LEFT = {g.GX_JOIN_SEMI_RIGHT: g.GX_JOIN_SEMI, g.GX_JOIN_ANTI_RIGHT: g.GX_JOIN_ANTI}


def plan_preds(plan, types):
    """the plan's quals as join_ref.quals takes them"""
    return [(plan.preds[p].col, plan.preds[p].op, plan.preds[p].fval if types[plan.preds[p].col] == g.GX_FLOAT8
             else plan.preds[p].ival) for p in range(plan.n_preds)]


def consumed(jt, bcols, bkey_col, pkey, bnulls=None, pnull=None, pkeep=None, bpreds=(), btypes=None):
    """the build rows (ascending) a join of type jt consumes.  bpreds: the build quals and the plan's quals together;
    pkeep: probe rows that passed the probe quals; pnull: the probe key's NULL flags"""
    n = len(bcols[0])
    nulls = bnulls or [None] * len(bcols)
    bkeep = J.quals(bcols, nulls, list(bpreds), n)
    o, _ = J.join(AS_LEFT[jt], bcols[bkey_col], pkey, nulls[bkey_col], pnull, bkeep, pkeep)
    return np.sort(o)


def expect_right_groups(plan, jt, bcols, btypes, bkey_col, pkey, bnulls=None, pnull=None, pkeep=None, bpreds=()):
    """{group key tuple: [Expect per aggregate]} (or "overflow") of the plan over the build rows the join consumes;
    count(DISTINCT) goes through tests/distinct_ref.py"""
    o = consumed(jt, bcols, bkey_col, pkey, bnulls, pnull, pkeep, list(bpreds) + plan_preds(plan, btypes))
    flat = type(plan).from_buffer_copy(bytes(plan))
    flat.n_preds = 0
    if any(plan.aggs[a].fn == g.GX_AGG_COUNT_DISTINCT for a in range(plan.n_aggs)):
        return D.expect_groups(flat, bcols, btypes, o, bnulls)
    nulls = bnulls or [None] * len(bcols)
    cols = [np.asarray(c)[o] for c in bcols]
    nl = [None if x is None else np.asarray(x)[o] for x in nulls]
    return X.expect_groups(flat, cols, nulls=nl, types=list(btypes))
