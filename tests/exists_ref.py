"""Exact per-group expectations of an aggregate over a SEMI or ANTI hash join, CPU only, built on tests/join_ref.py.

Semantics (gx_agg_plan.join_type, nodeHashjoin.c's SEMI / ANTI arms): the plan's quals select the outer rows before the
join; SEMI keeps an outer row once if a build row has its key, however many do; ANTI keeps an outer row without a
partner, a NULL key included; the GROUP BY and the aggregates read outer columns only."""
import opentenbase_b200 as g
import join_ref as J


def expect_exists_groups(plan, jt, outer_cols, outer_types, ikey, outer_nulls=None, inull=None, ikeep=None):
    """exact_ref.expect_groups of the plan over the rows a SEMI / ANTI join of type jt keeps.  ikey / inull: the build
    side's key column and its NULL flags; ikeep: build rows that passed the build side's quals."""
    assert jt in (g.GX_JOIN_SEMI, g.GX_JOIN_ANTI), jt
    n = len(outer_cols[0])
    nulls = outer_nulls or [None] * len(outer_cols)
    preds = [(plan.preds[p].col, plan.preds[p].op, plan.preds[p].fval if outer_types[plan.preds[p].col] == g.GX_FLOAT8
              else plan.preds[p].ival) for p in range(plan.n_preds)]
    okeep = J.quals(outer_cols, nulls, preds, n)
    kc = plan.outer_key_col
    pairs = J.join(jt, outer_cols[kc], ikey, nulls[kc], inull, okeep, ikeep)
    return J.expect_groups(plan, pairs, outer_cols, outer_types, [], [], outer_nulls=nulls)
