"""Exact per-group expectations of an aggregate over a chain of INNER hash joins (gx_hash_agg_joins), CPU only, built on
tests/join_ref.py and tests/exact_ref.py.

Semantics: the plan's quals select the outer rows first; then step 1, 2, ... each join the surviving rows to one build
side with join_ref.join (its build quals applied, NULL keys never matching, int4 / date keys compared by value with
int8 ones).  A step's key is an outer column (side 0) or a payload column of an earlier step (side s >= 1).  The
aggregates read outer columns; a group column is an outer column (side 0) or a payload column of step s (side s)."""
from collections import namedtuple

import numpy as np

import opentenbase_b200 as g
import join_ref as J

# one build side of the chain: key = (side, col) the probe key comes from, bkey / bnull its key column and NULL flags,
# payload / ptypes its payload columns, bkeep the build rows that passed its quals (None = all)
Step = namedtuple("Step", "key bkey payload ptypes bnull bkeep", defaults=(None, None))


def chain_rows(plan, outer_cols, outer_types, steps, outer_nulls=None):
    """(outer rows, [build row of step s for each]) of the rows that pass the quals and find a partner at every step,
    each outer row as often as the joins produce it"""
    n = len(outer_cols[0])
    nulls = outer_nulls or [None] * len(outer_cols)
    preds = [(plan.preds[p].col, plan.preds[p].op, plan.preds[p].fval if outer_types[plan.preds[p].col] == g.GX_FLOAT8
              else plan.preds[p].ival) for p in range(plan.n_preds)]
    o = np.flatnonzero(J.quals(outer_cols, nulls, preds, n))
    brows = []
    for st in steps:
        side, col = st.key
        if side == 0:
            kv = np.asarray(outer_cols[col])[o]
            kn = None if nulls[col] is None else np.asarray(nulls[col])[o]
        else:
            kv, kn = np.asarray(steps[side - 1].payload[col])[brows[side - 1]], None      # a payload is never NULL
        oi, ii = J.join(g.GX_JOIN_INNER, kv, st.bkey, kn, st.bnull, None, st.bkeep)
        o = o[oi]
        brows = [b[oi] for b in brows] + [ii]
    return o, brows


def expect_chain_groups(plan, outer_cols, outer_types, steps, outer_nulls=None):
    """exact_ref.expect_groups of the plan over the rows of the join chain: {group key tuple: [Expect per aggregate]}"""
    o, brows = chain_rows(plan, outer_cols, outer_types, steps, outer_nulls)
    # every step's payload gathered at its rows, side by side: (s, col) -> payload column offset[s] + col
    gathered, gtypes, offset = [], [], [0]
    for st, b in zip(steps, brows):
        gathered += [np.asarray(c)[b] for c in st.payload]
        gtypes += list(st.ptypes)
        offset.append(offset[-1] + len(st.payload))
    flat = type(plan).from_buffer_copy(bytes(plan))
    for c in range(plan.n_group_cols):
        side, col = plan.group_cols[c].side, plan.group_cols[c].col
        if side > 0:
            flat.group_cols[c].side, flat.group_cols[c].col = 1, offset[side - 1] + col
    return J.expect_groups(flat, (o, np.arange(len(o))), outer_cols, outer_types, gathered, gtypes, outer_nulls=outer_nulls)
