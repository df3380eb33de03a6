"""Exact per-group expectations of a plan with count(DISTINCT col) (GX_AGG_COUNT_DISTINCT), CPU only.

The input is the rows that reach the aggregate: the outer rows that passed the quals and the joins, each as often as
the joins produce it (tests/join_ref.py and tests/star_ref.py find them), with the payload columns of the join steps
gathered beside them.  A count(DISTINCT) is np.unique over the (group key with its NULL flags, argument) pairs of the
rows whose argument is not NULL, so a group whose arguments are all NULL counts 0.  Every other aggregate is
tests/exact_ref.py's expectation over the same rows and groups.  Group and argument columns are integer columns."""
import numpy as np

import opentenbase_b200 as g
import exact_ref as X


def _flat(plan, outer_cols, outer_types, o, outer_nulls, sides):
    """the rows o of the outer columns followed by every side's gathered payload columns, and the plan over them"""
    nulls = outer_nulls or [None] * len(outer_cols)
    cols = [np.asarray(c)[o] for c in outer_cols]
    fn = [None if nl is None else np.asarray(nl)[o] for nl in nulls]
    types = list(outer_types)
    offset = {}
    for s, (pcols, ptypes) in sorted((sides or {}).items()):
        offset[s] = len(cols)
        cols += [np.asarray(c) for c in pcols]
        fn += [None] * len(pcols)
        types += list(ptypes)
    flat = type(plan).from_buffer_copy(bytes(plan))
    for c in range(plan.n_group_cols):
        side, col = plan.group_cols[c].side, plan.group_cols[c].col
        flat.group_cols[c].side, flat.group_cols[c].col = 0, col + (offset[side] if side else 0)
    return flat, cols, fn, types


def _nl(nulls, c, n):
    return np.zeros(n, bool) if nulls[c] is None else np.asarray(nulls[c]).astype(bool)


def expect_groups(plan, outer_cols, outer_types, o, outer_nulls=None, sides=None):
    """{group key tuple: [Expect per aggregate]} (or "overflow") of the plan over the outer rows o.
    sides: {side s: (payload columns gathered at the rows o, their types)} for the group columns of side s >= 1."""
    flat, cols, nulls, types = _flat(plan, outer_cols, outer_types, np.asarray(o, np.int64), outer_nulls, sides)
    n = len(o)
    gcols = [flat.group_cols[c].col for c in range(flat.n_group_cols)]
    parts = []
    for c in gcols:
        nl = _nl(nulls, c, n)
        parts += [nl.astype(np.int64), np.where(nl, 0, cols[c].astype(np.int64))]
    if gcols:
        mat = np.stack(parts, 1) if n else np.zeros((0, 2 * len(gcols)), np.int64)
        uniq, gi = np.unique(mat, axis=0, return_inverse=True)
        gi = np.asarray(gi).reshape(-1)
        gkeys = [tuple(None if u[2 * j] else int(u[2 * j + 1]) for j in range(len(gcols))) for u in uniq]
    else:
        gi, gkeys = np.zeros(n, np.int64), [()]
    # the ordinary aggregates: exact_ref over the same groups
    other = type(flat).from_buffer_copy(bytes(flat))
    dist = [a for a in range(flat.n_aggs) if flat.aggs[a].fn == g.GX_AGG_COUNT_DISTINCT]
    keep_aggs = [a for a in range(flat.n_aggs) if a not in dist]
    for j, a in enumerate(keep_aggs):
        other.aggs[j] = flat.aggs[a]
    other.n_aggs = len(keep_aggs)
    if gcols:
        base = X.expect_groups(other, cols, nulls=nulls, types=types, gindex=gi, gkeys=gkeys)
    else:
        base = X.expect_groups(other, cols, nulls=nulls, types=types)
    if base == "overflow":
        return base
    # count(DISTINCT): distinct (group, argument) pairs with a non-NULL argument
    counts = {}
    if dist:
        c = flat.aggs[dist[0]].arg.ops[0].col
        assert all(flat.aggs[a].arg.ops[0].col == c for a in dist)
        ok = ~_nl(nulls, c, n)
        pairs = np.stack([gi[ok], cols[c][ok].astype(np.int64)], 1) if ok.any() else np.zeros((0, 2), np.int64)
        up = np.unique(pairs, axis=0)
        gid, cnt = np.unique(up[:, 0], return_counts=True)
        counts = {gkeys[int(k)]: int(v) for k, v in zip(gid, cnt)}
    out = {}
    for k, exp in base.items():
        it = iter(exp)
        out[k] = [X.Expect("value", counts.get(k, 0), None) if a in dist else next(it) for a in range(flat.n_aggs)]
    return out


def as_count(plan):
    """the plan with count(DISTINCT) read as count: how exact_ref.check compares its int64 results"""
    p = type(plan).from_buffer_copy(bytes(plan))
    for a in range(p.n_aggs):
        if p.aggs[a].fn == g.GX_AGG_COUNT_DISTINCT:
            p.aggs[a].fn = g.GX_AGG_COUNT
    return p


def check(plan, want, got, group_types=()):
    """got = fetch() output; raises AssertionError with the first difference"""
    X.check(as_count(plan), want, got, group_types)
