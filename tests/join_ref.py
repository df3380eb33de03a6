"""Exact hash-join reference in numpy, CPU only.

The build side is sorted once; every outer key finds its partners with searchsorted and the pairs are expanded with
repeat.  Semantics (nodeHashjoin.c's INNER / LEFT / SEMI / ANTI arms):

  - a NULL key never matches, on either side; INT64_MIN is an ordinary key value;
  - int4 / date keys are widened to int64 and compared by value, so mixed key widths join;
  - the outer and the build side's quals are applied first (a qual on a NULL fails);
  - LEFT keeps every outer row that passes its quals, an unmatched one once with a NULL inner side; SEMI keeps an
    outer row once if it has a partner; ANTI keeps it (NULL key included) if it has none.

Outputs: the multiset of output rows (`rows`, sorted, NULL as INT64_MIN as the oracle's exec_join reports it) and
per-group expectations of an aggregate over the join (`expect_groups`, through tests/exact_ref.py)."""
import numpy as np

import opentenbase_b200 as g
import exact_ref as X
import qual_ref as Q

NULL = np.iinfo(np.int64).min


def quals(cols, nulls, preds, n):
    """rows passing every qual (col, op, const[, is_float]) under tests/qual_ref.py's semantics: a NULL fails, float8
    compares as float8_cmp (NaN last), an int8 numpy column is "char" and compares as uint8"""
    return Q.quals(cols, nulls, preds, n)


def _key(v, nl):
    v = np.asarray(v).astype(np.int64)                  # int4 / date widened: compared by value
    nl = np.zeros(len(v), bool) if nl is None else np.asarray(nl).astype(bool)
    return v, nl


def join(jt, okey, ikey, onull=None, inull=None, okeep=None, ikeep=None):
    """(outer row, inner row) of every output row of join type jt; inner row -1 = the NULL inner side (LEFT), or
    no inner side at all (SEMI / ANTI).  okeep / ikeep: rows that passed the quals."""
    ov, on = _key(okey, onull)
    iv, inn = _key(ikey, inull)
    okeep = np.ones(len(ov), bool) if okeep is None else np.asarray(okeep, bool)
    ikeep = np.ones(len(iv), bool) if ikeep is None else np.asarray(ikeep, bool)
    irows = np.flatnonzero(ikeep & ~inn)
    order = np.argsort(iv[irows], kind="stable")
    skeys, srows = iv[irows][order], irows[order]
    scanned = np.flatnonzero(okeep)
    probing = scanned[~on[scanned]]
    lo = np.searchsorted(skeys, ov[probing], "left")
    cnt = np.searchsorted(skeys, ov[probing], "right") - lo
    matched = np.zeros(len(ov), bool)
    matched[probing[cnt > 0]] = True
    if jt == g.GX_JOIN_SEMI:
        o = np.flatnonzero(matched)
        return o, np.full(len(o), -1, np.int64)
    if jt == g.GX_JOIN_ANTI:
        o = scanned[~matched[scanned]]
        return o, np.full(len(o), -1, np.int64)
    o = np.repeat(probing, cnt)
    first = np.repeat(lo - (np.cumsum(cnt) - cnt), cnt)
    i = srows[first + np.arange(len(o))] if len(o) else np.zeros(0, np.int64)
    if jt == g.GX_JOIN_LEFT:
        miss = scanned[~matched[scanned]]
        o, i = np.concatenate([o, miss]), np.concatenate([i, np.full(len(miss), -1, np.int64)])
    else:
        assert jt == g.GX_JOIN_INNER, jt
    return o, i.astype(np.int64)


def _gather(v, nl, rows):
    out = np.full(len(rows), NULL, np.int64)
    ok = rows >= 0
    out[ok] = np.asarray(v)[rows[ok]].astype(np.int64)
    if nl is not None:
        out[ok & (np.asarray(nl)[np.maximum(rows, 0)] != 0)] = NULL
    return out


def rows(pairs, out_cols, inner_cols=(), out_nulls=None):
    """the output rows of (outer, inner) pairs as an int64 array [row, column], lexicographically sorted:
    the outer columns out_cols, then the inner columns (NULL where the inner row is -1)"""
    o, i = pairs
    out_nulls = out_nulls or [None] * len(out_cols)
    cols = [_gather(c, nl, o) for c, nl in zip(out_cols, out_nulls)] + [_gather(c, None, i) for c in inner_cols]
    if not cols:
        return np.zeros((len(o), 0), np.int64)
    w = np.stack(cols, 1)
    return w[np.lexsort(w.T[::-1])] if len(w) else w


def expect_groups(plan, pairs, outer_cols, outer_types, payload_cols, payload_types, outer_nulls=None):
    """exact_ref.expect_groups over the rows of an (INNER) join: aggregates read outer columns, group columns are
    (0, outer column) or (1, payload index) and must be integer columns.  Groups are found with np.unique."""
    o, i = pairs
    no = len(outer_cols)
    cols = [np.asarray(c)[o] for c in outer_cols] + [np.asarray(c)[i] for c in payload_cols]
    nulls = [None if outer_nulls is None or outer_nulls[c] is None else np.asarray(outer_nulls[c])[o] for c in range(no)]
    nulls += [None] * len(payload_cols)
    types = list(outer_types) + list(payload_types)
    flat = type(plan).from_buffer_copy(bytes(plan))             # the same plan over the joined columns
    for c in range(plan.n_group_cols):
        side, col = plan.group_cols[c].side, plan.group_cols[c].col
        flat.group_cols[c].side, flat.group_cols[c].col = 0, col + (no if side == 1 else 0)
    gcols = [flat.group_cols[c].col for c in range(plan.n_group_cols)]
    assert all(types[c] != g.GX_FLOAT8 for c in gcols), "integer group columns only"
    keep = quals(cols, nulls, [(plan.preds[p].col, plan.preds[p].op, plan.preds[p].fval if types[plan.preds[p].col] == g.GX_FLOAT8
                                else plan.preds[p].ival) for p in range(plan.n_preds)], len(o))
    if not gcols:
        return X.expect_groups(flat, cols, nulls=nulls, types=types, keep=keep)
    parts = []
    for c in gcols:
        nl = np.zeros(len(o), bool) if nulls[c] is None else nulls[c].astype(bool)
        parts += [nl.astype(np.int64), np.where(nl, 0, cols[c].astype(np.int64))]
    mat = np.stack(parts, 1) if len(o) else np.zeros((0, 2 * len(gcols)), np.int64)
    uniq, gi = np.unique(mat, axis=0, return_inverse=True)
    gkeys = [tuple(None if u[2 * j] else int(u[2 * j + 1]) for j in range(len(gcols))) for u in uniq]
    return X.expect_groups(flat, cols, nulls=nulls, types=types, keep=keep, gindex=np.asarray(gi).reshape(-1), gkeys=gkeys)
