"""Exact reference for grouped float8 aggregates, CPU only.

The oracle restates the reference's executor and so sums in ITS scan order; a GPU kernel sums in another
order.  This module instead computes what any summation order must land near: the exact sum (math.fsum,
Fractions where fsum itself overflows), min/max under float8_cmp (NaN sorts last), and the reference's result
class -- a value, NULL, or GX_ERR_OVERFLOW -- under the float8pl / float8mi / float8mul / float8_accum rules
(utils/adt/float.c, CHECKFLOATVAL):

  - an infinite input may give an infinite result; +inf + -inf is NaN;
  - finite operands must not give an infinite result, nor (float8mul) a zero from non-zero factors;
  - float8_accum also errors when Sxx, the sum of squared deviations, goes infinite from finite inputs.

Cases whose outcome in the reference depends on the scan order (a finite sum whose partial sums may or may not
overflow, min/max over both signs of zero) are not given an error class; the test data avoids them.

A float8 SUM is compared within |got - exact| <= 1.01 (n-1) 2^-53 sum|x_i| + n 2^-1074, the first-order worst
case of any summation order (atomics included); NaN, infinities and the sign of a zero bit for bit."""
import math
from fractions import Fraction

import numpy as np

import opentenbase_b200 as g

EPS = 2.0 ** -53
TINY = 2.0 ** -1074
NEG_ZERO_BITS = np.int64(-0x8000000000000000)


class Expect:
    """kind: "value" | "null" | "overflow".  tol None = bit for bit (NaN payloads canonicalised), else the
    absolute bound; zero_sign: the sign a zero result must carry (None = either)."""

    def __init__(self, kind, value=0.0, tol=None, zero_sign=None):
        self.kind, self.value, self.tol, self.zero_sign = kind, value, tol, zero_sign

    def __repr__(self):
        return f"Expect({self.kind}, {self.value!r}, tol={self.tol}, zero_sign={self.zero_sign})"

    def matches(self, got, isnull):
        if self.kind == "null":
            return bool(isnull)
        if isnull or self.kind != "value":
            return False
        if math.isnan(self.value) or math.isinf(self.value):
            return (math.isnan(got) and math.isnan(self.value)) or got == self.value
        if math.isnan(got) or math.isinf(got):
            return False
        if got == 0.0 and self.zero_sign is not None and math.copysign(1.0, got) != self.zero_sign:
            return False
        if self.tol is None:
            return got == self.value and math.copysign(1.0, got) == math.copysign(1.0, self.value)
        return abs(got - self.value) <= self.tol


def eval_arg(ops, cols, nulls=None):
    """The plan's postfix argument program [(op, col, k)] evaluated left to right with separately rounded
    + - * (no FMA), as float8pl / float8mi / float8mul do.  Returns (values, null, error) per row; error marks
    rows where a finite operation overflowed or (mul) underflowed to zero."""
    n = len(cols[0])
    st = []
    with np.errstate(all="ignore"):
        for op, col, k in ops:
            if op == g.GX_OP_COL:
                nl = np.zeros(n, bool) if nulls is None or nulls[col] is None else np.asarray(nulls[col]).astype(bool)
                st.append((np.asarray(cols[col]).astype(np.float64), nl, np.zeros(n, bool)))
            elif op == g.GX_OP_CONST:
                st.append((np.full(n, float(k)), np.zeros(n, bool), np.zeros(n, bool)))
            else:
                (b, bn, be), (a, an, ae) = st.pop(), st.pop()
                r = a + b if op == g.GX_OP_ADD else a - b if op == g.GX_OP_SUB else a * b
                nl = an | bn
                bad = np.isinf(r) & ~np.isinf(a) & ~np.isinf(b)
                if op == g.GX_OP_MUL:
                    bad |= (r == 0) & (a != 0) & (b != 0)
                st.append((r, nl, (ae | be | bad) & ~nl))
    assert len(st) == 1
    return st[0]


def _exact_sum(x):
    """(exact sum as a float or None on overflow, sum of |x|)"""
    try:
        s = math.fsum(x)
    except OverflowError:
        s = None
    if s is None or math.isinf(s):
        try:
            s = float(sum(Fraction(v) for v in x))
        except OverflowError:
            return None, math.inf
    try:
        a = math.fsum(abs(v) for v in x)
    except OverflowError:
        a = math.inf
    return s, a


def _special_sum(x):
    """NaN / infinite inputs decide the sum alone; None when all inputs are finite"""
    if np.isnan(x).any():
        return math.nan
    pinf, ninf = bool((x == np.inf).any()), bool((x == -np.inf).any())
    if pinf and ninf:
        return math.nan
    if pinf or ninf:
        return math.inf if pinf else -math.inf
    return None


def expect_sum(x, avg=False):
    x = np.asarray(x, np.float64)
    n = len(x)
    if n == 0:
        return Expect("null")
    sp = _special_sum(x)
    if sp is not None:
        return Expect("value", sp)                              # inf / N and NaN / N keep their class
    if not avg and (x == 0).all() and np.signbit(x).all():
        return Expect("value", -0.0)                            # the first input is the state: -0 + -0 = -0
    s, a = _exact_sum(x.tolist())
    if s is None:
        return Expect("overflow")
    bound = 1.01 * max(n - 1, 0) * EPS * a + n * TINY
    if not avg:
        return Expect("value", s, bound, zero_sign=1.0 if s == 0 else None)
    # float8_accum: Sxx = sum of squared deviations, an error when it goes infinite from finite inputs
    mean = Fraction(sum(Fraction(v) for v in x.tolist())) / n
    sxx = sum((Fraction(v) - mean) ** 2 for v in x.tolist())
    if sxx > Fraction(np.finfo(np.float64).max):
        return Expect("overflow")
    v = s / n
    return Expect("value", v, bound / n + EPS * abs(v) + TINY, zero_sign=1.0 if v == 0 else None)


def expect_minmax(x, want_max):
    x = np.asarray(x, np.float64)
    if len(x) == 0:
        return Expect("null")
    nan = np.isnan(x)
    if want_max and nan.any():
        return Expect("value", math.nan)
    if nan.all():
        return Expect("value", math.nan)
    y = x[~nan]
    v = float(y.max() if want_max else y.min())
    zs = None
    if v == 0:
        z = y[y == 0]
        signs = set(np.signbit(z).tolist())
        zs = (-1.0 if True in signs else 1.0) if len(signs) == 1 else None
    return Expect("value", v, 0.0 if zs is None else None, zero_sign=zs)


def canonical_key(types, values, nulls):
    """group key of one row as the reference's hash aggregate sees it: float8 +-0 fold, NaN keeps its bits"""
    out = []
    for t, v, nl in zip(types, values, nulls):
        if nl:
            out.append(None)
        elif t == g.GX_FLOAT8:
            b = np.float64(v).view(np.int64)
            out.append(0 if b == NEG_ZERO_BITS else int(b))
        else:
            out.append(int(v))
    return tuple(out)


def expect_groups(plan, cols, nulls=None, types=None, keep=None, gindex=None, gkeys=None):
    """Per group of a plan without a join: {key tuple: [Expect per aggregate]}, or "overflow" when the whole
    query errors (an expression overflow anywhere, or an aggregate state out of range in any group).
    keep: rows that pass the plan's quals (the caller evaluates them).  gindex/gkeys: the group of every row
    (an int array) and the key tuple of every group, when the caller already knows them (large inputs)."""
    n = len(cols[0])
    nulls = nulls or [None] * len(cols)
    keep = np.ones(n, bool) if keep is None else np.asarray(keep, bool)
    gcols = [plan.group_cols[c].col for c in range(plan.n_group_cols)]
    groups = {}
    if gindex is not None:
        rows = np.flatnonzero(keep)
        gi = np.asarray(gindex)[rows]
        order = np.argsort(gi, kind="stable")
        bounds = np.flatnonzero(np.diff(gi[order])) + 1
        for part in np.split(rows[order], bounds):
            if len(part):
                groups[gkeys[int(gindex[part[0]])]] = part
    elif gcols:
        kv = [np.asarray(cols[c]) for c in gcols]
        kn = [np.zeros(n, bool) if nulls[c] is None else np.asarray(nulls[c]).astype(bool) for c in gcols]
        kt = [types[c] for c in gcols]
        for i in np.flatnonzero(keep).tolist():
            groups.setdefault(canonical_key(kt, [v[i] for v in kv], [m[i] for m in kn]), []).append(i)
    else:
        groups = {(): np.flatnonzero(keep)}
    if not gcols and not groups:
        groups[()] = []
    out = {k: [] for k in groups}
    for a in range(plan.n_aggs):
        fn = plan.aggs[a].fn
        ops = [(plan.aggs[a].arg.ops[j].op, plan.aggs[a].arg.ops[j].col, plan.aggs[a].arg.ops[j].k)
               for j in range(plan.aggs[a].arg.nops)]
        if fn == g.GX_AGG_COUNT_STAR:
            for k, r in groups.items():
                out[k].append(Expect("value", len(r), None))
            continue
        if fn in (g.GX_AGG_COUNT, g.GX_AGG_SUM_I4, g.GX_AGG_SUM_I8):
            c = ops[0][1]
            nl = np.zeros(n, bool) if nulls[c] is None else np.asarray(nulls[c]).astype(bool)
            for k, r in groups.items():
                r = np.asarray(r, np.int64)
                r = r[~nl[r]]
                if fn == g.GX_AGG_COUNT:
                    out[k].append(Expect("value", len(r), None))
                elif len(r) == 0:
                    out[k].append(Expect("null"))
                else:
                    s = sum(int(v) for v in np.asarray(cols[c])[r].tolist())
                    if not -2**63 <= s < 2**63:
                        return "overflow"
                    out[k].append(Expect("value", s, None))
            continue
        v, nl, err = eval_arg(ops, cols, nulls)
        if (err & keep).any():
            return "overflow"
        for k, r in groups.items():
            r = np.asarray(r, np.int64)
            x = v[r[~nl[r]]]
            if fn == g.GX_AGG_SUM_F8:
                e = expect_sum(x)
            elif fn == g.GX_AGG_AVG_F8:
                e = expect_sum(x, avg=True)
            else:
                e = expect_minmax(x, fn == g.GX_AGG_MAX_F8)
            if e.kind == "overflow":
                return "overflow"
            out[k].append(e)
    return out


def result_keys(plan, types_of_group_cols, keys, nulls):
    """fetch()-format keys -> the canonical key tuples of expect_groups"""
    ng = plan.n_group_cols
    f8 = [c < len(types_of_group_cols) and types_of_group_cols[c] == g.GX_FLOAT8 for c in range(ng)]

    def one(i, c):
        if nulls[i, c]:
            return None
        v = int(keys[i, c])
        return 0 if f8[c] and v == int(NEG_ZERO_BITS) else v        # the reference keeps the first row's zero
    return [tuple(one(i, c) for c in range(ng)) for i in range(keys.shape[0])]


def check(plan, want, got, group_types=()):
    """got = fetch() output (keys, aggs, nulls); raises AssertionError with the first difference"""
    keys, aggs, nulls = got
    assert want != "overflow", "the reference errors, the result did not"
    ng = plan.n_group_cols
    gk = result_keys(plan, group_types, keys, nulls)
    assert len(gk) == len(set(gk)), "a group appears twice"
    assert set(gk) == set(want), f"group keys differ: {len(gk)} vs {len(want)}; extra {sorted(set(gk) - set(want), key=str)[:5]}, missing {sorted(set(want) - set(gk), key=str)[:5]}"
    for i, k in enumerate(gk):
        for a, e in enumerate(want[k]):
            fn = plan.aggs[a].fn
            isnull = bool(nulls[i, ng + a])
            if fn in (g.GX_AGG_COUNT_STAR, g.GX_AGG_COUNT, g.GX_AGG_SUM_I4, g.GX_AGG_SUM_I8):
                ok = (e.kind == "null" and isnull) or (e.kind == "value" and not isnull and int(aggs[i:i + 1, a].view(np.int64)[0]) == e.value)
                got_v = int(aggs[i:i + 1, a].view(np.int64)[0])
            else:
                got_v = float(aggs[i, a])
                ok = e.matches(got_v, isnull)
            assert ok, f"group {k}, aggregate {a} (fn {fn}): got {got_v!r} (null={isnull}), want {e}"
