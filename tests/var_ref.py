"""Exact reference for the float8 variance aggregates (GX_AGG_VAR_POP_F8 .. GX_AGG_STDDEV_SAMP_F8).

Sxx, the sum of squared deviations from the group mean, is computed as an exact rational over the argument values as
float8 evaluates them (exact_ref.eval_arg: separately rounded + - *).  A device Sxx passes when

    |got - Sxx| <= 2^-30 Sxx + 16 N^2 2^-52 D^2,      D = max |x_i - mean|

the bar DESIGN.md §3.2 states: the first term covers the relative rounding of well-conditioned data, the second the
cancellation of shifted sums on data like 1e9 + noise.  A constant group has D = 0 and must give exactly 0.  The final
functions divide by N (pop) or N - 1 (samp) and take the square root for stddev (float.c:3010-3096); a group with an
infinite or NaN input gives NaN, N == 0 (pop) or N <= 1 (samp) NULL."""
import math
from fractions import Fraction

import numpy as np

import opentenbase_b200 as g
import exact_ref as X

VAR_FNS = (g.GX_AGG_VAR_POP_F8, g.GX_AGG_VAR_SAMP_F8, g.GX_AGG_STDDEV_POP_F8, g.GX_AGG_STDDEV_SAMP_F8)
POP = (g.GX_AGG_VAR_POP_F8, g.GX_AGG_STDDEV_POP_F8)
STDDEV = (g.GX_AGG_STDDEV_POP_F8, g.GX_AGG_STDDEV_SAMP_F8)


def sxx_exact(x):
    """exact sum of squared deviations of the finite float64 values x, as a Fraction"""
    x = np.asarray(x, np.float64)
    n = len(x)
    if n == 0:
        return Fraction(0)
    vals, cnt = np.unique(x, return_counts=True)
    m, e = np.frexp(vals)                                  # vals = m 2^e, 0.5 <= |m| < 1
    mi = (m * 2.0 ** 53).astype(np.int64)                 # exact: 53-bit integer mantissas
    e = e.astype(np.int64) - 53
    emin = int(e.min())
    big = mi.astype(object) * np.array([1 << int(s) for s in (e - emin)], dtype=object)
    c = cnt.astype(object)
    s1 = int((c * big).sum())
    s2 = int((c * big * big).sum())
    return Fraction(n * s2 - s1 * s1, n) * Fraction(2) ** (2 * emin)


def sxx_tol(x, sxx):
    x = np.asarray(x, np.float64)
    n = len(x)
    if n == 0:
        return 0.0
    mean = float(Fraction(math.fsum(x)) / n) if np.isfinite(x).all() else 0.0
    d = max(abs(float(x.max()) - mean), abs(float(x.min()) - mean))
    return 2.0 ** -30 * float(sxx) + 16.0 * n * n * 2.0 ** -52 * d * d


def expect(fn, x):
    """what fn over the group's non-NULL values x must give: ("null",), ("nan",) or ("value", V, tol)"""
    x = np.asarray(x, np.float64)
    n = len(x)
    if n == 0 or (fn not in POP and n <= 1):
        return ("null",)
    if not np.isfinite(x).all():
        return ("nan",)
    sxx = sxx_exact(x)
    div = n if fn in POP else n - 1
    return ("value", float(sxx / div), sxx_tol(x, sxx) / div)


def matches(fn, want, got, isnull):
    if want[0] == "null":
        return bool(isnull)
    if isnull:
        return False
    if want[0] == "nan":
        return math.isnan(got)
    v, tol = want[1], want[2]
    if math.isnan(got) or got < 0:
        return False
    if fn in STDDEV:
        # got = sqrt(V') rounded: compare got^2 with V, allowing for the two roundings
        return abs(got * got - v) <= tol + 2.0 ** -49 * v
    return abs(got - v) <= tol + 2.0 ** -51 * v


def sxx_matches(x, got):
    """a fetched Sxx (gx_result_fetch_sxx) against the exact one: NaN for a non-finite input, 0 for no input"""
    x = np.asarray(x, np.float64)
    if len(x) == 0:
        return got == 0.0
    if not np.isfinite(x).all():
        return math.isnan(got)
    sxx = sxx_exact(x)
    return got >= 0 and abs(got - float(sxx)) <= sxx_tol(x, sxx)


def group_values(plan, a, cols, nulls, keys, rows=None):
    """{group key: non-NULL argument values of aggregate a} over the selected rows (keys: one int64 per row, -1 for a
    NULL key is the caller's business)"""
    vals, vnull, _ = X.eval_arg([(o.op, o.col, o.k) for o in plan.aggs[a].arg.ops[:plan.aggs[a].arg.nops]], cols, nulls)
    rows = np.arange(len(cols[0])) if rows is None else np.asarray(rows)
    keep = rows[~vnull[rows]]
    out = {int(k): vals[rows[0:0]] for k in np.unique(np.asarray(keys)[rows])}
    if len(keep) == 0:
        return out
    k = np.asarray(keys)[keep]
    order = np.argsort(k, kind="stable")
    ks, vs = k[order], vals[keep][order]
    bounds = np.flatnonzero(np.diff(ks)) + 1
    for seg_k, seg_v in zip(np.split(ks, bounds), np.split(vs, bounds)):
        out[int(seg_k[0])] = seg_v
    return out


def check(plan, cols, nulls, keys, got, rows=None, group_key=lambda row_keys: row_keys[:, 0]):
    """every variance aggregate of the fetched result got = (keys, aggs, nulls) against the exact reference; the
    result's groups must be exactly the groups of the selected rows"""
    gk, ga, gn = got
    ng = plan.n_group_cols
    rk = group_key(gk) if ng else np.zeros(len(ga), np.int64)
    checked = 0
    for a in range(plan.n_aggs):
        fn = plan.aggs[a].fn
        if fn not in VAR_FNS:
            continue
        per = group_values(plan, a, cols, nulls, keys, rows)
        if ng:
            assert sorted(int(k) for k in rk) == sorted(per), "group keys differ"
        for i, k in enumerate(rk):
            x = per.get(int(k), np.zeros(0))
            want = expect(fn, x)
            assert matches(fn, want, float(ga[i, a]), gn[i, ng + a]), (a, fn, int(k), want, float(ga[i, a]), int(gn[i, ng + a]), len(x))
            checked += 1
    return checked
