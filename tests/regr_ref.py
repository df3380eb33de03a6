"""Exact reference for the SQL:2003 binary aggregates (GX_AGG_REGR_COUNT .. GX_AGG_CORR_F8) over (Y, X) pairs.

N, Sx, Sy, Sxx, Syy and Sxy of float8_regr_accum's state are computed as exact rationals over the argument values as
float8 evaluates them (exact_ref.eval_arg), over the pairs whose Y and X are both non-NULL.  A device value passes when

    |got - Sxx| <= 2^-30 Sxx + 16 N^2 2^-52 Dx^2                 (the variance bar, var_ref.sxx_tol; Syy alike)
    |got - Sxy| <= 2^-30 sqrt(Sxx Syy) + 16 N^2 2^-52 Dx Dy       (Cauchy-Schwarz: |Sxy| <= sqrt(Sxx Syy))

Dx, Dy the largest deviations from the means, and each final within the first-order propagation of those bars through
its formula (float.c:3386-3642) plus a few ulps.  A constant X (Y) has Dx = 0 (Dy = 0): Sxx (Syy) must be exactly 0,
so the vertical- and horizontal-line branches are taken exactly.  As float8_regr_accum does, a non-finite X makes
Sxx and Sxy NaN, a non-finite Y Syy and Sxy; Sx and Sy are ordinary sums."""
import math
from fractions import Fraction

import numpy as np

import opentenbase_b200 as g
import exact_ref as X

REGR_FNS = tuple(range(g.GX_AGG_REGR_COUNT, g.GX_AGG_CORR_F8 + 1))
EPS = 2.0 ** -52


def _scaled(v):
    """v = big * 2^e exactly: big an object array of Python ints, e the common exponent"""
    m, e = np.frexp(np.asarray(v, np.float64))
    mi = (m * 2.0 ** 53).astype(np.int64)
    e = e.astype(np.int64) - 53
    emin = int(e.min())
    return mi.astype(object) * np.array([1 << int(s) for s in (e - emin)], dtype=object), emin


def exact_sums(x, y):
    """{N, Sx, Sy, Sxx, Syy, Sxy} of finite float64 pairs as Fractions"""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    n = len(x)
    if n == 0:
        return {k: Fraction(0) for k in ("N", "Sx", "Sy", "Sxx", "Syy", "Sxy")}
    bx, ex = _scaled(x)
    by, ey = _scaled(y)
    sx, sy = int(bx.sum()), int(by.sum())
    sxx, syy, sxy = int((bx * bx).sum()), int((by * by).sum()), int((bx * by).sum())
    two = Fraction(2)
    return {"N": Fraction(n), "Sx": Fraction(sx) * two ** ex, "Sy": Fraction(sy) * two ** ey,
            "Sxx": Fraction(n * sxx - sx * sx, n) * two ** (2 * ex), "Syy": Fraction(n * syy - sy * sy, n) * two ** (2 * ey),
            "Sxy": Fraction(n * sxy - sx * sy, n) * two ** (ex + ey)}


def _dev(v):
    v = np.asarray(v, np.float64)
    if len(v) == 0:
        return 0.0
    mean = Fraction(math.fsum(v)) / len(v)
    return max(abs(float(Fraction(float(v.max())) - mean)), abs(float(Fraction(float(v.min())) - mean)))


def bars(x, y, s):
    """(bar of Sxx, of Syy, of Sxy, of Sx, of Sy) for finite pairs with exact sums s"""
    n = len(x)
    dx, dy = _dev(x), _dev(y)
    bxx = 2.0 ** -30 * float(s["Sxx"]) + 16.0 * n * n * EPS * dx * dx
    byy = 2.0 ** -30 * float(s["Syy"]) + 16.0 * n * n * EPS * dy * dy
    bxy = 2.0 ** -30 * math.sqrt(float(s["Sxx"]) * float(s["Syy"])) + 16.0 * n * n * EPS * dx * dy
    bsx = n * EPS * float(np.abs(x).sum())
    bsy = n * EPS * float(np.abs(y).sum())
    return bxx, byy, bxy, bsx, bsy


def state(x, y):
    """the expected six values {N, Sx, Sxx, Sy, Syy, Sxy} as (value, tol) pairs, NaN where float8_regr_accum has NaN"""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    n = len(x)
    if n == 0:
        return [(0.0, 0.0)] * 6
    fx, fy = np.isfinite(x).all(), np.isfinite(y).all()
    with np.errstate(all="ignore"):
        sx_nf, sy_nf = float(np.sum(x)), float(np.sum(y))
    # a non-finite side's exact sums are not used: its own values are NaN or the float sum
    xf, yf = np.where(np.isfinite(x), x, 0.0), np.where(np.isfinite(y), y, 0.0)
    s = exact_sums(xf, yf)
    bxx, byy, bxy, bsx, bsy = bars(xf, yf, s)
    nan = (math.nan, 0.0)
    sxv = (float(s["Sx"]), bsx) if fx else (sx_nf, 0.0)
    syv = (float(s["Sy"]), bsy) if fy else (sy_nf, 0.0)
    return [(float(n), 0.0), sxv, (float(s["Sxx"]), bxx) if fx else nan, syv, (float(s["Syy"]), byy) if fy else nan,
            (float(s["Sxy"]), bxy) if fx and fy else nan]


def expect(fn, x, y):
    """what fn over the group's pairs must give: ("null",), ("nan",), ("int", n) or ("value", V, tol, maybe_null)"""
    n = len(x)
    if fn == g.GX_AGG_REGR_COUNT:
        return ("int", n)
    if n < (2 if fn == g.GX_AGG_COVAR_SAMP_F8 else 1):
        return ("null",)
    st = state(x, y)
    (N, _), (Sx, tsx), (Sxx, txx), (Sy, tsy), (Syy, tyy), (Sxy, txy) = st
    ulp = 8 * EPS

    def val(v, tol, maybe_null=False):
        if math.isnan(v):
            return ("nan",)
        return ("value", v, tol + ulp * abs(v), maybe_null)

    # exact zero takes the reference's branch; a value within its bar of zero may take either
    zxx, zyy = Sxx == 0, Syy == 0
    nxx, nyy = (not zxx) and Sxx <= txx, (not zyy) and Syy <= tyy
    if fn == g.GX_AGG_REGR_SXX_F8:
        return val(Sxx, txx)
    if fn == g.GX_AGG_REGR_SYY_F8:
        return val(Syy, tyy)
    if fn == g.GX_AGG_REGR_SXY_F8:
        return val(Sxy, txy)
    if fn == g.GX_AGG_REGR_AVGX_F8:
        return ("value", Sx / N, tsx / N + ulp * abs(Sx / N), False) if math.isfinite(Sx) else ("nan",) if math.isnan(Sx) else ("value", Sx, 0.0, False)
    if fn == g.GX_AGG_REGR_AVGY_F8:
        return ("value", Sy / N, tsy / N + ulp * abs(Sy / N), False) if math.isfinite(Sy) else ("nan",) if math.isnan(Sy) else ("value", Sy, 0.0, False)
    if fn == g.GX_AGG_COVAR_POP_F8:
        return val(Sxy / N, txy / N)
    if fn == g.GX_AGG_COVAR_SAMP_F8:
        return val(Sxy / (N - 1), txy / (N - 1))
    if fn == g.GX_AGG_CORR_F8:
        if zxx or zyy:
            return ("null",)
        if math.isnan(Sxx) or math.isnan(Syy) or math.isnan(Sxy):
            return ("nan",)
        r = Sxy / math.sqrt(Sxx * Syy)
        return val(r, txy / math.sqrt(Sxx * Syy) + abs(r) * (txx / (2 * Sxx) + tyy / (2 * Syy)), nxx or nyy)
    if zxx:
        return ("null",)
    if math.isnan(Sxx) or math.isnan(Sxy):
        return ("nan",)
    slope = Sxy / Sxx
    tslope = txy / Sxx + abs(slope) * txx / Sxx
    if fn == g.GX_AGG_REGR_SLOPE_F8:
        return val(slope, tslope, nxx)
    if fn == g.GX_AGG_REGR_INTERCEPT_F8:
        if not (math.isfinite(Sx) and math.isfinite(Sy)):
            return ("nan",)
        v = (Sy - Sx * slope) / N
        return val(v, (tsy + abs(Sx) * tslope + abs(slope) * tsx + 4 * EPS * (abs(Sy) + abs(Sx * slope))) / N, nxx)
    # regr_r2
    if zyy:
        return ("value", 1.0, 0.0, nxx)
    if math.isnan(Syy):
        return ("nan",)
    r2 = (Sxy * Sxy) / (Sxx * Syy)
    return val(r2, 2 * abs(Sxy) * txy / (Sxx * Syy) + r2 * (txx / Sxx + tyy / Syy), nxx or nyy)


def matches(want, got, isnull):
    if want[0] == "null":
        return bool(isnull)
    if want[0] == "int":
        return not isnull and int(np.array([got], np.float64).view(np.int64)[0]) == want[1]
    if isnull:
        return len(want) > 3 and want[3]
    if want[0] == "nan":
        return math.isnan(got)
    v, tol = want[1], want[2]
    if math.isinf(v):
        return got == v
    return not math.isnan(got) and abs(got - v) <= tol


def state_matches(st_want, got6):
    """a fetched six-value state (gx_result_fetch_regr) against state()"""
    for (v, tol), gv in zip(st_want, got6):
        if math.isnan(v):
            if not math.isnan(gv):
                return False
        elif math.isinf(v):
            if gv != v:
                return False
        elif abs(gv - v) > tol + 8 * EPS * abs(v):
            return False
    return True


def split(ops):
    """Y's and X's programs of a two-argument aggregate's ops"""
    k = [o[0] for o in ops].index(g.GX_OP_ARG2)
    return ops[:k], ops[k + 1:]


def pair_values(plan, a, cols, nulls, keys, rows=None):
    """{group key: (y, x) of aggregate a's non-NULL pairs} over the selected rows"""
    ops = [(o.op, o.col, o.k) for o in plan.aggs[a].arg.ops[:plan.aggs[a].arg.nops]]
    oy, ox = split(ops)
    yv, yn, _ = X.eval_arg(oy, cols, nulls)
    xv, xn, _ = X.eval_arg(ox, cols, nulls)
    rows = np.arange(len(cols[0])) if rows is None else np.asarray(rows)
    keys = np.asarray(keys)
    out = {int(k): (np.zeros(0), np.zeros(0)) for k in np.unique(keys[rows])}
    keep = rows[~(yn[rows] | xn[rows])]
    if len(keep) == 0:
        return out
    k = keys[keep]
    order = np.argsort(k, kind="stable")
    ks, ys, xs = k[order], yv[keep][order], xv[keep][order]
    bounds = np.flatnonzero(np.diff(ks)) + 1
    for sk, sy, sx in zip(np.split(ks, bounds), np.split(ys, bounds), np.split(xs, bounds)):
        out[int(sk[0])] = (sy, sx)
    return out


def check(plan, cols, nulls, keys, got, rows=None, group_key=lambda row_keys: row_keys[:, 0]):
    """every regression aggregate of the fetched result got = (keys, aggs, nulls) against the exact reference; the
    result's groups must be exactly the groups of the selected rows.  Returns the number of values checked."""
    gk, ga, gn = got
    ng = plan.n_group_cols
    rk = group_key(gk) if ng else np.zeros(len(ga), np.int64)
    checked = 0
    per = None
    for a in range(plan.n_aggs):
        fn = plan.aggs[a].fn
        if fn not in REGR_FNS:
            continue
        per = pair_values(plan, a, cols, nulls, keys, rows) if per is None else per
        if ng:
            assert sorted(int(k) for k in rk) == sorted(per), "group keys differ"
        for i, k in enumerate(rk):
            y, x = per.get(int(k), (np.zeros(0), np.zeros(0)))
            want = expect(fn, x, y)
            assert matches(want, float(ga[i, a]), gn[i, ng + a]), (a, fn, int(k), want, float(ga[i, a]), int(gn[i, ng + a]), len(x))
            checked += 1
    return checked
