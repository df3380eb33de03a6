"""tests/regr_ref.py, the exact reference of the SQL:2003 binary aggregates, checked on the CPU:

- its exact sums against plain Fraction sums over the pairs;
- the device's shifted sums and their re-centring merge with the cross term, restated in numpy, against it over
  random splits;
- the reference's own float8_regr_accum / float8_regr_combine and twelve final objects (oracle/_ref/libotbref.so,
  called through the fmgr interface) against the formulas this module expects, the NULL, 1.0 and NaN branches included;
- the reference's Youngs-Cramer state missing the bar on 1e9 + U(0,1), which is why the device keeps shifted sums."""
import ctypes as C
import math
import os
from fractions import Fraction

import numpy as np
import pytest

import opentenbase_b200 as g
import regr_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_PATH = os.path.join(ROOT, "oracle", "_ref", "libotbref.so")
HAVE_REF = os.path.exists(REF_PATH)
F8OID = 701
FINALS = {g.GX_AGG_REGR_SXX_F8: "float8_regr_sxx", g.GX_AGG_REGR_SYY_F8: "float8_regr_syy", g.GX_AGG_REGR_SXY_F8: "float8_regr_sxy",
          g.GX_AGG_REGR_AVGX_F8: "float8_regr_avgx", g.GX_AGG_REGR_AVGY_F8: "float8_regr_avgy", g.GX_AGG_REGR_R2_F8: "float8_regr_r2",
          g.GX_AGG_REGR_SLOPE_F8: "float8_regr_slope", g.GX_AGG_REGR_INTERCEPT_F8: "float8_regr_intercept",
          g.GX_AGG_COVAR_POP_F8: "float8_covar_pop", g.GX_AGG_COVAR_SAMP_F8: "float8_covar_samp", g.GX_AGG_CORR_F8: "float8_corr"}


def datasets():
    rng = np.random.default_rng(0)
    x = rng.standard_normal(3000) * 100.0
    return {
        "normal": (x * 0.5 + rng.standard_normal(3000), x),
        "offset": (1e9 + rng.random(3000), 1e9 + rng.random(3000)),
        "const_x": (rng.random(200), np.full(200, 7.25)),
        "const_y": (np.full(200, -3.0), rng.random(200)),
        "two": (np.array([1.0, 3.0]), np.array([2.0, 5.0])),
        "one": (np.array([3.5]), np.array([1.0])),
        "zeros": (np.array([-0.0, 0.0, -0.0]), np.array([0.0, -0.0, 1.0])),
        "ints": (rng.integers(-10**6, 10**6, 5000).astype(np.float64), rng.integers(-10**3, 10**3, 5000).astype(np.float64)),
        "anti": (-np.arange(100.0), np.arange(100.0)),
    }


@pytest.mark.parametrize("name", list(datasets()))
def test_exact_sums_are_the_fraction_sums(name):
    y, x = datasets()[name]
    fx, fy = [Fraction(float(v)) for v in x], [Fraction(float(v)) for v in y]
    n = len(fx)
    mx, my = sum(fx) / n, sum(fy) / n
    s = R.exact_sums(x, y)
    assert s["N"] == n and s["Sx"] == sum(fx) and s["Sy"] == sum(fy)
    assert s["Sxx"] == sum((a - mx) ** 2 for a in fx) and s["Syy"] == sum((b - my) ** 2 for b in fy)
    assert s["Sxy"] == sum((a - mx) * (b - my) for a, b in zip(fx, fy))


def test_constant_sides_are_exact_zero():
    y, x = datasets()["const_x"]
    st = R.state(x, y)
    assert st[2] == (0.0, 0.0) and st[5][0] == 0.0
    assert R.expect(g.GX_AGG_REGR_SLOPE_F8, x, y) == ("null",) and R.expect(g.GX_AGG_CORR_F8, x, y) == ("null",)
    y, x = datasets()["const_y"]
    assert R.expect(g.GX_AGG_REGR_R2_F8, x, y)[:2] == ("value", 1.0) and R.expect(g.GX_AGG_CORR_F8, x, y) == ("null",)
    assert R.expect(g.GX_AGG_REGR_SLOPE_F8, x, y)[:2] == ("value", 0.0)


def test_expectations_at_the_edges():
    e = np.zeros(0)
    assert R.expect(g.GX_AGG_REGR_COUNT, e, e) == ("int", 0)
    assert R.expect(g.GX_AGG_CORR_F8, e, e) == ("null",)
    assert R.expect(g.GX_AGG_COVAR_SAMP_F8, np.ones(1), np.ones(1)) == ("null",)
    assert R.expect(g.GX_AGG_COVAR_POP_F8, np.ones(1), np.ones(1))[:2] == ("value", 0.0)
    x, y = np.array([1.0, np.inf, 2.0]), np.array([1.0, 2.0, 4.0])
    assert R.expect(g.GX_AGG_REGR_SXX_F8, x, y) == ("nan",) and R.expect(g.GX_AGG_REGR_SYY_F8, x, y)[0] == "value"
    assert R.expect(g.GX_AGG_REGR_AVGX_F8, x, y)[:2] == ("value", np.inf) and R.expect(g.GX_AGG_REGR_SLOPE_F8, x, y) == ("nan",)
    assert R.expect(g.GX_AGG_REGR_SXY_F8, y, x) == ("nan",) and R.expect(g.GX_AGG_REGR_SXX_F8, y, x)[0] == "value"


# ---------------------------------------------------------------- the device's shifted sums and their merge
def shifted(x, y):
    """one partial state as a sink builds it: shifts at the first pair, then {Sx, Sy, Cx, S1x, S2x, Cy, S1y, S2y, Sxy'}"""
    cx, cy = x[0], y[0]
    st = [0.0] * 9
    st[2], st[5] = cx, cy
    for a, b in zip(x, y):
        dx, dy = a - cx, b - cy
        st[0] += a; st[1] += b
        st[3] += dx; st[4] += dx * dx; st[6] += dy; st[7] += dy * dy; st[8] += dx * dy
    return st, len(x)


def merge(t, nt, s, ns):
    """regr_merge / regr_combine: s re-centred on t's shifts"""
    if ns == 0:
        return t, nt
    if nt == 0:
        return list(s), ns
    dx, dy = s[2] - t[2], s[5] - t[5]
    o = list(t)
    o[0] += s[0]; o[1] += s[1]
    o[8] = t[8] + (((s[8] + dx * s[6]) + dy * s[3]) + (ns * dx) * dy)
    o[3] = t[3] + (s[3] + ns * dx); o[4] = t[4] + ((s[4] + (2.0 * dx) * s[3]) + (ns * dx) * dx)
    o[6] = t[6] + (s[6] + ns * dy); o[7] = t[7] + ((s[7] + (2.0 * dy) * s[6]) + (ns * dy) * dy)
    return o, nt + ns


def finish(st, n):
    """regr_state: {N, Sx, Sxx, Sy, Syy, Sxy}"""
    sxx = max(0.0, st[4] - st[3] * (st[3] / n))
    syy = max(0.0, st[7] - st[6] * (st[6] / n))
    return [n, st[0], sxx, st[1], syy, st[8] - st[3] * (st[6] / n)]


@pytest.mark.parametrize("name", ["normal", "offset", "const_x", "const_y", "two", "ints", "anti"])
def test_recentring_merge_over_random_splits(name):
    y, x = datasets()[name]
    rng = np.random.default_rng(len(x))
    want = R.state(x, y)
    for _ in range(5):
        p = rng.permutation(len(x))
        xs, ys = x[p], y[p]
        cuts = np.sort(rng.choice(np.arange(1, len(x)), size=min(len(x) - 1, 7), replace=False)) if len(x) > 1 else []
        acc, n = [0.0] * 9, 0
        for px, py in zip(np.split(xs, cuts), np.split(ys, cuts)):
            if len(px):
                acc, n = merge(acc, n, *shifted(list(px), list(py)))
        got = finish(acc, n)
        assert R.state_matches(want, got), (name, got, want)
        if want[2][0] == 0.0:
            assert got[2] == 0.0 and got[5] == 0.0
        if want[4][0] == 0.0:
            assert got[4] == 0.0 and got[5] == 0.0


# ---------------------------------------------------------------- the reference's own objects
class FcInfo(C.Structure):                 # FunctionCallInfoData (fmgr.h), FUNC_MAX_ARGS = 100
    _fields_ = [("flinfo", C.c_void_p), ("context", C.c_void_p), ("resultinfo", C.c_void_p), ("fncollation", C.c_uint32),
                ("isnull", C.c_bool), ("nargs", C.c_short), ("arg", C.c_uint64 * 100), ("argnull", C.c_bool * 100)]


def f8_array6(v):
    """a one-dimensional float8[6] ArrayType: 4-byte varlena header, ndim, dataoffset 0, elemtype, dims, lbounds, data"""
    buf = (C.c_char * 72)()
    C.memmove(buf, np.array([72 << 2, 1, 0, F8OID, 6, 1], np.int32).tobytes(), 24)
    C.memmove(C.byref(buf, 24), np.asarray(v, np.float64).tobytes(), 48)
    return buf


def bits(d):
    return int(np.array([d], np.float64).view(np.uint64)[0])


class Ref:
    def __init__(self):
        self.L = C.CDLL(REF_PATH)

    def call(self, name, *args):
        f = getattr(self.L, name)
        f.restype = C.c_uint64
        f.argtypes = [C.c_void_p]
        fc = FcInfo()
        fc.nargs = len(args)
        for i, a in enumerate(args):
            fc.arg[i] = a
        d = f(C.byref(fc))
        return None if fc.isnull else float(np.array([d], np.uint64).view(np.float64)[0])

    def accum(self, x, y):
        """float8_regr_accum over the pairs, in order (it modifies its state in place inside an aggregate)"""
        a = f8_array6([0.0] * 6)
        for xv, yv in zip(x, y):
            self.call("float8_regr_accum", C.addressof(a), bits(float(yv)), bits(float(xv)))
        return np.frombuffer(bytes(a)[24:72], np.float64).copy()

    def combine(self, s1, s2):
        a, b = f8_array6(s1), f8_array6(s2)
        self.call("float8_regr_combine", C.addressof(a), C.addressof(b))
        return np.frombuffer(bytes(a)[24:72], np.float64).copy()

    def final(self, fn, st):
        a = f8_array6(st)
        return self.call(FINALS[fn], C.addressof(a))


needs_ref = pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref/libotbref.so is built only where the reference sources are present")


@needs_ref
def test_finals_match_the_reference_objects():
    """the module's expectation of every final, computed from the exact state, against the reference's own final
    function over the same exact state"""
    ref = Ref()
    for name, (y, x) in datasets().items():
        st = [float(v) for v, _ in R.state(x, y)]
        for fn, fname in FINALS.items():
            want = R.expect(fn, x, y)
            got = ref.final(fn, st)
            if got is None:
                assert want == ("null",) or (len(want) > 3 and want[3]), (name, fname, want)
            else:
                assert R.matches(want, got, 0), (name, fname, want, got)
    assert ref.final(g.GX_AGG_CORR_F8, [0.0] * 6) is None
    assert ref.final(g.GX_AGG_COVAR_SAMP_F8, [1.0, 1.0, 0.0, 1.0, 0.0, 0.0]) is None
    assert ref.final(g.GX_AGG_REGR_R2_F8, [3.0, 3.0, 2.0, 6.0, 0.0, 0.0]) == 1.0
    assert ref.final(g.GX_AGG_REGR_SLOPE_F8, [3.0, 3.0, 0.0, 6.0, 2.0, 0.0]) is None
    assert math.isnan(ref.final(g.GX_AGG_CORR_F8, [3.0, 3.0, math.nan, 6.0, 2.0, math.nan]))


@needs_ref
def test_accum_nan_rules_match_the_module():
    """float8_regr_accum: a non-finite X makes Sxx and Sxy NaN, a non-finite Y Syy and Sxy, the sums stay sums; the
    inf - (-inf) cross case included"""
    ref = Ref()
    cases = [([1.0, np.inf, 2.0], [1.0, 2.0, 4.0]), ([1.0, 2.0, 4.0], [1.0, -np.inf, 2.0]), ([np.inf, 1.0], [-np.inf, 2.0]),
             ([1.0, np.nan], [2.0, 3.0]), ([np.inf], [1.0]), ([2.0, 3.0, -np.inf], [np.inf, 1.0, 2.0])]
    for x, y in cases:
        got = ref.accum(x, y)
        want = R.state(np.array(x), np.array(y))
        for k in (2, 4, 5):
            assert math.isnan(got[k]) == math.isnan(want[k][0]), (x, y, k, got, want)
        assert got[0] == want[0][0]
        for k in (1, 3):
            assert (got[k] == want[k][0]) or (math.isnan(got[k]) and math.isnan(want[k][0])), (x, y, k, got, want)


@needs_ref
def test_reference_combine_of_two_exact_halves():
    ref = Ref()
    y, x = datasets()["normal"]
    h = len(x) // 2
    s = ref.combine([float(v) for v, _ in R.state(x[:h], y[:h])], [float(v) for v, _ in R.state(x[h:], y[h:])])
    assert R.state_matches(R.state(x, y), s)


@needs_ref
def test_youngs_cramer_misses_the_bar_far_from_zero():
    """on 1e9 + U(0,1) the reference's own accumulation is off by far more than the bar the device meets"""
    ref = Ref()
    y, x = datasets()["offset"]
    got = ref.accum(x, y)
    want = R.state(x, y)
    assert got[0] == len(x)
    assert abs(got[2] - want[2][0]) > 10 * want[2][1] or abs(got[5] - want[5][0]) > 10 * want[5][1], (got, want)
