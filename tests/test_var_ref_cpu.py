"""tests/var_ref.py, the exact reference of the float8 variance aggregates, checked on the CPU:

- its exact Sxx against a plain Fraction sum over the values;
- its final functions against the reference's own float8_var_pop / _var_samp / _stddev_pop / _stddev_samp objects
  (oracle/_ref/libotbref.so, called through the fmgr interface);
- the Youngs-Cramer Sxx the oracle keeps in its float8_accum state against it, within the bar of DESIGN.md §3.2;
- the device's re-centring merge of shifted sums, restated in numpy, against it over random splits."""
import ctypes as C
import math
import os
from fractions import Fraction

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import var_ref as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_PATH = os.path.join(ROOT, "oracle", "_ref", "libotbref.so")
HAVE_REF = os.path.exists(REF_PATH)
F8OID = 701


def datasets():
    rng = np.random.default_rng(0)
    return {
        "normal": rng.standard_normal(3000) * 100.0,
        "offset": 1e9 + rng.random(3000),
        "constant": np.full(500, 7.25),
        "two": np.array([1.0, 2.0]),
        "one": np.array([3.5]),
        "zeros": np.array([-0.0, 0.0, -0.0]),
        "wide": np.concatenate([rng.random(100) * 1e-300, rng.random(100) * 1e150]),
        "ints": rng.integers(-10**6, 10**6, 5000).astype(np.float64),
    }


@pytest.mark.parametrize("name", list(datasets()))
def test_exact_sxx_is_the_fraction_sum(name):
    x = datasets()[name]
    fr = [Fraction(float(v)) for v in x]
    mean = sum(fr) / len(fr)
    assert V.sxx_exact(x) == sum((v - mean) ** 2 for v in fr)


def test_constant_groups_have_no_tolerance():
    x = np.full(1000, 1e9 + 0.5)
    assert V.sxx_exact(x) == 0 and V.sxx_tol(x, V.sxx_exact(x)) == 0.0
    assert V.matches(g.GX_AGG_VAR_SAMP_F8, V.expect(g.GX_AGG_VAR_SAMP_F8, x), 0.0, 0)
    assert not V.matches(g.GX_AGG_VAR_SAMP_F8, V.expect(g.GX_AGG_VAR_SAMP_F8, x), 1e-300, 0)


def test_expectations_at_the_edges():
    assert V.expect(g.GX_AGG_VAR_POP_F8, []) == ("null",)
    assert V.expect(g.GX_AGG_VAR_SAMP_F8, [1.0]) == ("null",)
    assert V.expect(g.GX_AGG_VAR_POP_F8, [1.0])[:2] == ("value", 0.0)
    assert V.expect(g.GX_AGG_STDDEV_SAMP_F8, [1.0, np.inf]) == ("nan",)
    assert V.expect(g.GX_AGG_STDDEV_POP_F8, [np.nan]) == ("nan",)


# ---------------------------------------------------------------- the reference's final functions
class FcInfo(C.Structure):                 # FunctionCallInfoData (fmgr.h), FUNC_MAX_ARGS = 100
    _fields_ = [("flinfo", C.c_void_p), ("context", C.c_void_p), ("resultinfo", C.c_void_p), ("fncollation", C.c_uint32),
                ("isnull", C.c_bool), ("nargs", C.c_short), ("arg", C.c_uint64 * 100), ("argnull", C.c_bool * 100)]


def f8_array3(v):
    """a one-dimensional float8[3] ArrayType: 4-byte varlena header, ndim, dataoffset 0, elemtype, dims, lbounds, data"""
    buf = (C.c_char * 48)()
    C.memmove(buf, np.array([48 << 2, 1, 0, F8OID, 3, 1], np.int32).tobytes(), 24)
    C.memmove(C.byref(buf, 24), np.asarray(v, np.float64).tobytes(), 24)
    return buf


def ref_final(L, name, state):
    f = getattr(L, name)
    f.restype = C.c_uint64
    f.argtypes = [C.c_void_p]
    a = f8_array3(state)
    fc = FcInfo()
    fc.nargs = 1
    fc.arg[0] = C.addressof(a)
    d = f(C.byref(fc))
    return None if fc.isnull else float(np.array([d], np.uint64).view(np.float64)[0])


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref/libotbref.so is built only where the reference sources are present")
def test_finals_match_the_reference_objects():
    L = C.CDLL(REF_PATH)
    names = {g.GX_AGG_VAR_POP_F8: "float8_var_pop", g.GX_AGG_VAR_SAMP_F8: "float8_var_samp",
             g.GX_AGG_STDDEV_POP_F8: "float8_stddev_pop", g.GX_AGG_STDDEV_SAMP_F8: "float8_stddev_samp"}
    for name, x in datasets().items():
        sxx = V.sxx_exact(x)
        for fn, ref in names.items():
            want = V.expect(fn, x)
            got = ref_final(L, ref, [len(x), math.fsum(x), float(sxx)])
            if got is None:
                assert want == ("null",), (name, ref)
            else:
                assert V.matches(fn, want, got, 0), (name, ref, want, got)
    assert ref_final(L, "float8_var_pop", [0.0, 0.0, 0.0]) is None
    assert ref_final(L, "float8_stddev_samp", [1.0, 5.0, 0.0]) is None
    assert math.isnan(ref_final(L, "float8_var_samp", [3.0, 1.0, math.nan]))


# ---------------------------------------------------------------- the oracle's Youngs-Cramer state
def sxx_mean(x):
    return sum(Fraction(float(v)) for v in x) / len(x)


@pytest.mark.parametrize("name", list(datasets()))
def test_oracle_youngs_cramer_sxx_within_the_bar(name):
    x = datasets()[name]
    n = len(x)
    plan = O.make_plan(aggs=[(g.GX_AGG_AVG_F8, [(g.GX_OP_COL, 1, 0)])])
    rel = O.Rel([O.GX_INT8, O.GX_FLOAT8], [np.zeros(n, np.int64), np.ascontiguousarray(x)])
    st = O.exec_agg(rel, plan).states[0, 0]
    assert st[0] == n
    sxx = V.sxx_exact(x)
    # float8_accum's tmp = N x - Sx rounds at the magnitude of N x, not of the deviations: far from zero (1e9 + noise)
    # the reference's own Sxx needs 4 N M D 2^-52 more than the bar the device meets (M = max |x|, D the largest deviation)
    m = float(np.abs(x).max())
    d = max(abs(float(x.max()) - float(sxx_mean(x))), abs(float(x.min()) - float(sxx_mean(x))))
    tol = V.sxx_tol(x, sxx) + (4.0 * n * m * d * 2.0 ** -52 if name == "offset" else 0.0)
    assert st[2] >= 0 and abs(st[2] - float(sxx)) <= tol, (name, st[2], float(sxx))


# ---------------------------------------------------------------- the device's shifted sums and their merge
def shifted(x):
    """one partial state as a sink builds it: C = the first value, S1 = sum(x - C), S2 = sum((x - C)^2) in float8"""
    c = x[0]
    d = x - c
    s1 = s2 = 0.0
    for v in d:
        s1 += v
        s2 += v * v
    return [c, s1, s2, len(x)]


def merge(t, s):
    """var_merge / var_combine: s re-centred on t's shift (t takes s's shift when it has no input)"""
    if s[3] == 0:
        return t
    if t[3] == 0:
        return list(s)
    d = s[0] - t[0]
    nd = s[3] * d
    return [t[0], t[1] + (s[1] + nd), t[2] + ((s[2] + (2.0 * d) * s[1]) + nd * d), t[3] + s[3]]


@pytest.mark.parametrize("name", ["normal", "offset", "constant", "two", "wide", "ints"])
def test_recentring_merge_over_random_splits(name):
    x = datasets()[name]
    rng = np.random.default_rng(len(x))
    sxx = V.sxx_exact(x)
    tol = V.sxx_tol(x, sxx)
    for _ in range(5):
        x = rng.permutation(x)
        cuts = np.sort(rng.choice(np.arange(1, len(x)), size=min(len(x) - 1, 7), replace=False)) if len(x) > 1 else []
        parts = [p for p in np.split(x, cuts) if len(p)]
        acc = [0.0, 0.0, 0.0, 0]
        for p in parts:
            acc = merge(acc, shifted(p))
        v = acc[2] - acc[1] * acc[1] / acc[3]
        got = 0.0 if v <= 0 else v
        assert abs(got - float(sxx)) <= tol, (name, got, float(sxx), tol)
        if sxx == 0:
            assert got == 0.0
