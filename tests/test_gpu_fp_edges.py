"""Float8 and integer aggregates at IEEE and overflow edges, on every aggregation kernel family, against the
exact reference of tests/exact_ref.py (itself pinned to the oracle by tests/test_exact_ref_cpu.py).

gx_hash_agg answers one aggregate with one of a dozen kernels, picked by plan shape, group estimate, key order
and a few switches; each has its own accumulators, tail handling and flush.  Every family is forced here by the
shape and estimate that select it (plus the switch where the shape alone is not enough), and the fixture checks
through the family's profile name that it answered.  Datasets: mixed-sign cancellation across decades with
ragged group sizes (warp, tile, warp-chunk and CTA edges), subnormals, NaN / +-inf / -0, whole-query overflow
errors, extreme group keys, and results on both sides of the host / device fetch split."""
import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import distinct_ref as DR
import exact_ref as X
import fp_edge_data as D
import regr_ref as R
import var_ref as V
from helpers import to_gpu_plan

pytestmark = pytest.mark.gpu

C, K, MUL = g.GX_OP_COL, g.GX_OP_CONST, g.GX_OP_MUL
SX, AX, NX, MX = (g.GX_AGG_SUM_F8, [(C, 1, 0)]), (g.GX_AGG_AVG_F8, [(C, 1, 0)]), (g.GX_AGG_MIN_F8, [(C, 1, 0)]), (g.GX_AGG_MAX_F8, [(C, 1, 0)])
CNT = (g.GX_AGG_COUNT_STAR, [])
SXY = (g.GX_AGG_SUM_F8, [(C, 1, 0), (C, 2, 0), (MUL, 0, 0)])
SY = (g.GX_AGG_SUM_F8, [(C, 2, 0)])
XX = [(C, 1, 0), (C, 1, 0), (MUL, 0, 0)]

# aggregate lists each shape admits: the fast / run-folding kernels take ONE float8 column sum (plus count(*)),
# the register kernels chains over NOT NULL float8 columns, gx_k_agg and radix everything
SHAPES = {
    "count": [[CNT]],
    "fast": [[SX, CNT], [AX]],
    "value": [[SX, AX, CNT, SXY]],
    "general": [[SX, AX, NX, MX, CNT, SXY]],
    "ra1": [[SX, CNT], [AX]],
    "ra2": [[SX, SXY]],
    "ra3": [[SX, SXY, SY]],
}

# family: (input kind, est_groups, strategy, switches, most groups the kernel holds, shape, profile name)
FAMILIES = {
    "agg_count_char":     ("char", 3, 0, {}, 8, "count", "agg_count_char"),
    "agg_fewgroups":      ("scan", 4, 0, {}, 4, "value", "agg_fewgroups"),
    "agg_fewgroups_512":  ("scan", 4, 0, {"GX_FG_VARIANT": "0"}, 4, "value", "agg_fewgroups"),
    "agg_lptile8":        ("scan", 16, 0, {"GX_NO_FEWGROUPS": "1"}, 16, "value", "agg_lptile8"),
    "agg_lptile4":        ("scan", 16, 0, {"GX_NO_FEWGROUPS": "1", "GX_LPTILE_K4": "1"}, 16, "value", "agg_lptile4"),
    "agg_smem_lp":        ("scan", 16, 0, {}, 16, "general", "agg_smem_lp"),
    "agg_smem":           ("scan", 1000, 1, {}, None, "general", "agg_smem"),
    "agg_global":         ("scan", 1000, 3, {}, None, "general", "agg_global"),
    "radix":              ("scan", 1000, 2, {}, None, "general", "scan_records"),
    "agg_fast":           ("scan", 1000, 1, {}, None, "fast", "agg_fast"),
    "probe_agg_fast":     ("join", 1000, 0, {"GX_NO_RUNJOIN": "1"}, None, "fast", "probe_agg_fast"),
    "probe_agg_tma1":     ("join", 1000, 0, {"GX_RUNJOIN_TMA": "1"}, None, "fast", "probe_agg_tma"),
    "probe_agg_tma2":     ("join", 1000, 0, {"GX_RUNJOIN_TMA": "2"}, None, "fast", "probe_agg_tma"),
    "probe_agg_tma3":     ("join", 1000, 0, {"GX_RUNJOIN_TMA": "3"}, None, "fast", "probe_agg_tma"),
    "probe_agg_run":      ("join", 1000, 0, {"GX_RUNJOIN_TMA": "0", "GX_RUNJOIN_SEG": "0"}, None, "fast", "probe_agg_run"),
    "probe_agg_seg":      ("join", 1000, 0, {"GX_RUNJOIN_TMA": "0", "GX_RUNJOIN_SEG": "1"}, None, "fast", "probe_agg_seg"),
    "probe_agg_run2":     ("join", 1000, 0, {"GX_RUNJOIN_V2": "1"}, None, "fast", "probe_agg_run2"),
    "probe_agg_run3":     ("join", 1000, 0, {"GX_RUNJOIN_CARRY": "1"}, None, "fast", "probe_agg_run3"),
    "runagg_dense":       ("runagg", 1000, 0, {"GX_RUNAGG_DENSE": "1"}, None, "ra1", "runagg_dense"),
    "runagg_small1":      ("runagg", 1000, 0, {"GX_RUNAGG_DENSE": "0"}, None, "ra1", "runagg_small1"),
    "runagg_small2":      ("runagg", 1000, 0, {}, None, "ra2", "runagg_small2"),
    "runagg_wide":        ("runagg", 1000, 0, {}, None, "ra3", "runagg_wide"),
}
GENERAL = ["agg_smem_lp", "agg_smem", "agg_global", "radix"]
SEEN = set()                     # profile names that answered somewhere in this module


class Family:
    def __init__(self, gx, name):
        self.gx, self.name = gx, name
        self.kind, self.est, self.strategy, self.env, self.limit, self.shape, self.profile = FAMILIES[name]

    def run(self, gi, x, y, aggs, gkey_of=lambda i: i * 7 - 3, keep_order=False):
        """aggregate (group index per row, x, y) through this family; returns (plan, want, got-or-GxError).
        keep_order: the join families see the rows in the order given (keys rise with the row number)"""
        gx = self.gx
        G = int(gi.max()) + 1 if len(gi) else 0
        if self.kind in ("scan", "char"):
            keys = np.array([gkey_of(i) for i in range(G)], np.int64)
            kt = (g.GX_CHAR, np.int8) if self.kind == "char" else (g.GX_INT4, np.int32)
            types, cols = [kt[0], g.GX_FLOAT8, g.GX_FLOAT8], [keys[gi].astype(kt[1]), x, y]
            plan = O.make_plan(group_cols=[(0, 0)], aggs=aggs, est_groups=self.est, strategy=self.strategy)
            outer, ht = gx.table_from(types, cols), None
        else:
            # inner (orders-like): dense sorted keys 1..M, at least 200k of them for the key-ordered compact table
            # the streamed-table kernel needs; join families group by the int4 payload, runagg by the key
            per = 1 if self.kind == "runagg" else -(-200_000 // G)
            M = G * per
            ikeys = np.arange(1, M + 1, dtype=np.int64)
            ipay = np.array([gkey_of(i) for i in range(G)], np.int32)[np.arange(M) % G]
            inner = gx.table_from([g.GX_INT8, g.GX_INT4], [ikeys, ipay])
            ht = gx.hash_build(inner, 0, [1], unique=True)
            rng = np.random.default_rng(len(gi))
            t = np.arange(len(gi)) if keep_order and per >= len(gi) else rng.integers(0, per, len(gi))
            okey = (gi + 1 + G * t).astype(np.int64)
            o = np.argsort(okey, kind="stable")                    # clustered on the key, as lineitem is
            okey, gi, x, y = okey[o], gi[o], x[o], y[o]
            outer = gx.table_from([g.GX_INT8, g.GX_FLOAT8, g.GX_FLOAT8], [okey, x, y])
            gc = [(0, 0)] if self.kind == "runagg" else [(1, 0)]
            plan = O.make_plan(outer_key_col=0, group_cols=gc, aggs=aggs, est_groups=self.est, strategy=self.strategy)
            keys = np.arange(1, G + 1, dtype=np.int64) if self.kind == "runagg" else np.array([gkey_of(i) for i in range(G)], np.int64)
            cols = [okey, x, y]
        want = X.expect_groups(plan, cols, gindex=gi, gkeys=[(int(k),) for k in keys])
        gx.profile(True)
        try:
            got = gx.hash_agg(outer, to_gpu_plan(plan), ht).fetch()
        except g.GxError as e:
            got = e
        used = gx.profile_get(self.profile)[1]
        gx.profile(False)
        assert used > 0, f"{self.name}: {self.profile} did not run"
        SEEN.add(self.profile)
        outer.free()
        if ht is not None:
            ht.free(); inner.free()
        return plan, want, got

    def check(self, gi, x, y, aggs, **kw):
        plan, want, got = self.run(gi, x, y, aggs, **kw)
        if want == "overflow":
            assert isinstance(got, g.GxError) and got.status == g.GX_ERR_OVERFLOW, f"{self.name}: want overflow, got {got!r}"[:400]
        else:
            assert not isinstance(got, g.GxError), f"{self.name}: {got}"
            X.check(plan, want, got, [g.GX_INT8 if self.kind == "runagg" else g.GX_INT4])


@pytest.fixture(params=list(FAMILIES))
def family(request, gx, monkeypatch):
    for k, v in FAMILIES[request.param][3].items():
        monkeypatch.setenv(k, v)
    return Family(gx, request.param)


def _plans(fam, avg_ok=True):
    return [a for a in SHAPES[fam.shape] if avg_ok or not any(f == g.GX_AGG_AVG_F8 for f, _ in a)]


def test_cancel(family):
    rng = np.random.default_rng(1)
    for aggs in _plans(family):
        has_avg = any(f == g.GX_AGG_AVG_F8 for f, _ in aggs)
        for sizes in D.batches(D.CANCEL_SIZES, family.limit or len(D.CANCEL_SIZES)):
            family.check(*D.cancel(rng, sizes, top=100 if has_avg else 300), aggs)


def test_subnormal(family):
    rng = np.random.default_rng(2)
    for aggs in _plans(family):
        family.check(*D.subnormal(rng, min(6, family.limit or 6)), aggs)


def test_special(family):
    """inf / -inf / both, NaN with finite values, only -0, mixed zeros, NaN-only min/max, avg with inf"""
    rng = np.random.default_rng(3)
    for aggs in _plans(family):
        for part in D.batches(D.SPECIAL_GROUPS, family.limit or len(D.SPECIAL_GROUPS)):
            family.check(*D.special(rng, part), aggs)


def test_sum_overflow_in_the_last_partial_tile(family):
    """finite inputs whose sum leaves the float8 range, in the last two rows: the whole query fails.  Group 2
    also sorts last for the run-aggregate kernels, whose outer side is in key order."""
    if family.shape == "count":
        pytest.skip("count(*) only")
    n = 3971
    gi = np.arange(n) % 3
    gi[-2:] = 2
    x = np.full(n, 0.25)
    x[-2:] = 1e308
    family.check(gi, x, np.ones(n), SHAPES[family.shape][0], keep_order=True)


def test_expression_overflow(family):
    """x * x leaving the range from finite x: an error for SUM, and for MIN / MAX where the kernel takes them"""
    if family.shape not in ("value", "general"):
        pytest.skip("the fast and run-aggregate kernels take plain column sums only")
    n = 300
    gi = np.arange(n) % 3
    x = np.full(n, 3.0)
    x[-1] = 1e200
    fns = [g.GX_AGG_SUM_F8] + ([g.GX_AGG_MIN_F8, g.GX_AGG_MAX_F8] if family.shape == "general" else [])
    for fn in fns:
        xv = np.full(n, 1e200) if fn == g.GX_AGG_MIN_F8 else x     # min(x*x) overflows only if every row does
        family.check(gi, xv, np.ones(n), [(fn, XX)] + SHAPES[family.shape][0])     # the shape's own words keep the family


@pytest.mark.parametrize("name", GENERAL)
def test_group_key_edges(gx, monkeypatch, name):
    """int8 keys at INT64_MIN / MAX, int4 keys at INT32_MIN, 0, -1 (the tag-key packing), float8 keys +-0 and
    NaN / -NaN (NaN keys group by their bits, as hashfloat8 does), sum(int4) over INT32_MIN / MAX exactly"""
    fam = Family(gx, name)
    i64, i32 = np.iinfo(np.int64), np.iinfo(np.int32)
    nan, nnan = np.float64(np.nan), -np.float64(np.nan)
    n = 4099
    rng = np.random.default_rng(4)
    k8 = rng.choice(np.array([i64.min, i64.max, 0, -1, 1], np.int64), n)
    k4 = rng.choice(np.array([i32.min, 0, -1, i32.max], np.int32), n)
    kf = rng.choice(np.array([0.0, -0.0, nan, nnan, 1.5]), n)
    v4 = rng.choice(np.array([i32.min, i32.max], np.int32), n)
    x = rng.random(n)
    types = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8, g.GX_INT4, g.GX_FLOAT8]
    cols = [k8, k4, kf, v4, x]
    t = gx.table_from(types, cols)
    for gcols in ([0], [1], [2], [1, 0], [2, 1]):
        plan = O.make_plan(group_cols=[(0, c) for c in gcols], aggs=[(g.GX_AGG_SUM_I4, [(C, 3, 0)]), (g.GX_AGG_SUM_F8, [(C, 4, 0)]), CNT],
                           est_groups=fam.est, strategy=fam.strategy)
        want = X.expect_groups(plan, cols, types=types)
        gx.profile(True)
        got = gx.hash_agg(t, to_gpu_plan(plan)).fetch()
        assert gx.profile_get(fam.profile)[1] > 0 or name == "agg_smem_lp"       # 2 x 5 keys exceed its estimate
        gx.profile(False)
        X.check(plan, want, got, [types[c] for c in gcols])
    t.free()


@pytest.mark.parametrize("ngroups", [8192, 8193])
@pytest.mark.parametrize("name", ["agg_global", "radix"])
def test_fetch_paths_see_special_values(gx, name, ngroups):
    """8192 groups are finalized on the host, 8193 on the device (gx_k_finalize): both see inf / NaN / -0"""
    fam = Family(gx, name)
    fam.est = ngroups
    groups = [D.SPECIAL_GROUPS[i % len(D.SPECIAL_GROUPS)] for i in range(ngroups)]
    gi, x, y = D.special(np.random.default_rng(5), groups)
    fam.check(gi, x, y, SHAPES["general"][0], gkey_of=lambda i: i * 3 - 9000)


INF, NAN = float("inf"), float("nan")
# test_finalize_paths_agree: group shapes as (x, y, v) rows, None for NULL; None for an ordinary group.  At most four
# inputs of small dyadic values per group: every state is exact in whatever order the rows arrive, so two runs over
# the same rows hold the same states
FINAL_SHAPES = [
    [(None, None, None)] * 2,                                            # all inputs NULL
    [(1.5, -2.5, 7)],                                                    # one input: the _samp variances, covar_samp NULL
    [(2.0, 1.0, 1), (2.0, 2.0, 1), (2.0, 4.0, 2), (2.0, 9.0, 3)],        # constant X: corr, regr_slope NULL
    [(1.0, 5.0, 4), (2.0, 5.0, 4), (3.0, 5.0, 4), (6.0, 5.0, 5)],        # constant Y, varying X: regr_r2 = 1
    [(INF, 1.0, 1), (1.0, 2.0, 2), (2.0, 3.0, 3), (3.0, 4.0, 4)],
    [(1.0, -INF, 1), (2.0, 1.0, 1), (0.5, 1.0, 2), (4.0, 2.0, 2)],
    [(NAN, 1.0, 6), (1.0, 1.0, 6), (2.0, NAN, 6), (3.0, 2.0, 6)],
    [(-0.0, -0.0, 0), (-0.0, -0.0, 0)],                                  # sums that end at -0
    None, None,
]
X1, Y2, V3 = [(C, 1, 0)], [(C, 2, 0)], [(C, 3, 0)]
PAIR = Y2 + [(g.GX_OP_ARG2, 0, 0)] + X1
# every aggregate function of the ABI but the declined sum(int8), in as many plans as GX_MAX_AGGS asks for
FINAL_PLANS = [
    [CNT, (g.GX_AGG_COUNT, V3), (g.GX_AGG_SUM_I4, V3), SX, AX, NX, MX],
    [(fn, X1) for fn in V.VAR_FNS] + [(fn, PAIR) for fn in R.REGR_FNS[:4]],
    [(fn, PAIR) for fn in R.REGR_FNS[4:]],
    [(g.GX_AGG_COUNT_DISTINCT, V3), CNT, SX],
]
INT_RESULTS = {g.GX_AGG_COUNT_STAR, g.GX_AGG_COUNT, g.GX_AGG_SUM_I4, g.GX_AGG_REGR_COUNT, g.GX_AGG_COUNT_DISTINCT}


def _final_bits(aggs, vals):
    """the result bits, NaN payloads canonicalised in the float8 results: a NaN the final itself makes (inf - inf in a
    variance's Sxx) is the default NaN of whichever processor finalized"""
    b = vals.view(np.int64).copy()
    for a, (fn, _) in enumerate(aggs):
        if fn not in INT_RESULTS:
            b[np.isnan(vals[:, a]), a] = np.float64(NAN).view(np.int64)
    return b


def test_finalize_paths_agree(gx):
    """8193 groups are finalized on the device (gx_k_finalize), the same rows without one ordinary group on the host
    (8192): every aggregate function over groups without input, with one input, a constant X or Y, +-inf, NaN and
    sums ending at -0 gives the same bits and NULL flags on both paths, and both match the exact references"""
    rng = np.random.default_rng(9)
    gi, xs, ys, vs = [], [], [], []
    for i in range(8193):
        shape = FINAL_SHAPES[i % len(FINAL_SHAPES)]
        if shape is None:
            shape = [(rng.integers(-8, 9) / 4, rng.integers(-8, 9) / 4, int(rng.integers(0, 3))) for _ in range(4)]
            if i % 3 == 0:
                shape.append((None, None, None))
        for x, y, v in shape:
            gi.append(i); xs.append(x); ys.append(y); vs.append(v)
    gi = np.array(gi)
    drop = max(i for i in range(8193) if FINAL_SHAPES[i % len(FINAL_SHAPES)] is None)
    gkeys = [(i * 3 - 9000,) for i in range(8193)]
    types = [g.GX_INT4, g.GX_FLOAT8, g.GX_FLOAT8, g.GX_INT4]
    runs = {}
    for ngroups, rows in ((8193, np.arange(len(gi))), (8192, np.flatnonzero(gi != drop))):
        key = (gi[rows] * 3 - 9000).astype(np.int32)
        cols = [key] + [np.array([0 if vals[r] is None else vals[r] for r in rows], t) for vals, t in ((xs, np.float64), (ys, np.float64), (vs, np.int32))]
        nulls = [None] + [np.array([vals[r] is None for r in rows], np.uint8) for vals in (xs, ys, vs)]
        t = gx.table_from(types, cols, nulls)
        runs[ngroups] = []
        for aggs in FINAL_PLANS:
            plan = g.make_plan(group_cols=[(0, 0)], aggs=aggs, est_groups=ngroups)
            gx.profile(True)
            got = gx.hash_agg(t, plan).fetch()
            on_device = gx.profile_get("finalize")[1] > 0
            gx.profile(False)
            assert on_device == (ngroups > 8192) and len(got[0]) == ngroups
            if aggs[0][0] == g.GX_AGG_COUNT_DISTINCT:
                DR.check(plan, DR.expect_groups(plan, cols, types, np.arange(len(rows)), nulls), got, [g.GX_INT4])
            elif aggs[0] == CNT:
                X.check(plan, X.expect_groups(plan, cols, nulls, gindex=gi[rows], gkeys=gkeys), got, [g.GX_INT4])
            else:
                checked = R.check(plan, cols, nulls, key.astype(np.int64), got)
                if aggs[0][0] in V.VAR_FNS:
                    checked += V.check(plan, cols, nulls, key.astype(np.int64), got)
                assert checked == ngroups * len(aggs)
            runs[ngroups].append(got)
        t.free()
    for aggs, (k0, a0, n0), (k1, a1, n1) in zip(FINAL_PLANS, runs[8193], runs[8192]):
        at = {int(k): i for i, k in enumerate(k0[:, 0])}
        rows = np.array([at[int(k)] for k in k1[:, 0]])
        assert (drop * 3 - 9000) not in set(k1[:, 0].tolist())
        np.testing.assert_array_equal(_final_bits(aggs, a0[rows]), _final_bits(aggs, a1))
        np.testing.assert_array_equal(n0[rows], n1)


def test_sum_int8_is_declined(gx):
    """sum(int8) would wrap in the int64 accumulators; the reference's sum(int8) returns numeric"""
    t = gx.table_from([g.GX_INT4, g.GX_INT8], [np.zeros(3, np.int32), np.array([2**62, 2**62, 5], np.int64)])
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[(g.GX_AGG_SUM_I8, [(C, 1, 0)])], est_groups=4)
    with pytest.raises(g.GxError) as ei:
        gx.hash_agg(t, plan)
    assert ei.value.status == g.GX_ERR_ARG
    t.free()


def test_quals_over_special_values(gx):
    """float8 quals over NaN / +-inf / -0 through the register kernels' vectorised qual (pred_tile):
    x >= 0 keeps -0, x < inf drops NaN (NaN sorts above everything)"""
    rng = np.random.default_rng(6)
    vals = np.array([-0.0, 0.0, np.nan, np.inf, -np.inf, 1.0, -1.0, 5e-324])
    n = 5000
    q = rng.choice(vals, n)
    gi = rng.integers(0, 3, n)
    x = rng.random(n)
    types = [g.GX_INT4, g.GX_FLOAT8, g.GX_FLOAT8]
    cols = [gi.astype(np.int32), x, q]
    t = gx.table_from(types, cols)
    for op, k, keep in ((g.GX_GE, 0.0, (q >= 0) | np.isnan(q)), (g.GX_LT, np.inf, q < np.inf), (g.GX_LE, -0.0, q <= 0), (g.GX_GT, -np.inf, (q > -np.inf) | np.isnan(q))):
        for est, fam in ((3, "agg_fewgroups"), (1000, "agg_smem")):
            plan = O.make_plan(preds=[(2, op, k, True)], group_cols=[(0, 0)], aggs=[SX, CNT], est_groups=est)
            want = X.expect_groups(plan, cols, types=types, keep=keep)
            gx.profile(True)
            got = gx.hash_agg(t, to_gpu_plan(plan)).fetch()
            assert gx.profile_get(fam)[1] > 0, f"{fam} did not run"
            gx.profile(False)
            X.check(plan, want, got, [g.GX_INT4])
    t.free()


def test_known_deviations_are_pinned(gx):
    """Two reference errors the kernels do not see (DESIGN.md §3.2, §7): float8mul underflow to zero from non-zero
    factors, and avg()'s sum of squares going infinite from finite inputs.  The oracle errors; the GPU answer is
    pinned here so that a change either way is noticed."""
    types = [g.GX_INT4, g.GX_FLOAT8, g.GX_FLOAT8]
    cols = [np.zeros(4, np.int32), np.array([1e-200, 2.0, 3.0, 4.0]), np.array([1e-200, 1.0, 1.0, 1.0])]
    plan = O.make_plan(group_cols=[(0, 0)], aggs=[SXY], est_groups=4)
    with pytest.raises(RuntimeError, match="status 6"):
        O.exec_agg(O.Rel(types, cols), plan)
    t = gx.table_from(types, cols)
    _, aggs, _ = gx.hash_agg(t, to_gpu_plan(plan)).fetch()
    t.free()
    assert aggs[0, 0] == 9.0                                  # 0 + 2 + 3 + 4: the underflowed product counts as 0
    cols = [np.zeros(4, np.int32), np.array([1e200, -1e200, 1e200, -1e200]), np.ones(4)]
    plan = O.make_plan(group_cols=[(0, 0)], aggs=[AX], est_groups=4)
    with pytest.raises(RuntimeError, match="status 6"):
        O.exec_agg(O.Rel(types, cols), plan)
    t = gx.table_from(types, cols)
    _, aggs, _ = gx.hash_agg(t, to_gpu_plan(plan)).fetch()
    t.free()
    assert aggs[0, 0] == 0.0 and not np.signbit(aggs[0, 0])


@pytest.mark.parametrize("name", ["agg_global", "radix"])
def test_fetch_states_see_special_values(gx, name):
    """partial states for a two-phase plan (gx_result_fetch_states): per aggregate N and Sx / min / max, with inf,
    NaN and -0 in them; avg's Sx starts at +0 as float8_accum's '{0,0,0}' does"""
    fam = Family(gx, name)
    gi, x, y = D.special(np.random.default_rng(8))
    keys = np.arange(len(D.SPECIAL_GROUPS)) * 7 - 3
    t = gx.table_from([g.GX_INT4, g.GX_FLOAT8, g.GX_FLOAT8], [keys[gi].astype(np.int32), x, y])
    aggs = [SX, AX, NX, MX, CNT]
    plan = O.make_plan(group_cols=[(0, 0)], aggs=aggs, est_groups=fam.est, strategy=fam.strategy)
    gx.profile(True)
    k, vals, cnts, nulls = gx.hash_agg(t, to_gpu_plan(plan)).fetch_states()
    assert gx.profile_get(fam.profile)[1] > 0
    gx.profile(False)
    t.free()
    assert sorted(k[:, 0].tolist()) == sorted(keys.tolist())
    for row in range(k.shape[0]):
        v = np.array(D.SPECIAL_GROUPS[int(np.flatnonzero(keys == k[row, 0])[0])])
        sx = X.expect_sum(v)
        ax = X.Expect("value", 0.0, None, zero_sign=1.0) if sx.value == 0 else sx      # Sx from '{0,0,0}'
        want = [sx, ax, X.expect_minmax(v, False), X.expect_minmax(v, True)]
        for a, e in enumerate(want):
            assert e.matches(float(vals[row, a]), bool(nulls[row, 1 + a])), (k[row, 0], a, vals[row, a], e)
            assert cnts[row, a] == len(v)
        assert cnts[row, 4] == len(v) and not nulls[row, 1:].any()


COUNT_FAMILIES = [("agg_count_char", [], 3, 0), ("agg_fewgroups", [(0, g.GX_GE, 0)], 3, 0), ("agg_smem", [], 1000, 1)]


def test_count_beyond_32_bits(gx):
    """count(*) GROUP BY l_returnflag over more than 2^32 lineitem rows (one column, generated on the device), through
    the kernels that keep 32-bit counters per thread or per CTA: gx_k_count_char, gx_k_fewgroups, gx_k_agg's
    shared-memory table.  The counts are checked against a host histogram of the same column."""
    torch = pytest.importorskip("torch")
    free, _ = torch.cuda.mem_get_info(0)
    if free < 16 << 30:
        pytest.skip("needs 16 GB of free device memory")
    sf, nord = 800, 1_100_000_000                              # about 4 lines per order: ~4.4e9 rows
    t = gx.table([g.GX_CHAR], 4_700_000_000).generate(g.T_LINEITEM, sf, 0, nord, colmap=[g.L_RETURNFLAG])
    n = t.nrows
    assert n > 2**32
    hist = np.zeros(256, np.int64)
    chunk = 1 << 28
    buf = np.empty(chunk, np.int8)
    for r0 in range(0, n, chunk):
        m = min(chunk, n - r0)
        gx._chk(g.lib().gx_table_read_column(t.h, 0, r0, m, buf.ctypes.data, None))
        hist += np.bincount(buf[:m].view(np.uint8), minlength=256)
    want = {int(np.int8(np.uint8(b))): int(c) for b, c in enumerate(hist) if c}
    for prof, preds, est, strategy in COUNT_FAMILIES:
        plan = g.make_plan(preds=preds, group_cols=[(0, 0)], aggs=[CNT], est_groups=est, strategy=strategy)
        gx.profile(True)
        keys, aggs, _ = gx.hash_agg(t, plan).fetch()
        assert gx.profile_get(prof)[1] > 0, f"{prof} did not run"
        gx.profile(False)
        got = {int(k): int(c) for k, c in zip(keys[:, 0], aggs[:, 0].view(np.int64))}
        assert got == want, (prof, got, want)
        SEEN.add(prof)
    t.free()


def test_zz_every_family_answered_somewhere(request):
    """runs last: a dispatch change that silently reroutes a shape shows up as a family nobody reached.  Judged only
    when every family's tests were collected in this session (not under -k or a partial selection)."""
    ids = {it.nodeid.split("::")[-1] for it in request.session.items}
    if not all(f"test_special[{f}]" in ids and f"test_cancel[{f}]" in ids for f in FAMILIES):
        pytest.skip("not every family's tests were selected")
    want = {f[6] for f in FAMILIES.values()}
    assert SEEN >= want, f"families that never ran: {sorted(want - SEEN)}"
