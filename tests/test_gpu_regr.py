"""regr_count / regr_sxx .. regr_intercept / covar_pop / covar_samp / corr over float8 pairs (GX_AGG_REGR_COUNT ..
GX_AGG_CORR_F8) on the device.

The state is shifted sums for X and Y plus their cross term, merged with re-centring wherever partial states meet.
Every case is compared with tests/regr_ref.py, exact rational sums with the bounds DESIGN.md §3.2 states, across every
sink of gx_k_agg (asserted by profile name), the join shapes that feed it, gx_exec_host, count(DISTINCT)'s fold, the
edge data of IEEE arithmetic, and the partial states a two-phase plan ships to the reference's float8_regr_combine."""
import os

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import regr_ref as R
import var_ref as V

pytestmark = pytest.mark.gpu

F8 = lambda c: [(g.GX_OP_COL, c, 0)]
SEP = [(g.GX_OP_ARG2, 0, 0)]
PAIR = F8(2) + SEP + F8(3)                     # (Y, X) = (column 2, column 3)
ALL = [(fn, PAIR) for fn in R.REGR_FNS]        # all twelve over one pair: one shared state
SINKS = {"agg_smem", "agg_smem_lp", "agg_global", "agg_records", "agg_fewgroups", "agg_lptile8", "agg_lptile4", "runagg",
         "agg_distinct_fold", "probe_agg_exist_wide", "probe_agg_exist_compact", "probe_agg_exist_narrow",
         "probe_agg_chain_wide", "probe_agg_chain_compact", "probe_agg_chain_narrow"}
# outer columns: 0 join key int8, 1 group int4, 2 y float8 (nullable), 3 x float8 (nullable), 4 int4, 5 float8
OTYPES = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8, g.GX_FLOAT8, g.GX_INT4, g.GX_FLOAT8]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_PATH = os.path.join(ROOT, "oracle", "_ref", "libotbref.so")
HAVE_REF = os.path.exists(REF_PATH)


def outer(rng, n, ngroups, null_frac=0.05, loc=0.0, scale=100.0, nkeys=1000):
    k = rng.integers(0, nkeys, n).astype(np.int64)
    grp = rng.integers(0, ngroups, n).astype(np.int32)
    x = loc + rng.standard_normal(n) * scale
    y = 0.5 * x + rng.standard_normal(n) * scale
    d = rng.integers(0, 50, n).astype(np.int32)
    z = rng.random(n) * 10.0
    ny = (rng.random(n) < null_frac).astype(np.uint8)
    nx = (rng.random(n) < null_frac).astype(np.uint8)
    return [k, grp, y, x, d, z], [None, None, ny, nx, None, None]


def run(gx, fn):
    gx.profile(True)
    try:
        res = fn()
        got = res.fetch()
        ran = {p for p in SINKS if gx.profile_get(p)[1] > 0}
    finally:
        gx.profile(False)
    return got, ran, res


def check(plan, cols, nulls, got, rows=None):
    keys = cols[1].astype(np.int64) if plan.n_group_cols else np.zeros(len(cols[0]), np.int64)
    assert R.check(plan, cols, nulls, keys, got, rows) > 0


def no_join(gx, cols, nulls, plan):
    t = gx.table_from(OTYPES, cols, nulls)
    got, ran, res = run(gx, lambda: gx.hash_agg(t, plan))
    check(plan, cols, nulls, got)
    return got, ran, res


# ---------------------------------------------------------------- every sink of gx_k_agg
@pytest.mark.parametrize("strategy,ngroups,est,sink", [(1, 8, 8, "agg_smem_lp"), (1, 2000, 2000, "agg_smem"),
                                                        (3, 2000, 2000, "agg_global"), (2, 50_000, 50_000, "agg_records")])
def test_sinks(gx, strategy, ngroups, est, sink):
    rng = np.random.default_rng(ngroups + strategy)
    cols, nulls = outer(rng, 400_000, ngroups)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=ALL[:7] + [(g.GX_AGG_COUNT_STAR, [])], est_groups=est, strategy=strategy)
    _, ran, _ = no_join(gx, cols, nulls, plan)
    assert sink in ran, sorted(ran)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=ALL[7:] + [(g.GX_AGG_SUM_F8, F8(5))], est_groups=est, strategy=strategy)
    _, ran, _ = no_join(gx, cols, nulls, plan)
    assert sink in ran, sorted(ran)


def test_mid_size_group_count_takes_the_global_table(gx):
    """groups that outgrow the shared table (a regression record is 12 words or more) but not L2's global table: the
    automatic strategy takes the global table, not the radix path's record per row"""
    rng = np.random.default_rng(3)
    cols, nulls = outer(rng, 400_000, 3000)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=ALL[:8], est_groups=3000)
    _, ran, _ = no_join(gx, cols, nulls, plan)
    assert "agg_global" in ran and "agg_records" not in ran, sorted(ran)


def test_specialised_kernels_not_taken(gx):
    """a plan the few-group and tiled kernels would take without the regression goes to gx_k_agg with it"""
    rng = np.random.default_rng(1)
    cols, _ = outer(rng, 300_000, 4, null_frac=0.0)
    nulls = [None] * 6
    base = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, F8(5))]
    t = gx.table_from(OTYPES, cols, nulls)
    _, ran, _ = run(gx, lambda: gx.hash_agg(t, g.make_plan(group_cols=[(0, 1)], aggs=base, est_groups=4)))
    assert ran & {"agg_fewgroups", "agg_lptile8", "agg_lptile4"}, sorted(ran)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=base + [(g.GX_AGG_CORR_F8, PAIR)], est_groups=4)
    got, ran, _ = run(gx, lambda: gx.hash_agg(t, plan))
    assert "agg_smem_lp" in ran and not ran & {"agg_fewgroups", "agg_lptile8", "agg_lptile4"}, sorted(ran)
    check(plan, cols, nulls, got)


# ---------------------------------------------------------------- joins and the host entry
def build(gx, fmt, n=50_000):
    """unique int8 keys in bunches of eight: key-ordered with a small int4 payload (narrow), key-ordered without
    payload (compact), or shuffled (wide)"""
    i = np.arange(n, dtype=np.int64)
    keys = (i // 8) * 32 + (i % 8) + 1
    if fmt == "wide":
        keys = np.random.default_rng(2).permutation(keys)
    pay = (keys % 2406 - 2922).astype(np.int32)
    t = gx.table_from([g.GX_INT8, g.GX_INT4], [keys, pay])
    return gx.hash_build(t, 0, [] if fmt == "compact" else [1], unique=True), t, keys


@pytest.mark.parametrize("jt", [g.GX_JOIN_INNER, g.GX_JOIN_SEMI, g.GX_JOIN_ANTI])
@pytest.mark.parametrize("fmt", ["wide", "compact", "narrow"])
@pytest.mark.parametrize("strategy", [1, 2])
def test_joins(gx, jt, fmt, strategy):
    rng = np.random.default_rng(jt * 10 + strategy)
    ht, _, bkeys = build(gx, fmt)
    cols, nulls = outer(rng, 300_000, 300, nkeys=200_000)
    plan = g.make_plan(outer_key_col=0, group_cols=[(0, 1)], aggs=ALL[:8], est_groups=300, strategy=strategy)
    plan.join_type = jt
    t = gx.table_from(OTYPES, cols, nulls)
    got, ran, _ = run(gx, lambda: gx.hash_agg(t, plan, ht))
    hit = np.isin(cols[0], bkeys)
    check(plan, cols, nulls, got, np.flatnonzero(~hit if jt == g.GX_JOIN_ANTI else hit))
    if jt != g.GX_JOIN_INNER:
        assert f"probe_agg_exist_{fmt}" in ran, sorted(ran)


def test_chain_of_two(gx):
    rng = np.random.default_rng(5)
    h1, _, k1 = build(gx, "narrow")
    k2 = np.arange(1000, dtype=np.int32)
    t2 = gx.table_from([g.GX_INT4, g.GX_INT4], [k2[::2].copy(), (k2[::2] % 7).astype(np.int32)])
    h2 = gx.hash_build(t2, 0, [1], unique=True)
    cols, nulls = outer(rng, 300_000, 100, nkeys=150_000)
    cols[4] = rng.integers(0, 1000, len(cols[0])).astype(np.int32)   # step 2 probes with column 4
    plan = g.make_plan(group_cols=[(0, 1)], aggs=ALL[4:], est_groups=100)
    t = gx.table_from(OTYPES, cols, nulls)
    got, ran, _ = run(gx, lambda: gx.hash_agg_joins(t, [(h1, (0, 0)), (h2, (0, 4))], plan))
    check(plan, cols, nulls, got, np.flatnonzero(np.isin(cols[0], k1) & np.isin(cols[4], k2[::2])))
    assert "probe_agg_chain_narrow" in ran, sorted(ran)


def test_exec_host(gx):
    rng = np.random.default_rng(6)
    cols, _ = outer(rng, 200_000, 50, null_frac=0.0, nkeys=100_000)
    nulls = [None] * 6
    bkeys = np.arange(0, 100_000, 2, dtype=np.int64)
    pay = (bkeys % 5).astype(np.int32)
    plan = g.make_plan(outer_key_col=0, group_cols=[(0, 1)], aggs=ALL[:8], est_groups=50)
    got = gx.exec_host(OTYPES, cols, len(cols[0]), plan, inner_types=[g.GX_INT8, g.GX_INT4], inner_ptrs=[bkeys, pay],
                       inner_nrows=len(bkeys), inner_key_col=0, payload_cols=[1], inner_unique=True).fetch()
    check(plan, cols, nulls, got, np.flatnonzero(np.isin(cols[0], bkeys)))


@pytest.mark.parametrize("strategy", [1, 2])
def test_with_count_distinct_and_a_variance(gx, strategy):
    """stage 1 keeps a regression state and a variance state per (group, value) pair; the fold re-centres both into the
    plan's groups"""
    rng = np.random.default_rng(7 + strategy)
    cols, nulls = outer(rng, 300_000, 40, loc=1e6)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_COUNT_DISTINCT, F8(4)), (g.GX_AGG_VAR_SAMP_F8, F8(5)),
                                                  (g.GX_AGG_CORR_F8, PAIR), (g.GX_AGG_REGR_SLOPE_F8, PAIR),
                                                  (g.GX_AGG_REGR_COUNT, PAIR)], est_groups=2000, strategy=strategy)
    got, ran, _ = no_join(gx, cols, nulls, plan)
    assert "agg_distinct_fold" in ran, sorted(ran)
    counts = got[1][:, 0].view(np.int64)
    for gi, k in enumerate(got[0][:, 0]):
        assert counts[gi] == len(np.unique(cols[4][cols[1] == k]))
    assert V.check(plan, cols, nulls, cols[1].astype(np.int64), got) == len(got[0])        # the var_samp next to them


# ---------------------------------------------------------------- edge data
@pytest.mark.parametrize("strategy,est,sink", [(1, 16, "agg_smem_lp"), (1, 30, "agg_smem"), (2, 30, "agg_records"),
                                               (3, 30, "agg_global")])
def test_edge_groups(gx, strategy, est, sink):
    """N = 0, 1, 2; NULL in Y only, X only, both; constant X, constant Y (exactly 0); 1e9 + U(0,1); -0.0; +-Inf and NaN
    in each argument, the inf - (-inf) cross case and the unset shift's own NaN bits among them"""
    sentinel = np.array([0x7FF4000000000001], np.uint64).view(np.float64)[0]
    rng = np.random.default_rng(strategy)
    r = lambda n: list(rng.random(n))
    groups = {   # group: (y values, x values)
        1: ([3.5], [1.0]), 2: ([1.0, 3.0], [2.0, 5.0]), 3: (r(300), [7.25] * 300), 4: ([-3.0] * 300, r(300)),
        5: (list(1e9 + rng.random(2000)), list(1e9 + rng.random(2000))), 6: ([-0.0] * 10 + [0.0] * 5, [0.0] * 5 + [-0.0] * 10),
        7: (r(100) + [np.inf], r(101)), 8: (r(101), r(100) + [np.inf]), 9: (r(50) + [np.nan], r(51)), 10: (r(51), r(50) + [np.nan]),
        11: ([1.0, -np.inf, 2.0], [2.0, np.inf, 3.0]), 12: ([np.inf, 2.0], [-np.inf, 1.0]), 13: ([sentinel] + r(300), r(300) + [sentinel]),
        15: ([1.0, 2.0, 3.0], [1e15] * 2 + [1e15 + 2.0]), 16: ([np.inf] * 3, [5.0] * 3),
    }
    grp, ys, xs, ny, nx = [], [], [], [], []
    for k, (yv, xv) in groups.items():
        n = len(yv)
        # the pairs, then a NULL Y, a NULL X and a NULL pair
        grp += [k] * (n + 3); ys += yv + [9.0, 1e300, 5.0]; xs += xv + [1e300, 9.0, 5.0]
        ny += [0] * n + [1, 0, 1]; nx += [0] * n + [0, 1, 1]
    grp += [17] * 4; ys += [1.0] * 4; xs += [2.0] * 4; ny += [1, 0, 1, 0]; nx += [0, 1, 1, 1]          # N = 0: no pair at all
    order = rng.permutation(len(grp))
    n = len(grp)
    cols = [np.zeros(n, np.int64), np.array(grp, np.int32)[order], np.array(ys)[order], np.array(xs)[order],
            np.zeros(n, np.int32), np.zeros(n)]
    nulls = [None, None, np.array(ny, np.uint8)[order], np.array(nx, np.uint8)[order], None, None]
    for aggs in (ALL[:6], ALL[6:]):
        plan = g.make_plan(group_cols=[(0, 1)], aggs=aggs, est_groups=est, strategy=strategy)
        got, ran, res = no_join(gx, cols, nulls, plan)
        assert sink in ran, sorted(ran)
    # constant X: Sxx exactly 0 and the vertical-line NULLs; constant Y: regr_r2 exactly 1.0, corr NULL
    plan = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_REGR_SXX_F8, PAIR), (g.GX_AGG_REGR_SYY_F8, PAIR),
                                                  (g.GX_AGG_REGR_R2_F8, PAIR), (g.GX_AGG_CORR_F8, PAIR)], est_groups=est, strategy=strategy)
    (k, a, nl), _, _ = no_join(gx, cols, nulls, plan)
    i3, i4 = list(k[:, 0]).index(3), list(k[:, 0]).index(4)
    assert a[i3, 0] == 0.0 and nl[i3, 1 + 2] and nl[i3, 1 + 3]
    assert a[i4, 1] == 0.0 and a[i4, 2] == 1.0 and nl[i4, 1 + 3]


def test_no_group_by_and_empty_input(gx):
    rng = np.random.default_rng(9)
    cols, nulls = outer(rng, 100_000, 1)
    no_join(gx, cols, nulls, g.make_plan(aggs=ALL[:8], est_groups=1))
    empty = [c[:0].copy() for c in cols]
    t = gx.table_from(OTYPES, empty, [None, None, np.zeros(0, np.uint8), np.zeros(0, np.uint8), None, None])
    plan = g.make_plan(aggs=ALL[:8], est_groups=1)
    r = gx.hash_agg(t, plan)
    _, aggs, nl = r.fetch()
    assert nl[0].tolist() == [0] + [1] * 7 and aggs[0, 0].view(np.int64) == 0
    _, vals, cnts, snl = r.fetch_states()
    assert vals[0].tolist() == [0.0] * 8 and cnts[0].tolist() == [0] * 8 and snl[0].tolist() == [0] * 8
    assert (r.fetch_regr() == 0.0).all()


def test_expression_argument(gx):
    """corr(l_extendedprice * (1 - l_discount), l_quantity) over lineitem rows: 7 of the 12 ops"""
    l = O.gen_lineitem(1, 0, 20_000)
    y = [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0), (g.GX_OP_CONST, 0, 1.0), (g.GX_OP_COL, g.L_DISCOUNT, 0), (g.GX_OP_SUB, 0, 0),
         (g.GX_OP_MUL, 0, 0)]
    pair = y + SEP + F8(g.L_QUANTITY)
    plan = g.make_plan(group_cols=[(0, g.L_RETURNFLAG)], aggs=[(fn, pair) for fn in R.REGR_FNS[:8]], est_groups=3)
    t = gx.table_from(g.SCHEMAS[g.T_LINEITEM], l)
    got = gx.hash_agg(t, plan).fetch()
    assert R.check(plan, l, None, l[g.L_RETURNFLAG].astype(np.int64), got) == 8 * 3


# ---------------------------------------------------------------- overflow
@pytest.mark.parametrize("strategy,est,sink", [(1, 3, "agg_smem_lp"), (2, 100, "agg_records")])
def test_overflow(gx, strategy, est, sink):
    """+-1e154 in X: (x - Cx)^2 overflows from finite inputs, GX_ERR_OVERFLOW.  The same values next to one infinite X
    per group give NaN, as float8_regr_accum's NaN rule makes them.  Next to one infinite Y per group they are not an
    overflow either: the device counts the inputs of both arguments (the known deviation of DESIGN.md §3.2; the
    reference raises there), so Sxx stays non-finite and corr, with Syy NaN, is NaN"""
    rng = np.random.default_rng(strategy)
    n = 100_000
    x = np.where(rng.random(n) < 0.5, 1e154, -1e154)
    grp = rng.integers(0, 3, n).astype(np.int32)
    cols = [np.zeros(n, np.int64), grp, rng.random(n), x, np.zeros(n, np.int32), np.zeros(n)]
    plan = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_REGR_SXX_F8, PAIR), (g.GX_AGG_CORR_F8, PAIR)],
                       est_groups=est, strategy=strategy)
    gx.profile(True)
    try:
        with pytest.raises(g.GxError) as e:
            gx.hash_agg(gx.table_from(OTYPES, cols), plan)
        ran = {p for p in SINKS if gx.profile_get(p)[1] > 0}
    finally:
        gx.profile(False)
    assert e.value.status == g.GX_ERR_OVERFLOW and sink in ran, (e.value, sorted(ran))
    cols[3] = x.copy()
    cols[3][[int(np.flatnonzero(grp == k)[-1]) for k in range(3)]] = np.inf         # one infinite X per group
    _, aggs, nl = gx.hash_agg(gx.table_from(OTYPES, cols), plan).fetch()
    assert np.isnan(aggs).all() and not nl.any()
    cols[3] = x
    cols[2] = cols[2].copy()
    cols[2][[int(np.flatnonzero(grp == k)[-1]) for k in range(3)]] = np.inf         # one infinite Y per group
    _, aggs, nl = gx.hash_agg(gx.table_from(OTYPES, cols), plan).fetch()
    assert not np.isfinite(aggs).any() and np.isnan(aggs[:, 1]).all() and not nl.any()


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref/libotbref.so is built only where the reference sources are present")
def test_overflow_next_to_the_reference(gx):
    """at +-1e154 in X the reference's float8_regr_accum raises too (its Sxx overflows from finite inputs): the
    reference library is run in a child process, where its ERROR is an abort"""
    import subprocess
    import sys
    code = ("import sys; sys.path[:0] = [%r, %r]; import numpy as np; import test_regr_ref_cpu as T; "
            "T.Ref().accum(np.array([1e154, -1e154] * 8), np.ones(16))") % (ROOT, os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert p.returncode != 0 and "reference ereport(ERROR)" in p.stderr, p.stderr
    cols = [np.zeros(16, np.int64), np.zeros(16, np.int32), np.ones(16), np.array([1e154, -1e154] * 8), np.zeros(16, np.int32), np.zeros(16)]
    with pytest.raises(g.GxError) as e:
        gx.hash_agg(gx.table_from(OTYPES, cols), g.make_plan(aggs=[(g.GX_AGG_REGR_SXX_F8, PAIR)], est_groups=1))
    assert e.value.status == g.GX_ERR_OVERFLOW


# ---------------------------------------------------------------- shared words, realistic sizes
def test_twins_share_one_state(gx):
    """every regression aggregate over one pair reads one state: unshared, two of them alone would need
    1 + 2 * 10 words > 18.  One pair (1 + 10) and three nullable sums (2 each) fit; a fourth does not"""
    rng = np.random.default_rng(10)
    cols, nulls = outer(rng, 200_000, 30)
    nulls[5] = (rng.random(len(cols[0])) < 0.1).astype(np.uint8)
    t = gx.table_from(OTYPES, cols, nulls)
    sums = [(g.GX_AGG_SUM_F8, F8(5)), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 5, 0), (g.GX_OP_CONST, 0, 1.0), (g.GX_OP_ADD, 0, 0)]),
            (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 5, 0), (g.GX_OP_CONST, 0, 2.0), (g.GX_OP_MUL, 0, 0)]),
            (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 5, 0), (g.GX_OP_CONST, 0, 3.0), (g.GX_OP_MUL, 0, 0)])]
    twins = [(g.GX_AGG_REGR_SLOPE_F8, PAIR), (g.GX_AGG_REGR_INTERCEPT_F8, PAIR), (g.GX_AGG_CORR_F8, PAIR), (g.GX_AGG_REGR_COUNT, PAIR)]
    plan = g.make_plan(group_cols=[(0, 1)], aggs=twins + sums[:3], est_groups=30)
    r = gx.hash_agg(t, plan)
    check(plan, cols, nulls, r.fetch())
    st = r.fetch_regr()
    assert (st[:, 0] == st[:, 1]).all() and (st[:, 1] == st[:, 2]).all() and (st[:, 3] == 0).all()
    _, _, cnts, _ = r.fetch_states()
    assert (cnts[:, 0] == cnts[:, 3]).all() and (cnts[:, 0] == st[:, 0, 0]).all()
    with pytest.raises(g.GxError) as e:
        gx.hash_agg(t, g.make_plan(group_cols=[(0, 1)], aggs=twins + sums, est_groups=30))
    assert e.value.status == g.GX_ERR_ARG and "state words" in str(e.value)


@pytest.fixture(scope="module")
def sf1(gx):
    nord = 1_500_000
    l = O.gen_lineitem(1, 0, nord)
    t = gx.table(g.SCHEMAS[g.T_LINEITEM], len(l[0])).generate(g.T_LINEITEM, 1, 0, nord)
    return l, t


def test_sf1_q1_shape(gx, sf1):
    l, t = sf1
    cut = int(np.quantile(l[g.L_SHIPDATE], 0.97))
    pair = F8(g.L_EXTENDEDPRICE) + SEP + F8(g.L_QUANTITY)
    plan = g.make_plan(preds=[(g.L_SHIPDATE, g.GX_LE, cut)], group_cols=[(0, g.L_RETURNFLAG), (0, g.L_LINESTATUS)],
                       aggs=[(g.GX_AGG_SUM_F8, F8(g.L_QUANTITY)), (g.GX_AGG_AVG_F8, F8(g.L_EXTENDEDPRICE)),
                             (g.GX_AGG_CORR_F8, pair), (g.GX_AGG_REGR_SLOPE_F8, pair), (g.GX_AGG_COVAR_SAMP_F8, pair),
                             (g.GX_AGG_COUNT_STAR, [])], est_groups=4)
    got = gx.hash_agg(t, plan).fetch()
    rows = np.flatnonzero(l[g.L_SHIPDATE] <= cut)
    key = l[g.L_RETURNFLAG].astype(np.int64) * 256 + l[g.L_LINESTATUS].astype(np.int64)
    assert R.check(plan, l, None, key, got, rows, group_key=lambda k: k[:, 0] * 256 + k[:, 1]) == 3 * 4


def test_sf1_config2_shape(gx, sf1):
    l, t = sf1
    pair = F8(g.L_EXTENDEDPRICE) + SEP + F8(g.L_DISCOUNT)
    plan = g.make_plan(group_cols=[(0, g.L_SHIPDATE)], aggs=[(g.GX_AGG_CORR_F8, pair), (g.GX_AGG_REGR_SLOPE_F8, pair),
                                                             (g.GX_AGG_AVG_F8, F8(g.L_EXTENDEDPRICE))], est_groups=2526)
    got = gx.hash_agg(t, plan).fetch()
    assert R.check(plan, l, None, l[g.L_SHIPDATE].astype(np.int64), got) > 4000


# ---------------------------------------------------------------- partial states through the reference's float8_regr_combine
@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref/libotbref.so is built only where the reference sources are present")
@pytest.mark.parametrize("strategy", [1, 2])
def test_partial_states_combine(gx, strategy):
    import test_regr_ref_cpu as T
    ref = T.Ref()
    rng = np.random.default_rng(12 + strategy)
    cols, nulls = outer(rng, 200_000, 60, loc=1e7)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_REGR_SLOPE_F8, PAIR), (g.GX_AGG_CORR_F8, PAIR), (g.GX_AGG_REGR_COUNT, PAIR)],
                       est_groups=60, strategy=strategy)
    states, counts = {}, {}
    half = len(cols[0]) // 2
    for part in (slice(0, half), slice(half, None)):
        pc = [c[part].copy() for c in cols]
        pn = [None if m is None else m[part].copy() for m in nulls]
        r = gx.hash_agg(gx.table_from(OTYPES, pc, pn), plan)
        keys, _, cnts, _ = r.fetch_states()
        st = r.fetch_regr()
        for i, k in enumerate(keys[:, 0]):
            assert (st[i, 0] == st[i, 1]).all() and st[i, 0, 0] == cnts[i, 2]
            states[int(k)] = ref.combine(states.get(int(k), [0.0] * 6), st[i, 0])
            counts[int(k)] = counts.get(int(k), 0) + int(cnts[i, 2])
    for k, s in states.items():
        sel = (cols[1] == k) & (nulls[2] == 0) & (nulls[3] == 0)
        want = R.state(cols[3][sel], cols[2][sel])
        assert s[0] == sel.sum() == counts[k] and R.state_matches(want, s), (k, s, want)
        assert R.matches(R.expect(g.GX_AGG_REGR_SLOPE_F8, cols[3][sel], cols[2][sel]), ref.final(g.GX_AGG_REGR_SLOPE_F8, s), 0)


# ---------------------------------------------------------------- refused plans
def test_arg_errors_leave_context_usable(gx):
    rng = np.random.default_rng(13)
    cols, nulls = outer(rng, 10_000, 5)
    t = gx.table_from(OTYPES, cols, nulls)
    ok = g.make_plan(group_cols=[(0, 1)], aggs=ALL[:4], est_groups=5)
    bad = {
        "no separator": [(g.GX_AGG_CORR_F8, F8(2))],
        "separator first": [(g.GX_AGG_CORR_F8, SEP + F8(2))],
        "separator last": [(g.GX_AGG_CORR_F8, F8(2) + SEP)],
        "two separators": [(g.GX_AGG_CORR_F8, F8(2) + SEP + F8(3) + SEP + F8(5))],
        "in a one-argument aggregate": [(g.GX_AGG_SUM_F8, PAIR)],
        "two pairs": [(g.GX_AGG_CORR_F8, PAIR), (g.GX_AGG_REGR_SLOPE_F8, F8(3) + SEP + F8(2))],
    }
    for name, aggs in bad.items():
        with pytest.raises(g.GxError) as e:
            gx.hash_agg(t, g.make_plan(group_cols=[(0, 1)], aggs=aggs, est_groups=5))
        assert e.value.status == g.GX_ERR_ARG, name
        check(ok, cols, nulls, gx.hash_agg(t, ok).fetch())
    # more than one rank: the Finalize across datanodes is the reference's float8_regr_combine
    parts = [gx.hash_agg(t, ok), gx.hash_agg(t, ok)]
    with pytest.raises(g.GxError) as e:
        gx.debug_combine(parts, 0)
    assert e.value.status == g.GX_ERR_ARG and "regression" in str(e.value)
    check(ok, cols, nulls, gx.hash_agg(t, ok).fetch())
