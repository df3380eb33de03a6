"""var_pop / var_samp / stddev_pop / stddev_samp over float8 (GX_AGG_VAR_POP_F8 .. GX_AGG_STDDEV_SAMP_F8) on the device.

The state is sums shifted by the group's first value, merged with re-centring wherever partial states meet.  Every
case is compared with tests/var_ref.py, an exact rational Sxx with the bound DESIGN.md §3.2 states, across every sink
of gx_k_agg (asserted by profile name), the join shapes that feed it, gx_exec_host, count(DISTINCT)'s fold, the edge
data of IEEE arithmetic, and the partial states a two-phase plan ships to the reference's float8_combine."""
import ctypes as C
import os

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import var_ref as V

pytestmark = pytest.mark.gpu

VAR_FNS = V.VAR_FNS
F8 = lambda c: [(g.GX_OP_COL, c, 0)]
SINKS = {"agg_smem", "agg_smem_lp", "agg_global", "agg_records", "agg_fewgroups", "agg_lptile8", "agg_lptile4", "runagg",
         "agg_distinct_fold", "probe_agg_exist_wide", "probe_agg_exist_compact", "probe_agg_exist_narrow",
         "probe_agg_chain_wide", "probe_agg_chain_compact", "probe_agg_chain_narrow"}
# outer columns: 0 join key int8, 1 group int4, 2 x float8 (nullable), 3 y float8, 4 int4 distinct argument
OTYPES = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8, g.GX_FLOAT8, g.GX_INT4]
ALL4 = [(fn, F8(2)) for fn in VAR_FNS]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_PATH = os.path.join(ROOT, "oracle", "_ref", "libotbref.so")
HAVE_REF = os.path.exists(REF_PATH)


def outer(rng, n, ngroups, null_frac=0.05, loc=0.0, scale=100.0, nkeys=1000):
    k = rng.integers(0, nkeys, n).astype(np.int64)
    grp = rng.integers(0, ngroups, n).astype(np.int32)
    x = loc + rng.standard_normal(n) * scale
    y = rng.random(n) * 10.0
    d = rng.integers(0, 50, n).astype(np.int32)
    nx = (rng.random(n) < null_frac).astype(np.uint8)
    return [k, grp, x, y, d], [None, None, nx, None, None]


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
    assert V.check(plan, cols, nulls, keys, got, rows) > 0


def no_join(gx, cols, nulls, plan):
    t = gx.table_from(OTYPES, cols, nulls)
    got, ran, _ = run(gx, lambda: gx.hash_agg(t, plan))
    check(plan, cols, nulls, got)
    return got, ran


# ---------------------------------------------------------------- every sink of gx_k_agg
@pytest.mark.parametrize("strategy,ngroups,est,sink", [(1, 8, 8, "agg_smem_lp"), (1, 2000, 2000, "agg_smem"),
                                                        (3, 2000, 2000, "agg_global"), (2, 50_000, 50_000, "agg_records")])
def test_sinks(gx, strategy, ngroups, est, sink):
    rng = np.random.default_rng(ngroups + strategy)
    cols, nulls = outer(rng, 400_000, ngroups)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=ALL4 + [(g.GX_AGG_AVG_F8, F8(2)), (g.GX_AGG_COUNT_STAR, [])],
                       est_groups=est, strategy=strategy)
    _, ran = no_join(gx, cols, nulls, plan)
    assert sink in ran, sorted(ran)


def test_specialised_kernels_not_taken(gx):
    """a plan the few-group, tiled and fast kernels would take without the variance goes to gx_k_agg with it"""
    rng = np.random.default_rng(1)
    cols, _ = outer(rng, 300_000, 4, null_frac=0.0)
    nulls = [None] * 5
    base = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, F8(3))]
    t = gx.table_from(OTYPES, cols, nulls)
    _, ran, _ = run(gx, lambda: gx.hash_agg(t, g.make_plan(group_cols=[(0, 1)], aggs=base, est_groups=4)))
    assert ran & {"agg_fewgroups", "agg_lptile8", "agg_lptile4"}, sorted(ran)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=base + [(g.GX_AGG_STDDEV_SAMP_F8, F8(3))], est_groups=4)
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
    ht, bt, bkeys = build(gx, fmt)
    cols, nulls = outer(rng, 300_000, 300, nkeys=200_000)
    plan = g.make_plan(outer_key_col=0, group_cols=[(0, 1)], aggs=ALL4, est_groups=300, strategy=strategy)
    plan.join_type = jt
    t = gx.table_from(OTYPES, cols, nulls)
    got, ran, _ = run(gx, lambda: gx.hash_agg(t, plan, ht))
    hit = np.isin(cols[0], bkeys)
    rows = np.flatnonzero(~hit if jt == g.GX_JOIN_ANTI else hit)
    check(plan, cols, nulls, got, rows)
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
    plan = g.make_plan(group_cols=[(0, 1)], aggs=ALL4, est_groups=100)
    t = gx.table_from(OTYPES, cols, nulls)
    got, ran, _ = run(gx, lambda: gx.hash_agg_joins(t, [(h1, (0, 0)), (h2, (0, 4))], plan))
    rows = np.flatnonzero(np.isin(cols[0], k1) & np.isin(cols[4], k2[::2]))
    check(plan, cols, nulls, got, rows)
    assert ran & {"probe_agg_chain_narrow"}, sorted(ran)


def test_exec_host(gx):
    rng = np.random.default_rng(6)
    cols, nulls = outer(rng, 200_000, 50, null_frac=0.0, nkeys=100_000)
    nulls = [None] * 5
    bkeys = np.arange(0, 100_000, 2, dtype=np.int64)
    pay = (bkeys % 5).astype(np.int32)
    plan = g.make_plan(outer_key_col=0, group_cols=[(0, 1)], aggs=ALL4 + [(g.GX_AGG_SUM_F8, F8(2))], est_groups=50)
    got = gx.exec_host(OTYPES, cols, len(cols[0]), plan, inner_types=[g.GX_INT8, g.GX_INT4], inner_ptrs=[bkeys, pay],
                       inner_nrows=len(bkeys), inner_key_col=0, payload_cols=[1], inner_unique=True).fetch()
    check(plan, cols, nulls, got, np.flatnonzero(np.isin(cols[0], bkeys)))


@pytest.mark.parametrize("strategy", [1, 2])
def test_with_count_distinct(gx, strategy):
    """stage 1 keeps a variance state per (group, value) pair; the fold re-centres them into the plan's groups"""
    rng = np.random.default_rng(7 + strategy)
    cols, nulls = outer(rng, 300_000, 40, loc=1e6)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_COUNT_DISTINCT, [(g.GX_OP_COL, 4, 0)])] + ALL4,
                       est_groups=2000, strategy=strategy)
    got, ran = no_join(gx, cols, nulls, plan)
    assert "agg_distinct_fold" in ran, sorted(ran)
    counts = got[1][:, 0].view(np.int64)
    for gi, k in enumerate(got[0][:, 0]):
        assert counts[gi] == len(np.unique(cols[4][cols[1] == k]))


# ---------------------------------------------------------------- edge data
@pytest.mark.parametrize("strategy,est,sink", [(1, 15, "agg_smem_lp"), (1, 20, "agg_smem"), (2, 20, "agg_records"),
                                               (3, 20, "agg_global")])
def test_edge_groups(gx, strategy, est, sink):
    """N = 0, 1, 2; NULL and all-NULL groups; constant groups (exactly 0); 1e9 + U(0,1); -0.0; +-Inf and NaN, the
    NaN with the unset shift's own bits among them"""
    sentinel = np.array([0x7FF4000000000001], np.uint64).view(np.float64)[0]
    rng = np.random.default_rng(strategy)
    groups = {
        0: [], 1: [3.5], 2: [1.0, 2.0], 3: [7.25] * 500, 4: list(1e9 + rng.random(2000)), 5: [-0.0] * 10 + [0.0] * 5,
        6: list(rng.random(100)) + [np.inf], 7: [np.inf, -np.inf, 1.0], 8: list(rng.random(50)) + [np.nan],
        9: [sentinel] + list(rng.random(300)), 10: list(rng.random(300)) + [sentinel], 11: [-np.inf] * 3,
        12: [sentinel] * 4, 13: [1e15] * 3 + [1e15 + 2.0],
    }
    grp, x, nx = [], [], []
    for k, vals in groups.items():
        grp += [k] * (len(vals) + 3); x += vals + [5.0] * 3; nx += [0] * len(vals) + [1] * 3    # three NULLs each
    grp += [14] * 4; x += [1.0] * 4; nx += [1] * 4                                           # all NULL
    order = rng.permutation(len(grp))
    n = len(grp)
    cols = [np.zeros(n, np.int64), np.array(grp, np.int32)[order], np.array(x)[order], np.zeros(n), np.zeros(n, np.int32)]
    nulls = [None, None, np.array(nx, np.uint8)[order], None, None]
    plan = g.make_plan(group_cols=[(0, 1)], aggs=ALL4 + [(g.GX_AGG_AVG_F8, F8(2))], est_groups=est, strategy=strategy)
    got, ran = no_join(gx, cols, nulls, plan)
    assert sink in ran, sorted(ran)
    k = list(got[0][:, 0])
    const = k.index(3)
    assert (got[1][const, :4] == 0.0).all() and not np.signbit(got[1][const, :4]).any()


def test_no_group_by_and_empty_input(gx):
    rng = np.random.default_rng(9)
    cols, nulls = outer(rng, 100_000, 1)
    no_join(gx, cols, nulls, g.make_plan(aggs=ALL4, est_groups=1))
    empty = [c[:0].copy() for c in cols]
    t = gx.table_from(OTYPES, empty, [None, None, np.zeros(0, np.uint8), None, None])
    plan = g.make_plan(aggs=ALL4 + [(g.GX_AGG_AVG_F8, F8(2))], est_groups=1)
    r = gx.hash_agg(t, plan)
    _, aggs, nl = r.fetch()
    assert nl[0].tolist() == [1, 1, 1, 1, 1]
    _, vals, cnts, snl = r.fetch_states()
    assert vals[0].tolist() == [0.0] * 5 and cnts[0].tolist() == [0] * 5 and snl[0].tolist() == [0] * 5
    assert r.fetch_sxx()[0].tolist() == [0.0] * 5


def test_expression_argument(gx):
    """stddev(l_extendedprice * (1 - l_discount)) over lineitem rows"""
    l = O.gen_lineitem(1, 0, 20_000)
    arg = [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0), (g.GX_OP_CONST, 0, 1.0), (g.GX_OP_COL, g.L_DISCOUNT, 0), (g.GX_OP_SUB, 0, 0),
           (g.GX_OP_MUL, 0, 0)]
    plan = g.make_plan(group_cols=[(0, g.L_RETURNFLAG)], aggs=[(fn, arg) for fn in VAR_FNS], est_groups=3)
    t = gx.table_from(g.SCHEMAS[g.T_LINEITEM], l)
    got = gx.hash_agg(t, plan).fetch()
    assert V.check(plan, l, None, l[g.L_RETURNFLAG].astype(np.int64), got) == 4 * 3


@pytest.mark.parametrize("strategy,est,sink", [(1, 3, "agg_smem_lp"), (1, 100, "agg_smem"), (2, 100, "agg_records"),
                                               (3, 100, "agg_global")])
@pytest.mark.parametrize("n", [1000, 1_000_000])
def test_overflow(gx, strategy, est, sink, n):
    """+-1e154 in random order: (x - C)^2 overflows from finite inputs.  Over many rows every CTA and lane holds both
    signs, and the re-centring merge of two overflowed states can end as NaN (Inf + -Inf) rather than Inf: either is
    GX_ERR_OVERFLOW.  The same values next to an infinite input give NaN."""
    rng = np.random.default_rng(n + strategy)
    x = np.where(rng.random(n) < 0.5, 1e154, -1e154)
    grp = rng.integers(0, 3, n).astype(np.int32)
    cols = [np.zeros(n, np.int64), grp, x, np.zeros(n), np.zeros(n, np.int32)]
    plan = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_VAR_POP_F8, F8(2)), (g.GX_AGG_STDDEV_SAMP_F8, F8(2))],
                       est_groups=est, strategy=strategy)
    t = gx.table_from(OTYPES, cols)
    gx.profile(True)
    try:
        with pytest.raises(g.GxError) as e:
            gx.hash_agg(t, plan)
        ran = {p for p in SINKS if gx.profile_get(p)[1] > 0}
    finally:
        gx.profile(False)
    assert e.value.status == g.GX_ERR_OVERFLOW and sink in ran, (e.value, sorted(ran))
    cols[2] = x.copy()
    cols[2][[int(np.flatnonzero(grp == k)[-1]) for k in range(3)]] = np.inf        # one infinite input per group
    _, aggs, nl = gx.hash_agg(gx.table_from(OTYPES, cols), plan).fetch()
    assert np.isnan(aggs).all() and not nl.any()


def test_overflow_deviation_next_to_the_oracle(gx):
    """DESIGN.md §3.2: the device decides an overflow on Sx, S1 and S2, the reference on its own N x - Sx and Sxx
    (float.c:2846).  At +-1e154 both raise.  Where the first value lies far from the others, S2 = sum((x - x0)^2)
    overflows while the reference's Sxx, about S2 / N, does not: the device raises and the reference returns a
    variance.  32 rows take one warp of one CTA, whose lane 0 holds the first row, so the shift is x0 = 0."""
    plan = g.make_plan(aggs=[(g.GX_AGG_VAR_SAMP_F8, F8(2))], est_groups=1, strategy=1)
    oplan = O.make_plan(aggs=[(g.GX_AGG_AVG_F8, [(g.GX_OP_COL, 1, 0)])])
    both = np.array([1e154, -1e154] * 8)
    with pytest.raises(RuntimeError, match="status 6"):
        O.exec_agg(O.Rel([O.GX_INT8, O.GX_FLOAT8], [np.zeros(len(both), np.int64), both]), oplan)
    cols = [np.zeros(len(both), np.int64), np.zeros(len(both), np.int32), both, np.zeros(len(both)), np.zeros(len(both), np.int32)]
    with pytest.raises(g.GxError) as e:
        gx.hash_agg(gx.table_from(OTYPES, cols), plan)
    assert e.value.status == g.GX_ERR_OVERFLOW
    apart = np.array([0.0] + [3.2e153] * 31)
    st = O.exec_agg(O.Rel([O.GX_INT8, O.GX_FLOAT8], [np.zeros(32, np.int64), apart]), oplan).states[0, 0]
    assert st[0] == 32 and np.isfinite(st[2]) and abs(st[2] - float(V.sxx_exact(apart))) <= 1e-12 * st[2]
    cols = [np.zeros(32, np.int64), np.zeros(32, np.int32), apart, np.zeros(32), np.zeros(32, np.int32)]
    with pytest.raises(g.GxError) as e:
        gx.hash_agg(gx.table_from(OTYPES, cols), plan)
    assert e.value.status == g.GX_ERR_OVERFLOW


# ---------------------------------------------------------------- shared words, realistic sizes
def test_avg_and_stddev_share_the_sum(gx):
    rng = np.random.default_rng(10)
    cols, nulls = outer(rng, 200_000, 30)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_AVG_F8, F8(2)), (g.GX_AGG_STDDEV_SAMP_F8, F8(2)),
                                                  (g.GX_AGG_SUM_F8, F8(2)), (g.GX_AGG_VAR_POP_F8, F8(2))], est_groups=30)
    t = gx.table_from(OTYPES, cols, nulls)
    r = gx.hash_agg(t, plan)
    got = r.fetch()
    check(plan, cols, nulls, got)
    _, vals, cnts, _ = r.fetch_states()
    assert (vals[:, 0] == vals[:, 1]).all() and (vals[:, 1] == vals[:, 2]).all() and (vals[:, 2] == vals[:, 3]).all()
    assert (cnts[:, 0] == cnts[:, 1]).all() and (cnts[:, 0] == cnts[:, 3]).all()
    sxx = r.fetch_sxx()
    assert (sxx[:, 1] == sxx[:, 3]).all() and (sxx[:, 0] == 0).all() and (sxx[:, 2] == 0).all()


@pytest.fixture(scope="module")
def sf1(gx):
    nord = 1_500_000
    l = O.gen_lineitem(1, 0, nord)
    t = gx.table(g.SCHEMAS[g.T_LINEITEM], len(l[0])).generate(g.T_LINEITEM, 1, 0, nord)
    return l, t


def test_sf1_q1_shape(gx, sf1):
    l, t = sf1
    cut = int(np.quantile(l[g.L_SHIPDATE], 0.97))
    disc = [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0), (g.GX_OP_CONST, 0, 1.0), (g.GX_OP_COL, g.L_DISCOUNT, 0), (g.GX_OP_SUB, 0, 0),
            (g.GX_OP_MUL, 0, 0)]
    plan = g.make_plan(preds=[(g.L_SHIPDATE, g.GX_LE, cut)], group_cols=[(0, g.L_RETURNFLAG), (0, g.L_LINESTATUS)],
                       aggs=[(g.GX_AGG_SUM_F8, F8(g.L_QUANTITY)), (g.GX_AGG_AVG_F8, F8(g.L_EXTENDEDPRICE)),
                             (g.GX_AGG_STDDEV_SAMP_F8, F8(g.L_EXTENDEDPRICE)), (g.GX_AGG_VAR_POP_F8, disc),
                             (g.GX_AGG_COUNT_STAR, [])], est_groups=4)
    got = gx.hash_agg(t, plan).fetch()
    rows = np.flatnonzero(l[g.L_SHIPDATE] <= cut)
    key = l[g.L_RETURNFLAG].astype(np.int64) * 256 + l[g.L_LINESTATUS].astype(np.int64)
    assert V.check(plan, l, None, key, got, rows, group_key=lambda k: k[:, 0] * 256 + k[:, 1]) == 2 * 4


def test_sf1_config2_shape(gx, sf1):
    l, t = sf1
    plan = g.make_plan(group_cols=[(0, g.L_SHIPDATE)], aggs=[(g.GX_AGG_STDDEV_SAMP_F8, F8(g.L_EXTENDEDPRICE)),
                                                             (g.GX_AGG_AVG_F8, F8(g.L_EXTENDEDPRICE))], est_groups=2526)
    got = gx.hash_agg(t, plan).fetch()
    assert V.check(plan, l, None, l[g.L_SHIPDATE].astype(np.int64), got) > 2000


# ---------------------------------------------------------------- partial states through the reference's float8_combine
@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref/libotbref.so is built only where the reference sources are present")
@pytest.mark.parametrize("strategy", [1, 2])
def test_partial_states_combine(gx, strategy):
    R = C.CDLL(REF_PATH)
    R.ref_float8_combine.argtypes = [C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(12 + strategy)
    cols, nulls = outer(rng, 200_000, 60, loc=1e7)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_VAR_SAMP_F8, F8(2)), (g.GX_AGG_STDDEV_POP_F8, F8(2))],
                       est_groups=60, strategy=strategy)
    states = {}
    half = len(cols[0]) // 2
    for part in (slice(0, half), slice(half, None)):
        pc = [c[part].copy() for c in cols]
        pn = [None if m is None else m[part].copy() for m in nulls]
        r = gx.hash_agg(gx.table_from(OTYPES, pc, pn), plan)
        keys, vals, cnts, _ = r.fetch_states()
        sxx = r.fetch_sxx()
        for i, k in enumerate(keys[:, 0]):
            s2 = np.array([cnts[i, 0], vals[i, 0], sxx[i, 0]], np.float64)
            assert cnts[i, 0] == cnts[i, 1] and vals[i, 0] == vals[i, 1] and sxx[i, 0] == sxx[i, 1]
            s1 = states.setdefault(int(k), np.zeros(3))
            R.ref_float8_combine(s1.ctypes.data, s2.ctypes.data)
    for k, s in states.items():
        x = cols[2][(cols[1] == k) & (nulls[2] == 0)]
        assert s[0] == len(x)
        assert V.sxx_matches(x, s[2]), (k, s, float(V.sxx_exact(x)))


# ---------------------------------------------------------------- refused plans
def test_arg_errors_leave_context_usable(gx):
    rng = np.random.default_rng(13)
    cols, nulls = outer(rng, 10_000, 5)
    t = gx.table_from(OTYPES, cols, nulls)
    ok = g.make_plan(group_cols=[(0, 1)], aggs=ALL4, est_groups=5)
    # four variances over four different nullable arguments: 1 + 4 * 5 state words > GX_MAX_WORDS
    args = [F8(2), [(g.GX_OP_COL, 2, 0), (g.GX_OP_CONST, 0, 1.0), (g.GX_OP_ADD, 0, 0)],
            [(g.GX_OP_COL, 2, 0), (g.GX_OP_CONST, 0, 2.0), (g.GX_OP_MUL, 0, 0)], [(g.GX_OP_COL, 2, 0), (g.GX_OP_COL, 3, 0), (g.GX_OP_ADD, 0, 0)]]
    too_many = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_VAR_POP_F8, a) for a in args], est_groups=5)
    with pytest.raises(g.GxError) as e:
        gx.hash_agg(t, too_many)
    assert e.value.status == g.GX_ERR_ARG and "state words" in str(e.value)
    check(ok, cols, nulls, gx.hash_agg(t, ok).fetch())
    # three of them fit: 1 + 3 * 5 words
    three = g.make_plan(group_cols=[(0, 1)], aggs=[(g.GX_AGG_VAR_POP_F8, a) for a in args[:3]], est_groups=5)
    check(three, cols, nulls, gx.hash_agg(t, three).fetch())
