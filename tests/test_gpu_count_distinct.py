"""count(DISTINCT col) (GX_AGG_COUNT_DISTINCT) on the device: the plan aggregated with col as one more group column,
then folded back into the plan's own groups (profile name agg_distinct_fold).

Every case is compared with tests/distinct_ref.py: distinct counts and integer aggregates bit for bit, float8 within
the bounds tests/exact_ref.py derives for the summation order.  Stage 1 takes whatever kernel the plan with the extra
group column takes, so the routes below are asserted by their profile names next to the fold's."""
import numpy as np
import pytest

import opentenbase_b200 as g
import distinct_ref as D
import join_ref as J
import star_ref as S

pytestmark = pytest.mark.gpu

I64, I32 = np.iinfo(np.int64), np.iinfo(np.int32)
CD = g.GX_AGG_COUNT_DISTINCT
# outer columns: 0 join key int8, 1 group int4, 2 x float8, 3 int4 arg, 4 int8 arg, 5 date arg, 6 char arg, 7 int4 v
OTYPES = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8, g.GX_INT4, g.GX_INT8, g.GX_DATE, g.GX_CHAR, g.GX_INT4]
ARG = {"int4": 3, "int8": 4, "date": 5, "char": 6}
NAMES = {"agg_distinct_fold", "agg", "probe_agg", "probe_agg_chain", "agg_smem", "agg_smem_lp", "agg_global", "agg_records",
         "agg_fewgroups", "agg_count_char", "agg_lptile8", "agg_lptile4", "runagg", "probe_agg_exist_wide", "probe_agg_exist_compact",
         "probe_agg_exist_narrow", "probe_agg_chain_wide", "probe_agg_chain_compact", "probe_agg_chain_narrow"}
SEEN = set()                      # route names that answered in this module


def outer(rng, n, ngroups, nvals, null_frac=0.05, keys=None, gnull=False):
    """n rows: group in [0, ngroups), every argument column with nvals distinct values plus its type's edge values, and
    NULLs in the arguments (and the group column when gnull)"""
    k = np.asarray(keys if keys is not None else rng.integers(0, 1000, n), np.int64)
    grp = rng.integers(0, ngroups, n).astype(np.int32)
    x = rng.standard_normal(n) * 100.0
    base = rng.integers(0, nvals, n)
    a4 = (base * 7919 - nvals * 3000).astype(np.int64)
    a8 = (base * 1_000_000_007 - 2**62).astype(np.int64)
    edge = rng.random(n) < 0.02
    a4 = np.where(edge, np.where(rng.random(n) < 0.5, I32.min, I32.max), a4).astype(np.int32)
    a8 = np.where(edge, np.where(rng.random(n) < 0.5, I64.min, I64.max), a8).astype(np.int64)
    ad = (base % 3000 - 1500).astype(np.int32)
    ac = (base % 256 - 128).astype(np.int8)
    v = rng.integers(-1000, 1000, n).astype(np.int32)
    cols = [k, grp, x, a4, a8, ad, ac, v]
    nl = lambda: (rng.random(n) < null_frac).astype(np.uint8)
    nulls = [None, nl() if gnull else None, None, nl(), nl(), nl(), nl(), None]
    return cols, nulls


def mixed(arg, extra=True):
    aggs = [(CD, [(g.GX_OP_COL, ARG[arg], 0)])]
    if extra:
        aggs += [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_COUNT, [(g.GX_OP_COL, ARG[arg], 0)]), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)]),
                 (g.GX_AGG_AVG_F8, [(g.GX_OP_COL, 2, 0)]), (g.GX_AGG_MIN_F8, [(g.GX_OP_COL, 2, 0)]),
                 (g.GX_AGG_MAX_F8, [(g.GX_OP_COL, 2, 0)]), (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 7, 0)])]
    return aggs


def run(gx, fn):
    gx.profile(True)
    try:
        got = fn().fetch()
        ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
    finally:
        gx.profile(False)
    assert "agg_distinct_fold" in ran, sorted(ran)
    SEEN.update(ran)
    return got, ran


def gtypes(plan, types):
    return [types[plan.group_cols[c].col] for c in range(plan.n_group_cols)]


def no_join(gx, cols, nulls, plan, types=OTYPES):
    ot = gx.table_from(types, cols, nulls)
    got, ran = run(gx, lambda: gx.hash_agg(ot, plan))
    preds = [(plan.preds[p].col, plan.preds[p].op, plan.preds[p].fval if types[plan.preds[p].col] == g.GX_FLOAT8 else plan.preds[p].ival)
             for p in range(plan.n_preds)]
    o = np.flatnonzero(J.quals(cols, nulls, preds, len(cols[0])))
    want = D.expect_groups(plan, cols, types, o, nulls)
    D.check(plan, want, got, gtypes(plan, types))
    ot.free()
    return got, ran


# ---------------------------------------------------------------- no join: argument types, kernels, strategies
@pytest.mark.parametrize("arg", list(ARG))
@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
def test_no_join_types_and_strategies(gx, arg, strategy):
    rng = np.random.default_rng(strategy * 10 + len(arg))
    cols, nulls = outer(rng, 200_000, 50, 400, gnull=True)
    plan = g.make_plan(preds=[(2, g.GX_LT, 150.0, True)], group_cols=[(0, 1)], aggs=mixed(arg), est_groups=20_000, strategy=strategy)
    _, ran = no_join(gx, cols, nulls, plan)
    want = {1: {"agg_smem", "agg_smem_lp"}, 2: {"agg_records"}, 3: {"agg_global"}}.get(strategy)
    if want:
        assert ran & want, sorted(ran)


def test_few_groups_kernel(gx):
    """few (group, value) pairs without NULLs: stage 1 is the register-accumulator kernel"""
    rng = np.random.default_rng(3)
    cols, nulls = outer(rng, 300_000, 2, 3, null_frac=0.0)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=[(CD, [(g.GX_OP_COL, 6, 0)]), (g.GX_AGG_COUNT_STAR, []),
                                                  (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)])], est_groups=6)
    _, ran = no_join(gx, cols, [None] * 8, plan)
    assert "agg_fewgroups" in ran, sorted(ran)
    # an int4 sum keeps the same few pairs off the register kernels: the lane-private shared-memory sink
    _, ran = no_join(gx, cols, [None] * 8, g.make_plan(group_cols=[(0, 1)], aggs=mixed("char"), est_groups=6))
    assert "agg_smem_lp" in ran, sorted(ran)


def test_count_char_kernel(gx):
    """no GROUP BY, a NOT NULL "char" argument with a few values and count(*): stage 1 is gx_k_count_char"""
    rng = np.random.default_rng(5)
    cols, _ = outer(rng, 300_000, 1, 6, null_frac=0.0)
    _, ran = no_join(gx, cols, [None] * 8, g.make_plan(aggs=[(CD, [(g.GX_OP_COL, 6, 0)]), (g.GX_AGG_COUNT_STAR, [])], est_groups=6))
    assert "agg_count_char" in ran, sorted(ran)


@pytest.mark.parametrize("arg", list(ARG))
def test_no_group_by(gx, arg):
    rng = np.random.default_rng(7)
    cols, nulls = outer(rng, 100_000, 1, 5000)
    no_join(gx, cols, nulls, g.make_plan(aggs=mixed(arg), est_groups=5000))


def test_nulls_all_null_groups_and_null_keys(gx):
    """groups whose arguments are all NULL count 0; a NULL group key is a group of its own"""
    rng = np.random.default_rng(11)
    cols, nulls = outer(rng, 50_000, 20, 100, null_frac=0.3, gnull=True)
    for c in (3, 4, 5, 6):
        nulls[c][cols[1] < 4] = 1                      # groups 0..3: every argument NULL
    for arg in ARG:
        got, _ = no_join(gx, cols, nulls, g.make_plan(group_cols=[(0, 1)], aggs=mixed(arg), est_groups=2000))
        keys, aggs, nl = got
        zero = (keys[:, 0] < 4) & (nl[:, 0] == 0)
        assert zero.sum() == 4 and (aggs[zero, 0].view(np.int64) == 0).all()


@pytest.mark.parametrize("grouped", [True, False])
def test_empty_input_and_quals_removing_every_row(gx, grouped):
    rng = np.random.default_rng(13)
    gc = [(0, 1)] if grouped else []
    cols, nulls = outer(rng, 10_000, 10, 100)
    for preds in ([(2, g.GX_GT, 1e300, True)], []):
        c = cols if preds else [x[:0] for x in cols]
        nl = nulls if preds else [None if x is None else x[:0] for x in nulls]
        got, _ = no_join(gx, c, nl, g.make_plan(preds=preds, group_cols=gc, aggs=mixed("int8"), est_groups=100))
        assert got[0].shape[0] == (0 if grouped else 1)


def test_one_pair_per_row_sf1(gx):
    """lineitem at SF1: count(DISTINCT l_orderkey) GROUP BY l_shipdate, close to one pair per row"""
    t = gx.table(g.SCHEMAS[g.T_LINEITEM], 7_000_000).generate(g.T_LINEITEM, 1, 0, 1_500_000)
    cols = [t.read(c) for c in range(len(g.SCHEMAS[g.T_LINEITEM]))]
    plan = g.make_plan(group_cols=[(0, g.L_SHIPDATE)], aggs=[(CD, [(g.GX_OP_COL, g.L_ORDERKEY, 0)]), (g.GX_AGG_COUNT_STAR, []),
                                                             (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, g.L_QUANTITY, 0)])], est_groups=len(cols[0]))
    got, _ = run(gx, lambda: gx.hash_agg(t, plan))
    D.check(plan, D.expect_groups(plan, cols, g.SCHEMAS[g.T_LINEITEM], np.arange(len(cols[0]))), got, [g.GX_DATE])
    t.free()


def test_sf10_slice(gx):
    """an SF10 slice of orders: count(DISTINCT o_custkey) GROUP BY o_orderdate"""
    t = gx.table(g.SCHEMAS[g.T_ORDERS], 2_000_000).generate(g.T_ORDERS, 10, 3_000_000, 5_000_000)
    cols = [t.read(c) for c in range(4)]
    plan = g.make_plan(group_cols=[(0, g.O_ORDERDATE)], aggs=[(CD, [(g.GX_OP_COL, g.O_CUSTKEY, 0)]), (g.GX_AGG_COUNT_STAR, [])],
                       est_groups=len(cols[0]))
    got, _ = run(gx, lambda: gx.hash_agg(t, plan))
    D.check(plan, D.expect_groups(plan, cols, g.SCHEMAS[g.T_ORDERS], np.arange(len(cols[0]))), got, [g.GX_DATE])
    t.free()


# ---------------------------------------------------------------- joins
def bunched(n):
    i = np.arange(n, dtype=np.int64)
    return (i // 8) * 32 + (i % 8) + 1


def build(gx, fmt, keys, pay):
    t = gx.table_from([g.GX_INT8, g.GX_INT4], [keys, pay])
    ht = gx.hash_build(t, 0, [] if fmt == "compact" else [1], unique=True)
    return ht, t


@pytest.mark.parametrize("fmt", ["wide", "compact", "narrow"])
@pytest.mark.parametrize("jt", [g.GX_JOIN_INNER, g.GX_JOIN_SEMI, g.GX_JOIN_ANTI])
def test_join_types_and_slot_formats(gx, fmt, jt):
    rng = np.random.default_rng(17)
    bkeys = bunched(50_000)
    if fmt == "wide":
        bkeys = rng.permutation(bkeys)
    pay = (bkeys % 97).astype(np.int32)
    ht, bt = build(gx, fmt, bkeys, pay)
    okeys = np.where(rng.random(200_000) < 0.7, rng.choice(bkeys, 200_000), rng.integers(0, 2_000_000, 200_000))
    cols, nulls = outer(rng, 200_000, 30, 300, keys=okeys)
    gc = [(1, 0)] if jt == g.GX_JOIN_INNER and fmt != "compact" else [(0, 1)]
    plan = g.make_plan(preds=[(2, g.GX_LT, 200.0, True)], outer_key_col=0, group_cols=gc, aggs=mixed("int4"),
                       est_groups=5000, join_type=jt)
    ot = gx.table_from(OTYPES, cols, nulls)
    got, ran = run(gx, lambda: gx.hash_agg(ot, plan, ht))
    keep = J.quals(cols, nulls, [(2, g.GX_LT, 200.0, True)], len(okeys))
    o, i = J.join(jt, okeys, bkeys, okeep=keep)
    sides = {1: ([pay[i]], [g.GX_INT4])} if gc[0][0] == 1 else None
    want = D.expect_groups(plan, cols, OTYPES, o, nulls, sides)
    D.check(plan, want, got, [g.GX_INT4])
    if jt != g.GX_JOIN_INNER:
        assert {"probe_agg_exist_wide", "probe_agg_exist_compact", "probe_agg_exist_narrow"} & ran, sorted(ran)
    ot.free(); ht.free(); bt.free()


def test_run_aggregate_route(gx):
    """count(DISTINCT join key) GROUP BY a payload column over a key-ordered outer side: stage 1 is gx_k_runagg"""
    rng = np.random.default_rng(19)
    bkeys = bunched(100_000)
    pay = (bkeys % 2406 - 1000).astype(np.int32)
    ht, bt = build(gx, "narrow", bkeys, pay)
    okeys = np.sort(rng.choice(bkeys, 600_000))
    x = rng.standard_normal(600_000)
    ot = gx.table_from([g.GX_INT8, g.GX_FLOAT8], [okeys, x])
    plan = g.make_plan(outer_key_col=0, group_cols=[(1, 0)], aggs=[(CD, [(g.GX_OP_COL, 0, 0)]), (g.GX_AGG_COUNT_STAR, []),
                                                                    (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])], est_groups=100_000)
    got, ran = run(gx, lambda: gx.hash_agg(ot, plan, ht))
    assert "runagg" in ran, sorted(ran)
    o, i = J.join(g.GX_JOIN_INNER, okeys, bkeys)
    want = D.expect_groups(plan, [okeys, x], [g.GX_INT8, g.GX_FLOAT8], o, None, {1: ([pay[i]], [g.GX_INT4])})
    D.check(plan, want, got, [g.GX_INT4])
    ot.free(); ht.free(); bt.free()


@pytest.mark.parametrize("nsteps", [2, 3])
def test_join_chains(gx, nsteps):
    rng = np.random.default_rng(23 + nsteps)
    d1k = rng.permutation(bunched(20_000)); d1p = (d1k % 5000).astype(np.int32)
    d2k = np.arange(5000, dtype=np.int64); d2p = (d2k % 41).astype(np.int32)
    d3k = np.arange(41, dtype=np.int64); d3p = (d3k % 7).astype(np.int32)
    hts = []
    for k, p in ((d1k, d1p), (d2k, d2p), (d3k, d3p))[:nsteps]:
        t = gx.table_from([g.GX_INT8, g.GX_INT4], [k, p])
        hts.append((gx.hash_build(t, 0, [1], unique=True), t))
    okeys = np.where(rng.random(150_000) < 0.8, rng.choice(d1k, 150_000), -5)
    cols, nulls = outer(rng, 150_000, 10, 500, keys=okeys)
    steps = [(hts[0][0], (0, 0)), (hts[1][0], (1, 0))] + ([(hts[2][0], (2, 0))] if nsteps == 3 else [])
    plan = g.make_plan(preds=[(2, g.GX_GT, -250.0, True)], group_cols=[(nsteps, 0), (0, 1)], aggs=mixed("date"), est_groups=20_000)
    ot = gx.table_from(OTYPES, cols, nulls)
    got, ran = run(gx, lambda: gx.hash_agg_joins(ot, steps, plan))
    assert "probe_agg_chain" in ran, sorted(ran)
    ref = [S.Step((0, 0), d1k, [d1p], [g.GX_INT4]), S.Step((1, 0), d2k, [d2p], [g.GX_INT4]), S.Step((2, 0), d3k, [d3p], [g.GX_INT4])][:nsteps]
    o, brows = S.chain_rows(plan, cols, OTYPES, ref, nulls)
    side = ref[nsteps - 1]
    want = D.expect_groups(plan, cols, OTYPES, o, nulls, {nsteps: ([side.payload[0][brows[-1]]], [g.GX_INT4])})
    D.check(plan, want, got, [g.GX_INT4, g.GX_INT4])
    ot.free()
    for ht, t in hts:
        ht.free(); t.free()


def test_exec_host(gx):
    rng = np.random.default_rng(29)
    bkeys = rng.permutation(bunched(30_000)); pay = (bkeys % 53).astype(np.int32)
    okeys = rng.choice(bkeys, 100_000)
    cols, _ = outer(rng, 100_000, 10, 700, keys=okeys)
    plan = g.make_plan(outer_key_col=0, group_cols=[(1, 0)], aggs=mixed("int8"), est_groups=5000)
    got, _ = run(gx, lambda: gx.exec_host(OTYPES, cols, len(okeys), plan, inner_types=[g.GX_INT8, g.GX_INT4], inner_ptrs=[bkeys, pay],
                                         inner_nrows=len(bkeys), inner_key_col=0, payload_cols=[1], inner_unique=True))
    o, i = J.join(g.GX_JOIN_INNER, okeys, bkeys)
    D.check(plan, D.expect_groups(plan, cols, OTYPES, o, None, {1: ([pay[i]], [g.GX_INT4])}), got, [g.GX_INT4])


# ---------------------------------------------------------------- key width, overflow, declines
def test_key_width_16_bytes_accepted_17_declined(gx):
    rng = np.random.default_rng(31)
    cols, nulls = outer(rng, 20_000, 10, 50)
    # int8 group (k0) + int4 group + int4 argument (k1): 16 bytes
    plan = g.make_plan(group_cols=[(0, 4), (0, 1)], aggs=mixed("int4"), est_groups=20_000)
    no_join(gx, cols, nulls, plan)
    # int8 + int4 + char groups, int4 argument: 17 bytes
    bad = g.make_plan(group_cols=[(0, 4), (0, 1), (0, 6)], aggs=mixed("int4"), est_groups=20_000)
    ot = gx.table_from(OTYPES, cols, nulls)
    with pytest.raises(g.GxError) as e:
        gx.hash_agg(ot, bad)
    assert e.value.status == g.GX_ERR_ARG
    ot.free()
    no_join(gx, cols, nulls, plan)                  # the context answers the next call


def test_fold_overflow(gx):
    """two pairs of one group each sum to a finite 1.5e308: the fold's sum overflows, and no input was infinite"""
    n = 4
    cols = [np.zeros(n, np.int64), np.zeros(n, np.int32), np.full(n, 0.75e308), np.array([1, 1, 2, 2], np.int32),
            np.zeros(n, np.int64), np.zeros(n, np.int32), np.zeros(n, np.int8), np.zeros(n, np.int32)]
    ot = gx.table_from(OTYPES, cols)
    plan = g.make_plan(group_cols=[(0, 1)], aggs=[(CD, [(g.GX_OP_COL, 3, 0)]), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)])], est_groups=4)
    with pytest.raises(g.GxError) as e:
        gx.hash_agg(ot, plan)
    assert e.value.status == g.GX_ERR_OVERFLOW
    cols[2] = np.array([0.75e308, np.inf, 0.75e308, 0.75e308])   # an infinite input: an infinite sum is the answer
    ot2 = gx.table_from(OTYPES, cols)
    got = gx.hash_agg(ot2, plan).fetch()
    assert got[1][0, 1] == np.inf and got[1][0:1, 0].view(np.int64)[0] == 2
    ot.free(); ot2.free()


def test_argument_errors_leave_the_context_usable(gx):
    rng = np.random.default_rng(37)
    cols, nulls = outer(rng, 5000, 5, 50)
    ot = gx.table_from(OTYPES, cols, nulls)
    good = g.make_plan(group_cols=[(0, 1)], aggs=mixed("char"), est_groups=300)
    bad = [
        g.make_plan(group_cols=[(0, 1)], aggs=[(CD, [(g.GX_OP_COL, 2, 0)])]),                                       # float8
        g.make_plan(group_cols=[(0, 1)], aggs=[(CD, [(g.GX_OP_COL, 3, 0), (g.GX_OP_CONST, 0, 1.0), (g.GX_OP_ADD, 0, 0)])]),
        g.make_plan(group_cols=[(0, 1)], aggs=[(CD, [(g.GX_OP_COL, 3, 0)]), (CD, [(g.GX_OP_COL, 4, 0)])]),        # two columns
        g.make_plan(group_cols=[(0, 1), (0, 3), (0, 5), (0, 6)], aggs=[(CD, [(g.GX_OP_COL, 4, 0)])]),             # no slot left
        g.make_plan(group_cols=[(0, 1)], aggs=[(CD, [(g.GX_OP_COL, 99, 0)])]),                                      # out of range
    ]
    for p in bad:
        with pytest.raises(g.GxError) as e:
            gx.hash_agg(ot, p)
        assert e.value.status == g.GX_ERR_ARG
        r = gx.hash_agg(ot, good)
        assert r.ngroups > 0
        r.free()
    # the same column twice is one DISTINCT word
    two = g.make_plan(group_cols=[(0, 1)], aggs=[(CD, [(g.GX_OP_COL, 3, 0)]), (CD, [(g.GX_OP_COL, 3, 0)])], est_groups=300)
    got = gx.hash_agg(ot, two).fetch()
    assert (got[1][:, 0].view(np.int64) == got[1][:, 1].view(np.int64)).all()
    # no partial states to fetch
    r = gx.hash_agg(ot, good)
    with pytest.raises(g.GxError) as e:
        r.fetch_states()
    assert e.value.status == g.GX_ERR_ARG
    r.combine()                                     # one rank: a no-op
    r.fetch()
    r.free(); ot.free()


def test_every_route_ran():
    """the stage-1 routes this module exercises each answered at least once, each with the fold"""
    want = {"agg_smem", "agg_smem_lp", "agg_records", "agg_global", "agg_fewgroups", "agg_count_char", "runagg", "probe_agg_chain",
            "probe_agg_exist_wide", "probe_agg_exist_compact", "probe_agg_exist_narrow", "agg_distinct_fold"}
    if not SEEN:
        pytest.skip("needs the cases of this module")
    assert want <= SEEN, sorted(want - SEEN)
