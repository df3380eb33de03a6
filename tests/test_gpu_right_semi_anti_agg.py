"""Aggregates over right semi and right anti hash joins (gx_hash_agg_right): the marking probe gx_k_probe_mark (a unique
table read in the wide or compact form its build wrote, a non-unique one walked in its 16-byte form), the compaction of
the consumed build rows by gx_k_filter_onepass, and the ordinary aggregate over them.

Every case is compared exactly against tests/right_ref.py (join_ref's SEMI / ANTI with the build side as the outer side,
aggregated by exact_ref): counts and integer sums bit for bit, float8 within the bounds exact_ref derives.  The profile
names probe_mark_wide / _compact / _walk tell which marking probe ran."""
import os
import tempfile

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import join_ref as J
import right_ref as R
import var_ref as V
import regr_ref as RG
import distinct_ref as D
from test_gpu_semi_anti_agg import skewed

pytestmark = pytest.mark.gpu

I64, I32 = np.iinfo(np.int64), np.iinfo(np.int32)
SEMI_R, ANTI_R = g.GX_JOIN_SEMI_RIGHT, g.GX_JOIN_ANTI_RIGHT
JTS = (SEMI_R, ANTI_R)
FORM = {"wide": "probe_mark_wide", "compact": "probe_mark_compact", "walk": "probe_mark_walk"}
NAMES = set(FORM.values()) | {"probe_mark", "filter", "filter_marked", "agg_fewgroups", "agg_smem_lp", "agg_fast", "agg_smem",
                              "agg_global", "agg_records", "agg_lptile4", "agg_lptile8", "build_expand"}
SEEN = set()
# build side: key, group (int4), x (float8, NULLs), i (int4), d (date)
BTYPES = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8, g.GX_INT4, g.GX_DATE]
PTYPES = [g.GX_INT8, g.GX_INT4]          # probe side: key, qual column


def base_plan(grouped=True, est=0, preds=(), aggs=None):
    aggs = aggs or [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_COUNT, [(g.GX_OP_COL, 2, 0)]), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)]),
                    (g.GX_AGG_AVG_F8, [(g.GX_OP_COL, 2, 0)]), (g.GX_AGG_MIN_F8, [(g.GX_OP_COL, 2, 0)]),
                    (g.GX_AGG_MAX_F8, [(g.GX_OP_COL, 2, 0)]), (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 3, 0)])]
    return g.make_plan(preds=list(preds), group_cols=[(0, 1)] if grouped else [], aggs=aggs, est_groups=est)


def build_cols(rng, keys, ngroups=50, xnull=0.1, special=True):
    n = len(keys)
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)
    if special and n >= 8:
        x[rng.choice(n, 3, replace=False)] = [np.inf, -np.inf, np.nan]
    cols = [keys, rng.integers(0, ngroups, n).astype(np.int32), x, rng.integers(-1000, 1000, n).astype(np.int32),
            rng.integers(-3000, 3000, n).astype(np.int32)]
    nulls = [None, None, (rng.random(n) < xnull).astype(np.uint8), None, None]
    return cols, nulls


def build_keys(form, n=120_000, seed=0):
    """key-ordered unique int8 keys give the compact table, the same keys shuffled the 16-byte one; every third key
    twice (non-unique) is walked"""
    i = np.arange(n, dtype=np.int64)
    keys = (i // 8) * 32 + (i % 8) + 1
    if form == "walk":
        keys = np.sort(np.concatenate([keys, keys[::3]]))
    if form != "compact":
        keys = np.random.default_rng(seed).permutation(keys)
    return keys


def run(gx, pt, bt, ht, jt, plan, pkey_col=0, ppreds=()):
    gx.profile(True)
    try:
        got = gx.hash_agg_right(pt, pkey_col, bt, ht, jt, plan, probe_preds=ppreds).fetch()
    finally:
        ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
        gx.profile(False)
    SEEN.update(ran)
    return got, ran


def check(gx, pt, bt, ht, jt, plan, bcols, bnulls, pcols, pnulls=None, ppreds=(), bpreds=(), btypes=BTYPES, ptypes=PTYPES,
          gtypes=None):
    pnulls = pnulls or [None] * len(pcols)
    pkeep = J.quals(pcols, pnulls, list(ppreds), len(pcols[0]))
    want = R.expect_right_groups(plan, jt, bcols, btypes, 0, pcols[0], bnulls, pnulls[0], pkeep, bpreds)
    got, ran = run(gx, pt, bt, ht, jt, plan, ppreds=ppreds)
    if gtypes is None:
        gtypes = [btypes[plan.group_cols[c].col] for c in range(plan.n_group_cols)]
    X.check(plan, want, got, gtypes)
    return got, ran, want


# ---------------------------------------------------------------- marking probe forms x probe sides
PROBES = ["ordered", "shuffled", "descending", "ragged", "one", "empty", "filtered", "all_miss", "all_hit"]


def probe_side(rng, kind, bkeys):
    """probe keys of the given shape (about four rows per build key where they hit, as lineitem has per order)"""
    ks = np.sort(np.unique(bkeys))
    if kind == "empty":
        k = np.zeros(0, np.int64)
    elif kind == "one":
        k = np.array([ks[len(ks) // 2]], np.int64)
    elif kind == "all_miss":
        k = rng.choice(ks, 50_000) + 9                               # between the bunches: no build key
    elif kind == "all_hit":
        k = np.repeat(ks, 4)
    else:
        k = np.concatenate([np.repeat(rng.choice(ks, len(ks) // 3, replace=False), rng.integers(1, 8, len(ks) // 3)),
                            rng.choice(ks, 20_000) + 9, rng.integers(-10**6, 10**7, 5000)])
        if kind == "ragged":
            k = k[:32 * 4 * (len(k) // 128) + 37]
    if kind in ("ordered", "ragged", "filtered", "all_hit", "all_miss"):
        k = np.sort(k)
    elif kind == "descending":
        k = np.sort(k)[::-1].copy()
    else:
        k = rng.permutation(k)
    q = rng.integers(0, 10, len(k)).astype(np.int32)
    ppreds = [(1, g.GX_GE, 10)] if kind == "filtered" else [(1, g.GX_LT, 8)] if kind in ("shuffled", "ragged") else []
    return [k.astype(np.int64), q], ppreds


def table(gx, types, cols, nulls=None):
    if len(cols[0]) == 0:
        return gx.table(types, 1)
    return gx.table_from(types, cols, nulls)


@pytest.mark.parametrize("kind", PROBES)
@pytest.mark.parametrize("form", list(FORM))
def test_form_and_probe_side(gx, form, kind):
    rng = np.random.default_rng(len(form) * 100 + PROBES.index(kind))
    bkeys = build_keys(form, seed=len(kind))
    bcols, bnulls = build_cols(rng, bkeys)
    bt = gx.table_from(BTYPES, bcols, bnulls)
    ht = gx.hash_build(bt, 0, [], unique=form != "walk")
    pcols, ppreds = probe_side(rng, kind, bkeys)
    pt = table(gx, PTYPES, pcols)
    for jt in JTS:
        _, ran, want = check(gx, pt, bt, ht, jt, base_plan(est=50), bcols, bnulls, pcols, ppreds=ppreds)
        if len(pcols[0]):
            assert FORM[form] in ran and "probe_mark" in ran and "filter_marked" in ran, sorted(ran)
        if kind in ("empty", "filtered", "all_miss"):
            total = sum(e[0].value for e in want.values())
            assert total == (0 if jt == SEMI_R else len(bkeys)), total
        if kind == "all_hit":
            assert sum(e[0].value for e in want.values()) == (len(bkeys) if jt == SEMI_R else 0)
    for jt in JTS:                                                   # no GROUP BY: one row, count 0 / sum NULL when empty
        check(gx, pt, bt, ht, jt, base_plan(grouped=False), bcols, bnulls, pcols, ppreds=ppreds)
    pt.free(); ht.free(); bt.free()


# ---------------------------------------------------------------- keys
@pytest.mark.parametrize("unique", [True, False])
def test_null_keys_on_both_sides(gx, unique):
    """ANTI_RIGHT keeps the build rows with a NULL key, SEMI_RIGHT drops them; a NULL probe key matches nothing"""
    rng = np.random.default_rng(5 + unique)
    bkeys = rng.permutation(np.arange(30_000, dtype=np.int64)) if unique else rng.integers(-5000, 5000, 30_000)
    bcols, bnulls = build_cols(rng, bkeys)
    bnulls[0] = (rng.random(len(bkeys)) < 0.2).astype(np.uint8)
    bt = gx.table_from(BTYPES, bcols, bnulls)
    ht = gx.hash_build(bt, 0, [], unique=unique)
    pk = np.concatenate([rng.choice(bkeys, 20_000), rng.integers(-10**5, 10**5, 5000)])
    pcols = [rng.permutation(pk), rng.integers(0, 10, len(pk)).astype(np.int32)]
    pnulls = [(rng.random(len(pk)) < 0.3).astype(np.uint8), None]
    pt = gx.table_from(PTYPES, pcols, pnulls)
    for jt in JTS:
        check(gx, pt, bt, ht, jt, base_plan(est=50), bcols, bnulls, pcols, pnulls)
        got, _, _ = check(gx, pt, bt, ht, jt, base_plan(grouped=False, preds=[(4, g.GX_GE, -3000)]), bcols, bnulls, pcols, pnulls)
        o = R.consumed(jt, bcols, 0, pcols[0], bnulls, pnulls[0])
        nnull = int(bnulls[0][o].sum())
        assert nnull == (int(bnulls[0].sum()) if jt == ANTI_R else 0)
    pt.free(); ht.free(); bt.free()


@pytest.mark.parametrize("side", ["build", "probe", "both"])
def test_int64_min_keys(gx, side):
    """INT64_MIN is an ordinary key: its build rows live in the side list, and are marked by a probe row carrying it"""
    rng = np.random.default_rng(len(side))
    bkeys = rng.integers(-10**6, 10**6, 30_000)
    if side != "probe":
        bkeys[rng.choice(len(bkeys), 3, replace=False)] = I64.min
    bcols, bnulls = build_cols(rng, bkeys)
    bt = gx.table_from(BTYPES, bcols, bnulls)
    ht = gx.hash_build(bt, 0, [], unique=False)
    pk = np.concatenate([rng.choice(bkeys, 10_000), [I64.max, 0]] + ([[I64.min] * 40] if side != "build" else []))
    pcols = [rng.permutation(pk).astype(np.int64), np.zeros(len(pk), np.int32)]
    pt = gx.table_from(PTYPES, pcols)
    for jt in JTS:
        check(gx, pt, bt, ht, jt, base_plan(est=50), bcols, bnulls, pcols)
    pt.free(); ht.free(); bt.free()


@pytest.mark.parametrize("form", ["compact", "walk"])
def test_int4_probe_against_int8_build(gx, form):
    """an int4 probe key widens to int8: the build keys around +-2^31 match only the equal values"""
    rng = np.random.default_rng(77)
    bkeys = build_keys(form, n=100_000) - 3 * 10**5
    bkeys = np.concatenate([bkeys, [I32.min, I32.max, 2**31, -2**31 - 1, 2**32]]) if form == "walk" else bkeys
    bcols, bnulls = build_cols(rng, bkeys.astype(np.int64))
    bt = gx.table_from(BTYPES, bcols, bnulls)
    ht = gx.hash_build(bt, 0, [], unique=form != "walk")
    pk = np.concatenate([rng.choice(bkeys[np.abs(bkeys) < 2**31], 50_000), [I32.min, I32.max, 0, -1]]).astype(np.int32)
    pcols = [rng.permutation(pk), np.zeros(len(pk), np.int32)]
    pt = gx.table_from([g.GX_INT4, g.GX_INT4], pcols)
    for jt in JTS:
        _, ran, _ = check(gx, pt, bt, ht, jt, base_plan(est=50), bcols, bnulls, pcols, ptypes=[g.GX_INT4, g.GX_INT4])
        assert FORM[form] in ran, sorted(ran)
    pt.free(); ht.free(); bt.free()


# ---------------------------------------------------------------- build sides
@pytest.mark.parametrize("nplan", [1, 2])
def test_build_quals_and_plan_quals(gx, nplan):
    """the build quals and the plan's quals both select build rows (3 + 2 quals do not fit one list: the aggregate
    applies the plan's)"""
    rng = np.random.default_rng(31 + nplan)
    bkeys = rng.integers(0, 40_000, 60_000)
    bcols, bnulls = build_cols(rng, bkeys)
    bpreds = [(3, g.GX_GE, -500), (4, g.GX_NE, 7), (1, g.GX_LT, 45)][:3 if nplan == 2 else 2]
    bt = gx.table_from(BTYPES, bcols, bnulls)
    ht = gx.hash_build(bt, 0, [], unique=False, preds=bpreds)
    pk = rng.integers(0, 40_000, 30_000)
    pcols = [pk, rng.integers(0, 10, len(pk)).astype(np.int32)]
    pt = gx.table_from(PTYPES, pcols)
    ppreds = [(2, g.GX_LT, 1.5, True), (4, g.GX_GT, -2000)][:nplan]
    for jt in JTS:
        check(gx, pt, bt, ht, jt, base_plan(est=50, preds=ppreds), bcols, bnulls, pcols, bpreds=bpreds, ppreds=[(1, g.GX_LT, 9)])
    pt.free(); ht.free(); bt.free()


def test_empty_build_side(gx):
    bt = gx.table(BTYPES, 1)
    ht = gx.hash_build(bt, 0, [], unique=True)
    pcols = [np.arange(1000, dtype=np.int64), np.zeros(1000, np.int32)]
    pt = gx.table_from(PTYPES, pcols)
    bcols = [np.zeros(0, np.int64), np.zeros(0, np.int32), np.zeros(0), np.zeros(0, np.int32), np.zeros(0, np.int32)]
    for jt in JTS:
        keys, aggs, nulls = run(gx, pt, bt, ht, jt, base_plan(est=5))[0]
        assert len(keys) == 0
        got = run(gx, pt, bt, ht, jt, base_plan(grouped=False))[0]
        X.check(base_plan(grouped=False), R.expect_right_groups(base_plan(grouped=False), jt, bcols, BTYPES, 0, pcols[0]), got)
    pt.free(); ht.free(); bt.free()


def test_2047_copies_of_one_key(gx):
    """every build row of a matched key is consumed, however many share it"""
    rng = np.random.default_rng(2047)
    bkeys, hot = skewed(rng, 2047)                 # the other keys hash into other sub-tables, as the build needs
    bcols, bnulls = build_cols(rng, bkeys)
    bt = gx.table_from(BTYPES, bcols, bnulls)
    ht = gx.hash_build(bt, 0, [], unique=False)
    pk = np.concatenate([[hot] * 3, rng.choice(bkeys, 500)]).astype(np.int64)
    pcols = [rng.permutation(pk), np.zeros(len(pk), np.int32)]
    pt = gx.table_from(PTYPES, pcols)
    for jt in JTS:
        got, ran, want = check(gx, pt, bt, ht, jt, base_plan(grouped=False), bcols, bnulls, pcols)
        nmatch = int(np.isin(bkeys, pk).sum())
        assert nmatch >= 2047 and want[()][0].value == (nmatch if jt == SEMI_R else len(bkeys) - nmatch)
        assert "probe_mark_walk" in ran
    pt.free(); ht.free(); bt.free()


# ---------------------------------------------------------------- aggregates and group keys
def simple_side(gx, rng, n=80_000, ngroups=50):
    bkeys = rng.permutation(np.arange(n, dtype=np.int64) * 3)
    bcols, bnulls = build_cols(rng, bkeys, ngroups)
    pk = np.concatenate([rng.choice(bkeys, n // 2), rng.integers(0, 3 * n, n // 4)])
    pcols = [pk.astype(np.int64), np.zeros(len(pk), np.int32)]
    return bcols, bnulls, pcols


def test_variance_regression_and_distinct(gx):
    rng = np.random.default_rng(91)
    bcols, bnulls, pcols = simple_side(gx, rng)
    bt = gx.table_from(BTYPES, bcols, bnulls)
    ht = gx.hash_build(bt, 0, [], unique=True)
    pt = gx.table_from(PTYPES, pcols)
    gkeys = bcols[1].astype(np.int64)
    for jt in JTS:
        o = R.consumed(jt, bcols, 0, pcols[0], bnulls)
        # variance and regression, the exact references over the consumed rows
        vplan = base_plan(est=50, aggs=[(g.GX_AGG_VAR_SAMP_F8, [(g.GX_OP_COL, 2, 0)]), (g.GX_AGG_STDDEV_POP_F8, [(g.GX_OP_COL, 3, 0)])])
        got = run(gx, pt, bt, ht, jt, vplan)[0]
        assert V.check(vplan, bcols, bnulls, gkeys, got, rows=o) == 2 * len(got[0])
        rplan = base_plan(est=50, aggs=[(g.GX_AGG_REGR_SLOPE_F8, [(g.GX_OP_COL, 3, 0), (g.GX_OP_ARG2, 0, 0), (g.GX_OP_COL, 4, 0)]),
                                        (g.GX_AGG_CORR_F8, [(g.GX_OP_COL, 3, 0), (g.GX_OP_ARG2, 0, 0), (g.GX_OP_COL, 4, 0)])])
        got = run(gx, pt, bt, ht, jt, rplan)[0]
        assert RG.check(rplan, bcols, bnulls, gkeys, got, rows=o) > 0
        # count(DISTINCT) next to ordinary aggregates
        dplan = base_plan(est=50, aggs=[(g.GX_AGG_COUNT_DISTINCT, [(g.GX_OP_COL, 4, 0)]), (g.GX_AGG_COUNT_STAR, []),
                                        (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)])])
        want = R.expect_right_groups(dplan, jt, bcols, BTYPES, 0, pcols[0], bnulls)
        D.check(dplan, want, run(gx, pt, bt, ht, jt, dplan)[0], [g.GX_INT4])
    pt.free(); ht.free(); bt.free()


@pytest.mark.parametrize("keys", ["every_type", "date_char", "wide16", "many_groups", "none"])
def test_group_keys(gx, keys):
    """group columns of every type with NULLs, a 16-byte key, more than 8192 groups (finalized on the device)"""
    rng = np.random.default_rng(len(keys))
    n = 120_000
    bkeys = rng.permutation(np.arange(n, dtype=np.int64))
    types = [g.GX_INT8, g.GX_INT4, g.GX_DATE, g.GX_CHAR, g.GX_FLOAT8, g.GX_INT8, g.GX_FLOAT8]
    f8 = rng.choice([0.0, -0.0, 1.5, np.nan, np.inf], n)
    cols = [bkeys, rng.integers(0, 3, n).astype(np.int32), rng.integers(-2, 2, n).astype(np.int32),
            rng.integers(-3, 3, n).astype(np.int8), f8, rng.integers(0, 20_000, n) * 2**40, rng.standard_normal(n)]
    nulls = [None] + [(rng.random(n) < 0.1).astype(np.uint8) for _ in range(5)] + [None]
    bt = gx.table_from(types, cols, nulls)
    ht = gx.hash_build(bt, 0, [], unique=True)
    pk = rng.choice(bkeys, n // 2)
    pcols = [pk, np.zeros(len(pk), np.int32)]
    pt = gx.table_from(PTYPES, pcols)
    gc = {"every_type": [1, 3, 4], "date_char": [2, 3], "wide16": [5, 0], "many_groups": [5], "none": []}[keys]
    plan = g.make_plan(group_cols=[(0, c) for c in gc], aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 6, 0)])],
                       est_groups=20_000 if keys in ("wide16", "many_groups") else 200)
    for jt in JTS:
        got, _, want = check(gx, pt, bt, ht, jt, plan, cols, nulls, pcols, btypes=types)
        if keys == "many_groups":
            assert len(got[0]) > 8192
    pt.free(); ht.free(); bt.free()


@pytest.mark.parametrize("jt", JTS)
def test_float8_overflow_only_in_consumed_rows(gx, jt):
    """sum(x) overflows in build rows the join drops: no error; in rows it consumes: GX_ERR_OVERFLOW"""
    rng = np.random.default_rng(21 + jt)
    bkeys = rng.permutation(np.arange(20_000, dtype=np.int64))
    pk = np.arange(0, 20_000, 2, dtype=np.int64)
    pcols = [pk, np.zeros(len(pk), np.int32)]
    pt = gx.table_from(PTYPES, pcols)
    hit = np.isin(bkeys, pk)
    kept = hit if jt == SEMI_R else ~hit
    for where, want_error in (("dropped", False), ("kept", True)):
        bcols, bnulls = build_cols(rng, bkeys, 4, xnull=0.0, special=False)
        bcols[2] = np.ones(len(bkeys))
        bcols[2][np.flatnonzero((~kept if where == "dropped" else kept) & (bcols[1] == 1))[:3]] = 1.5e308
        bt = gx.table_from(BTYPES, bcols, bnulls)
        ht = gx.hash_build(bt, 0, [], unique=True)
        plan = base_plan(est=4)
        if want_error:
            assert R.expect_right_groups(plan, jt, bcols, BTYPES, 0, pk, bnulls) == "overflow"
            with pytest.raises(g.GxError) as ei:
                gx.hash_agg_right(pt, 0, bt, ht, jt, plan)
            assert ei.value.status == g.GX_ERR_OVERFLOW
        else:
            check(gx, pt, bt, ht, jt, plan, bcols, bnulls, pcols)
        ht.free(); bt.free()
    pt.free()


@pytest.mark.parametrize("jt", JTS)
def test_partial_states_and_combine(gx, jt):
    """two datanodes, each with its own build rows and the whole probe side: fetch_states per part, and
    gx_debug_combine's union equals the reference over both parts' build rows"""
    rng = np.random.default_rng(60 + jt)
    bcols, bnulls, pcols = simple_side(gx, rng, n=60_000, ngroups=3000)
    half = len(bcols[0]) // 2
    parts = [([c[:half] for c in bcols], [None if x is None else x[:half] for x in bnulls]),
             ([c[half:] for c in bcols], [None if x is None else x[half:] for x in bnulls])]
    pt = gx.table_from(PTYPES, pcols)
    tabs = []
    for c, nl in parts:
        bt = gx.table_from(BTYPES, c, nl)
        tabs.append((bt, gx.hash_build(bt, 0, [], unique=True)))
    plan = base_plan(est=3000)
    # partial states of part 0: count(*) per group
    r = gx.hash_agg_right(pt, 0, tabs[0][0], tabs[0][1], jt, plan)
    keys, val, cnt, nulls = r.fetch_states()
    r.free()
    o = R.consumed(jt, parts[0][0], 0, pcols[0], parts[0][1])
    want = np.bincount(parts[0][0][1][o], minlength=3000)
    assert dict(zip(keys[:, 0].tolist(), cnt[:, 0].tolist())) == {k: int(v) for k, v in enumerate(want) if v}
    outs = []
    for rank in range(2):
        res = [gx.hash_agg_right(pt, 0, bt, ht, jt, plan) for bt, ht in tabs]
        gx.debug_combine(res, rank)
        outs.append(res[rank].fetch())
        for x in res:
            x.free()
    got = tuple(np.concatenate([o_[i] for o_ in outs]) for i in range(3))
    X.check(plan, R.expect_right_groups(plan, jt, bcols, BTYPES, 0, pcols[0], bnulls), got, [g.GX_INT4])
    for bt, ht in tabs:
        ht.free(); bt.free()
    pt.free()


# ---------------------------------------------------------------- arguments
def test_argument_errors_leave_the_context_usable(gx):
    rng = np.random.default_rng(3)
    bcols, bnulls, pcols = simple_side(gx, rng, n=5000)
    bt = gx.table_from(BTYPES, bcols, bnulls)
    ht = gx.hash_build(bt, 0, [], unique=True)
    hp = gx.hash_build(bt, 0, [3], unique=True)                      # carries a payload column
    other = gx.table_from(BTYPES, bcols, bnulls)
    pt = gx.table_from(PTYPES + [g.GX_FLOAT8], pcols + [np.zeros(len(pcols[0]))])
    good = base_plan(est=50)
    bad_outer = base_plan(est=50); bad_outer.outer_key_col = 0
    bad_jt = base_plan(est=50); bad_jt.join_type = g.GX_JOIN_SEMI
    bad_col = base_plan(est=50, aggs=[(g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 9, 0)])])
    bad_side = g.make_plan(group_cols=[(1, 0)], aggs=[(g.GX_AGG_COUNT_STAR, [])])
    bad_f8_distinct = base_plan(aggs=[(g.GX_AGG_COUNT_DISTINCT, [(g.GX_OP_COL, 2, 0)])])
    cases = [(pt, 0, bt, ht, g.GX_JOIN_SEMI, good), (pt, 0, bt, ht, g.GX_JOIN_ANTI, good), (pt, 0, bt, ht, 7, good),
             (pt, 0, bt, ht, 0, good), (pt, 0, bt, hp, SEMI_R, good), (pt, 0, other, ht, ANTI_R, good),
             (pt, 3, bt, ht, SEMI_R, good), (pt, 2, bt, ht, SEMI_R, good), (pt, -1, bt, ht, SEMI_R, good),
             (pt, 0, bt, None, SEMI_R, good), (pt, 0, bt, ht, SEMI_R, bad_outer), (pt, 0, bt, ht, ANTI_R, bad_jt),
             (pt, 0, bt, ht, SEMI_R, bad_col), (pt, 0, bt, ht, SEMI_R, bad_side), (pt, 0, bt, ht, ANTI_R, bad_f8_distinct)]
    for i, c in enumerate(cases):
        with pytest.raises(g.GxError) as ei:
            gx.hash_agg_right(*c)
        assert ei.value.status == g.GX_ERR_ARG, (i, ei.value)
        check(gx, pt, bt, ht, SEMI_R, good, bcols, bnulls, pcols)
    # a plan the aggregate rejects is rejected before any device work: no marking probe, no compaction
    gx.profile(True)
    for plan in (bad_f8_distinct, bad_col):
        with pytest.raises(g.GxError) as ei:
            gx.hash_agg_right(pt, 0, bt, ht, ANTI_R, plan)
        assert ei.value.status == g.GX_ERR_ARG
    assert gx.profile_get("probe_mark")[1] == 0 and gx.profile_get("filter")[1] == 0
    gx.profile(False)
    # a table changed after the build is no longer the one the join table describes, even at the same row count
    bt.truncate()
    bt.append(bcols, bnulls)
    with pytest.raises(g.GxError) as ei:
        gx.hash_agg_right(pt, 0, bt, ht, SEMI_R, good)
    assert ei.value.status == g.GX_ERR_ARG
    ht2 = gx.hash_build(bt, 0, [], unique=True)
    check(gx, pt, bt, ht2, SEMI_R, good, bcols, bnulls, pcols)
    for x in (pt, other, hp, ht, ht2, bt):
        x.free()


def test_hash_agg_still_rejects_right_join_types(gx):
    bkeys = np.arange(1000, dtype=np.int64)
    bt = gx.table_from([g.GX_INT8], [bkeys])
    ht = gx.hash_build(bt, 0, [], unique=True)
    ot = gx.table_from([g.GX_INT8], [bkeys])
    for jt in (7, SEMI_R, ANTI_R):
        plan = g.make_plan(outer_key_col=0, aggs=[(g.GX_AGG_COUNT_STAR, [])], join_type=jt)
        with pytest.raises(g.GxError) as ei:
            gx.hash_agg(ot, plan, ht)
        assert ei.value.status == g.GX_ERR_ARG
        with pytest.raises(g.GxError) as ei:
            gx.exec_host([g.GX_INT8], [bkeys], len(bkeys), plan, inner_types=[g.GX_INT8], inner_ptrs=[bkeys],
                         inner_nrows=len(bkeys), inner_key_col=0)
        assert ei.value.status == g.GX_ERR_ARG
    ot.free(); ht.free(); bt.free()


# ---------------------------------------------------------------- SF1: the right form against the left form
def groups_of(got):
    keys, aggs, _ = got
    return dict(zip(keys[:, 0].tolist(), aggs[:, 0].view(np.int64).tolist()))


def test_sf1_right_form_equals_left_form(gx):
    """Q4: lineitem[l_shipdate > d] probing orders, GROUP BY o_orderdate count(*), against orders [NOT] EXISTS lineitem;
    Q22: orders probing customer, ANTI, GROUP BY c_mktsegment, against customer NOT EXISTS orders"""
    sf, nord = 1, 1_500_000
    ot = gx.table(g.SCHEMAS[g.T_ORDERS], nord).generate(g.T_ORDERS, sf, 0, nord)
    lt = gx.table(g.SCHEMAS[g.T_LINEITEM], nord * 7).generate(g.T_LINEITEM, sf, 0, nord)
    ct = gx.table(g.SCHEMAS[g.T_CUSTOMER], 150_000 * sf).generate(g.T_CUSTOMER, sf, 0, 150_000 * sf)
    d = int(np.median(lt.read(g.L_SHIPDATE)))
    lq = [(g.L_SHIPDATE, g.GX_GT, d)]
    # right form: build orders (key-ordered: compact), probe lineitem
    ho = gx.hash_build(ot, g.O_ORDERKEY, [], unique=True)
    # left form: build lineitem[l_shipdate > d], probe orders
    hl = gx.hash_build(lt, g.L_ORDERKEY, [], unique=False, preds=lq)
    rplan = g.make_plan(group_cols=[(0, g.O_ORDERDATE)], aggs=[(g.GX_AGG_COUNT_STAR, [])], est_groups=2406)
    for jt, lj in ((SEMI_R, g.GX_JOIN_SEMI), (ANTI_R, g.GX_JOIN_ANTI)):
        right, ran = run(gx, lt, ot, ho, jt, rplan, pkey_col=g.L_ORDERKEY, ppreds=lq)
        left = gx.hash_agg(ot, g.make_plan(outer_key_col=g.O_ORDERKEY, group_cols=[(0, g.O_ORDERDATE)],
                                           aggs=[(g.GX_AGG_COUNT_STAR, [])], est_groups=2406, join_type=lj), hl).fetch()
        assert groups_of(right) == groups_of(left) and len(groups_of(left)) > 1000
        assert "probe_mark_compact" in ran, sorted(ran)
        SEEN.add(("q4", tuple(sorted(ran))))
    hc = gx.hash_build(ct, g.C_CUSTKEY, [], unique=True)
    ho2 = gx.hash_build(ot, g.O_CUSTKEY, [], unique=False)
    cplan = g.make_plan(group_cols=[(0, g.C_MKTSEGMENT)], aggs=[(g.GX_AGG_COUNT_STAR, [])], est_groups=5)
    right = run(gx, ot, ct, hc, ANTI_R, cplan, pkey_col=g.O_CUSTKEY)[0]
    left = gx.hash_agg(ct, g.make_plan(outer_key_col=g.C_CUSTKEY, group_cols=[(0, g.C_MKTSEGMENT)], aggs=[(g.GX_AGG_COUNT_STAR, [])],
                                       est_groups=5, join_type=g.GX_JOIN_ANTI), ho2).fetch()
    assert groups_of(right) == groups_of(left) and sum(groups_of(left).values()) > 0
    for x in (ho2, hc, hl, ho, ct, lt, ot):
        x.free()


# ---------------------------------------------------------------- the provider's executor
HARNESS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "opentenbase_b200", "provider", "harness", "gpuexec_harness")


@pytest.mark.skipif(not os.path.exists(HARNESS), reason="harness binary not built (needs the OpenTenBase headers at build time)")
@pytest.mark.parametrize("jt", JTS)
def test_harness_right_semi_anti_through_begin_exec_end(jt):
    """lineitem[l_shipdate > d] probing orders, GROUP BY o_orderdate count(*), through the CustomScan's Begin / Exec / End
    (orders in the outer slot, lineitem in the join step), against the oracle's aggregate over ExecHashJoinImpl's SEMI /
    ANTI arm with orders as the outer relation"""
    from test_provider_harness import run_harness
    from test_right_semi_anti_provider_cpu import _case
    with tempfile.TemporaryDirectory() as td:
        case, sd, (orel, lrel) = _case(td, jt)
        rows, err = run_harness(case)
    lj = g.GX_JOIN_SEMI if jt == SEMI_R else g.GX_JOIN_ANTI
    want = O.exec_agg(orel, O.make_plan(outer_key_col=g.O_ORDERKEY, group_cols=[(0, g.O_ORDERDATE)], aggs=[(g.GX_AGG_COUNT_STAR, [])]),
                      lrel, O.make_join(g.L_ORDERKEY, inner_unique=0, inner_preds=[(g.L_SHIPDATE, g.GX_GT, sd)], jointype=lj)).sorted()
    got = sorted((int(r[0]), int(r[1])) for r in rows)
    assert len(got) == want.ngroups > 100
    np.testing.assert_array_equal([x[0] for x in got], want.keys[:, 0])
    np.testing.assert_array_equal([x[1] for x in got], want.aggs[:, 0].view(np.int64))
    assert f"GPU Join Type: {'Right Semi' if jt == SEMI_R else 'Right Anti'}" in err


def test_every_variant_ran(request):
    """every marking probe variant answered some case above, and the Q4 shape's compacted aggregate reached a
    specialised kernel.  Judged only when the whole module was selected."""
    ids = {it.nodeid.split("::")[-1] for it in request.session.items}
    if sum(i.startswith("test_form_and_probe_side[") for i in ids) < len(FORM) * len(PROBES) or \
            "test_sf1_right_form_equals_left_form" not in ids:
        pytest.skip("not every case of this module was selected")
    assert set(FORM.values()) <= SEEN, f"never ran: {sorted(set(FORM.values()) - SEEN)}"
    q4 = [set(s[1]) for s in SEEN if isinstance(s, tuple) and s[0] == "q4"]
    assert q4 and all(r & {"agg_fewgroups", "agg_fast", "agg_lptile4", "agg_lptile8"} for r in q4), q4
