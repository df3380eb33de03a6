"""Aggregates over SEMI and ANTI hash joins (gx_agg_plan.join_type): gx_k_agg's existence probe, which reads the join
table in the format the build wrote (wide 16-byte, compact 8-byte, narrow 4-byte slots) and feeds every sink of the
aggregate (lane-private and dense shared-memory tables, the global table, the records of the radix path).

Every case is compared exactly against tests/exists_ref.py, tests/join_ref.py's SEMI / ANTI rows aggregated by
tests/exact_ref.py: count and integer sums bit for bit, float8 within the bounds exact_ref derives for the summation
order.  The profile names
probe_agg_exist_wide / _compact / _narrow and agg_smem_lp / agg_smem / agg_records / agg_global show which instantiation
answered, and build_expand must never run: an existence test reads no payload."""
import os
import tempfile

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import join_ref as J
import exists_ref as E
from helpers import to_gpu_plan

pytestmark = pytest.mark.gpu

I64, I32 = np.iinfo(np.int64), np.iinfo(np.int32)
SEMI, ANTI = g.GX_JOIN_SEMI, g.GX_JOIN_ANTI
FMT = {"wide": "probe_agg_exist_wide", "compact": "probe_agg_exist_compact", "narrow": "probe_agg_exist_narrow"}
SINK = {"lp": "agg_smem_lp", "smem": "agg_smem", "radix": "agg_records", "global": "agg_global", "plain": "agg_smem_lp"}
NAMES = set(FMT.values()) | set(SINK.values()) | {"probe_agg", "build_expand", "build_narrow", "build_compact"}
SEEN = set()                       # (sink, format) profile-name pairs that answered somewhere in this module
OTYPES = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8]          # key, group column, value


def bunched(n):
    i = np.arange(n, dtype=np.int64)
    return (i // 8) * 32 + (i % 8) + 1


def build_side(gx, fmt, n=100_000, seed=0):
    """a non-unique build side (every third key twice) of the given slot format: key-ordered int8 keys with one int4
    payload of a small range (narrow) or none (compact); the same keys shuffled give the 16-byte form (the build tries
    the key-ordered forms first and drops them when it finds the keys out of order: the probe's profile name tells)"""
    keys = bunched(n)
    keys = np.sort(np.concatenate([keys, keys[::3]]))
    if fmt == "wide":
        keys = np.random.default_rng(seed).permutation(keys)
    pay = (keys % 2406 - 2922).astype(np.int32)
    t = gx.table_from([g.GX_INT8, g.GX_INT4], [keys, pay])
    gx.profile(True)
    ht = gx.hash_build(t, 0, [] if fmt == "compact" else [1], unique=False)
    ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    if fmt == "narrow":
        assert "build_narrow" in ran, sorted(ran)
    elif fmt == "compact":
        assert "build_compact" in ran and "build_narrow" not in ran, sorted(ran)
    return ht, t, keys


def outer_side(rng, bkeys, n, ngroups, null_frac=0.05):
    """hits, misses next to hits, keys +- 2^31 / 2^32 off the build keys, INT64_MIN / INT64_MAX; NULL keys"""
    parts = [rng.choice(bkeys, n // 2), rng.choice(bkeys, n // 4) + 2, rng.choice(bkeys, n // 16) + 2**31,
             rng.choice(bkeys, n // 16) - 2**32, rng.integers(-10**6, 10**6, n // 16)]
    k = np.concatenate(parts)
    k = np.concatenate([k, rng.choice(bkeys, n - len(k) - 4), [I64.min, I64.max, 0, -1]]).astype(np.int64)
    k = rng.permutation(k)
    knull = (rng.random(n) < null_frac).astype(np.uint8)
    grp = rng.integers(0, ngroups, n).astype(np.int32)
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)
    return [k, grp, x], [knull, None, None]


def make_plan(jt, grouped=True, est=0, strategy=0, preds=((2, g.GX_LT, 2.5, True),)):
    aggs = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)]), (g.GX_AGG_MAX_F8, [(g.GX_OP_COL, 2, 0)]),
            (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 1, 0)])]
    return g.make_plan(preds=list(preds), outer_key_col=0, group_cols=[(0, 1)] if grouped else [], aggs=aggs, est_groups=est,
                       strategy=strategy, join_type=jt)


def run(gx, ot, plan, ht):
    gx.profile(True)
    got = gx.hash_agg(ot, to_gpu_plan(plan), ht).fetch()
    ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    return got, ran


def check(gx, ot, plan, ht, cols, nulls, bkeys, bnull=None, bkeep=None, types=OTYPES):
    want = E.expect_exists_groups(plan, plan.join_type, cols, types, bkeys, outer_nulls=nulls, inull=bnull, ikeep=bkeep)
    got, ran = run(gx, ot, plan, ht)
    X.check(plan, want, got, [types[1]] if plan.n_group_cols else [])
    assert "probe_agg" in ran and "build_expand" not in ran, sorted(ran)
    fmts = [f for f, p in FMT.items() if p in ran]
    sinks = [s for s in set(SINK.values()) if s in ran]
    assert len(fmts) == 1 and len(sinks) == 1, sorted(ran)
    SEEN.add((sinks[0], FMT[fmts[0]]))
    return got, ran, want


# ---------------------------------------------------------------- every slot format x every sink
SINK_CASES = {               # grouped, groups in the data, est_groups, strategy
    "lp": (True, 5, 5, 0),
    "smem": (True, 2500, 2500, 1),
    "radix": (True, 40_000, 40_000, 2),
    "global": (True, 2500, 2500, 3),
    "plain": (False, 7, 0, 0),
}


@pytest.mark.parametrize("sink", list(SINK_CASES))
@pytest.mark.parametrize("fmt", list(FMT))
def test_format_and_sink(gx, fmt, sink):
    grouped, ngroups, est, strategy = SINK_CASES[sink]
    ht, bt, bkeys = build_side(gx, fmt, seed=len(sink))
    rng = np.random.default_rng(len(fmt) * 10 + len(sink))
    cols, nulls = outer_side(rng, bkeys, 300_000, ngroups)
    ot = gx.table_from(OTYPES, cols, nulls)
    for jt in (SEMI, ANTI):
        _, ran, _ = check(gx, ot, make_plan(jt, grouped, est, strategy), ht, cols, nulls, bkeys)
        assert FMT[fmt] in ran and SINK[sink] in ran, sorted(ran)
    ot.free(); ht.free(); bt.free()


# ---------------------------------------------------------------- key multiplicity
def skewed(rng, m, nfill=3000, hot=123456789):
    """one key m times among nfill distinct keys that hash into other sub-tables (tests/test_gpu_join_edges.py)"""
    n = m + nfill
    nslots = 1
    while nslots < n + n // 2 + 16:
        nslots *= 2
    cand = np.unique(rng.integers(-2**60, 2**60, 3 * nfill + 1000))
    h = cand.view(np.uint64).copy()
    with np.errstate(over="ignore"):
        h ^= h >> np.uint64(33); h *= np.uint64(0xff51afd7ed558ccd)
        h ^= h >> np.uint64(33); h *= np.uint64(0xc4ceb9fe1a85ec53)
        h ^= h >> np.uint64(33)
    hh = np.uint64(hot)
    with np.errstate(over="ignore"):
        hh ^= hh >> np.uint64(33); hh *= np.uint64(0xff51afd7ed558ccd)
        hh ^= hh >> np.uint64(33); hh *= np.uint64(0xc4ceb9fe1a85ec53)
        hh ^= hh >> np.uint64(33)
    sub = lambda v: (v & np.uint64(nslots - 1)) >> np.uint64(11)
    cand = cand[(sub(h) != sub(hh)) & (cand != hot)]
    return rng.permutation(np.concatenate([np.full(m, hot, np.int64), rng.choice(cand, nfill, replace=False)])), hot


@pytest.mark.parametrize("m", [1, 2, 2047])
def test_build_key_multiplicity(gx, m):
    """a build key held 1, 2 or 2047 times: a SEMI row with that key is counted once, an ANTI row not at all"""
    rng = np.random.default_rng(m)
    bkeys, hot = skewed(rng, m)
    bt = gx.table_from([g.GX_INT8], [bkeys])
    ht = gx.hash_build(bt, 0, [], unique=False)
    assert ht.nentries == len(bkeys)
    ok = np.concatenate([np.full(300, hot, np.int64), rng.choice(bkeys, 2000), rng.integers(-2**60, 2**60, 2000)])
    cols = [rng.permutation(ok), rng.integers(0, 3, len(ok)).astype(np.int32), rng.standard_normal(len(ok))]
    ot = gx.table_from(OTYPES, cols)
    for jt in (SEMI, ANTI):
        plan = make_plan(jt, grouped=False, preds=())
        got, _, want = check(gx, ot, plan, ht, cols, [None] * 3, bkeys)
        nhit = int(np.isin(cols[0], bkeys).sum())
        assert int(got[1][0:1, 0].view(np.int64)[0]) == (nhit if jt == SEMI else len(ok) - nhit)
    ot.free(); ht.free(); bt.free()


def test_2047_copies_key_ordered(gx):
    """2047 copies of one key in a key-ordered build (the compact table): the same rule"""
    keys = np.int64(0) + np.arange(1_500_000, dtype=np.int64) * 4
    hot = int(keys[len(keys) // 2])
    keys = np.sort(np.concatenate([keys[np.abs(keys - hot) > 200_000], np.full(2047, hot, np.int64)]))
    bt = gx.table_from([g.GX_INT8], [keys])
    ht = gx.hash_build(bt, 0, [], unique=False)
    rng = np.random.default_rng(2047)
    ok = np.concatenate([np.full(500, hot, np.int64), rng.choice(keys, 100_000), rng.choice(keys, 50_000) + 1])
    cols = [rng.permutation(ok), rng.integers(0, 50, len(ok)).astype(np.int32), rng.standard_normal(len(ok))]
    ot = gx.table_from(OTYPES, cols)
    for jt in (SEMI, ANTI):
        _, ran, _ = check(gx, ot, make_plan(jt, est=50), ht, cols, [None] * 3, keys)
        assert FMT["compact"] in ran, sorted(ran)
    ot.free(); ht.free(); bt.free()


# ---------------------------------------------------------------- NULL keys, empty build sides, INT64_MIN
def test_null_keys_on_both_sides(gx):
    """ANTI keeps an outer row with a NULL key, SEMI drops it; a NULL build key matches nothing"""
    rng = np.random.default_rng(5)
    bkeys = rng.integers(-5000, 5000, 20_000)
    bnull = (rng.random(len(bkeys)) < 0.2).astype(np.uint8)
    bt = gx.table_from([g.GX_INT8], [bkeys], [bnull])
    ht = gx.hash_build(bt, 0, [], unique=False)
    cols, nulls = outer_side(rng, bkeys, 100_000, 40, null_frac=0.15)
    ot = gx.table_from(OTYPES, cols, nulls)
    for jt in (SEMI, ANTI):
        plan = make_plan(jt, est=40)
        _, _, want = check(gx, ot, plan, ht, cols, nulls, bkeys, bnull=bnull)
        # the NULL-key rows alone
        sel = nulls[0].astype(bool) & (cols[2] < 2.5)
        only = make_plan(jt, grouped=False)
        part = E.expect_exists_groups(only, jt, [c[sel] for c in cols], OTYPES, bkeys, outer_nulls=[nulls[0][sel], None, None],
                                      inull=bnull)
        assert part[()][0].value == (int(sel.sum()) if jt == ANTI else 0)
    ot.free(); ht.free(); bt.free()


@pytest.mark.parametrize("kind", ["empty", "quals_reject_all"])
@pytest.mark.parametrize("grouped", [True, False])
def test_build_side_without_rows(gx, kind, grouped):
    """ANTI gives every outer row that passes its quals, SEMI no group (count 0 / sum NULL without GROUP BY)"""
    rng = np.random.default_rng(11 + grouped)
    bkeys = np.zeros(0, np.int64) if kind == "empty" else rng.integers(0, 1000, 5000)
    bt = gx.table_from([g.GX_INT8], [bkeys]) if len(bkeys) else gx.table([g.GX_INT8], 1)
    bpreds = [(0, g.GX_LT, -1)] if kind != "empty" else []
    ht = gx.hash_build(bt, 0, [], unique=False, preds=bpreds)
    bkeep = J.quals([bkeys], None, bpreds, len(bkeys))
    cols, nulls = outer_side(rng, np.arange(1000, dtype=np.int64), 50_000, 30)
    ot = gx.table_from(OTYPES, cols, nulls)
    for jt in (SEMI, ANTI):
        plan = make_plan(jt, grouped, est=30)
        got, _, _ = check(gx, ot, plan, ht, cols, nulls, bkeys, bkeep=bkeep)
        keys, aggs, gnulls = got
        if jt == SEMI and grouped:
            assert len(keys) == 0
        elif jt == SEMI:
            assert aggs[0:1, 0].view(np.int64)[0] == 0 and gnulls[0, 1] == 1
        else:
            assert int(aggs[:, 0].view(np.int64).sum()) == int((cols[2] < 2.5).sum())
    ot.free(); ht.free(); bt.free()


@pytest.mark.parametrize("build_has_min", [True, False])
def test_int64_min_keys(gx, build_has_min):
    """INT64_MIN is an ordinary key: it lives in the 16-byte table's side list, and a SEMI row with it has a partner
    exactly when a build row carries it"""
    rng = np.random.default_rng(3 + build_has_min)
    bkeys = np.concatenate([rng.integers(-10**6, 10**6, 30_000), np.full(3 if build_has_min else 0, I64.min, np.int64),
                            np.array([I64.max], np.int64)])
    bt = gx.table_from([g.GX_INT8], [rng.permutation(bkeys)])
    ht = gx.hash_build(bt, 0, [], unique=False)
    ok = np.concatenate([np.full(700, I64.min, np.int64), rng.choice(bkeys, 20_000), rng.integers(-10**6, 10**6, 20_000)])
    cols = [rng.permutation(ok), rng.integers(0, 20, len(ok)).astype(np.int32), rng.standard_normal(len(ok))]
    ot = gx.table_from(OTYPES, cols)
    for jt in (SEMI, ANTI):
        check(gx, ot, make_plan(jt, est=20), ht, cols, [None] * 3, bkeys)
    ot.free(); ht.free(); bt.free()


# ---------------------------------------------------------------- key widths and the compact span's edges
@pytest.mark.parametrize("outer_int4", [False, True])
def test_int4_outer_and_compact_span_edges(gx, outer_int4):
    """a compact table over int8 keys crossing zero, probed with int4 keys or with int8 keys k +- 2^31 and k +- 2^32,
    which share the low 31 / 32 bits of a stored key and must not match it"""
    bkeys = np.int64(-300_000) + np.arange(200_000, dtype=np.int64) * 3
    bkeys = np.sort(np.concatenate([bkeys, bkeys[::5]]))
    bt = gx.table_from([g.GX_INT8], [bkeys])
    ht = gx.hash_build(bt, 0, [], unique=False)
    rng = np.random.default_rng(17 + outer_int4)
    parts = [rng.choice(bkeys, 40_000), rng.choice(bkeys, 20_000) + 1, [int(bkeys[0]) - 1, int(bkeys[-1]) + 1, int(bkeys[0]), int(bkeys[-1])]]
    if outer_int4:
        parts += [[I32.min, I32.max, 0]]
    else:
        for d in (2**31, 2**32, 2**31 - 1, 2**32 + 1):
            parts += [rng.choice(bkeys, 5000) + d, rng.choice(bkeys, 5000) - d]
    ok = rng.permutation(np.concatenate(parts).astype(np.int64))
    types = [g.GX_INT4 if outer_int4 else g.GX_INT8, g.GX_INT4, g.GX_FLOAT8]
    cols = [ok.astype(np.int32) if outer_int4 else ok, rng.integers(0, 100, len(ok)).astype(np.int32), rng.standard_normal(len(ok))]
    ot = gx.table_from(types, cols)
    for jt in (SEMI, ANTI):
        _, ran, _ = check(gx, ot, make_plan(jt, est=100), ht, cols, [None] * 3, bkeys, types=types)
        assert FMT["compact"] in ran, sorted(ran)
    ot.free(); ht.free(); bt.free()


# ---------------------------------------------------------------- layout, overflow, the host entry point, arguments
def test_shuffled_outer_side_gives_the_same_answer(gx):
    ht, bt, bkeys = build_side(gx, "narrow", seed=9)
    rng = np.random.default_rng(9)
    cols, nulls = outer_side(rng, np.sort(bkeys), 400_000, 2500)
    order = np.argsort(cols[0], kind="stable")                   # clustered on the key, as a table read in key order is
    cols, nulls = [c[order] for c in cols], [None if x is None else x[order] for x in nulls]
    ot = gx.table_from(OTYPES, cols, nulls)
    pt = ot.permuted(seed=12345)
    for jt in (SEMI, ANTI):
        plan = make_plan(jt, est=2500)
        a = run(gx, ot, plan, ht)[0]
        b = run(gx, pt, plan, ht)[0]
        want = E.expect_exists_groups(plan, jt, cols, OTYPES, bkeys, outer_nulls=nulls)
        X.check(plan, want, a, [g.GX_INT4])
        X.check(plan, want, b, [g.GX_INT4])
        ka, kb = np.argsort(a[0][:, 0]), np.argsort(b[0][:, 0])
        np.testing.assert_array_equal(a[0][ka], b[0][kb])
        np.testing.assert_array_equal(a[1][ka][:, [0, 3]].view(np.int64), b[1][kb][:, [0, 3]].view(np.int64))
    pt.free(); ot.free(); ht.free(); bt.free()


@pytest.mark.parametrize("jt", [SEMI, ANTI])
def test_float8_overflow_only_in_the_rows_the_join_keeps(gx, jt):
    """sum(x) overflows in rows the join drops: no error; in rows it keeps: GX_ERR_OVERFLOW (float8pl's CHECKFLOATVAL)"""
    rng = np.random.default_rng(21 + jt)
    bkeys = np.arange(0, 20_000, 2, dtype=np.int64)
    bt = gx.table_from([g.GX_INT8], [rng.permutation(bkeys)])
    ht = gx.hash_build(bt, 0, [], unique=False)
    ok = rng.integers(0, 20_000, 50_000).astype(np.int64)
    grp = (ok // 2 % 4).astype(np.int32)                 # every group holds rows with and without a partner
    kept = np.isin(ok, bkeys) if jt == SEMI else ~np.isin(ok, bkeys)
    for where, want_error in (("dropped", False), ("kept", True)):
        x = np.ones(len(ok))
        rows = np.flatnonzero((~kept if where == "dropped" else kept) & (grp == 1))[:3]
        x[rows] = 1.5e308
        cols = [ok, grp, x]
        ot = gx.table_from(OTYPES, cols)
        plan = make_plan(jt, est=4, preds=())
        want = E.expect_exists_groups(plan, jt, cols, OTYPES, bkeys)
        if want_error:
            assert want == "overflow"
            with pytest.raises(g.GxError) as ei:
                gx.hash_agg(ot, to_gpu_plan(plan), ht)
            assert ei.value.status == g.GX_ERR_OVERFLOW
        else:
            check(gx, ot, plan, ht, cols, [None] * 3, bkeys)
        ot.free()
    ht.free(); bt.free()


@pytest.mark.parametrize("jt", [SEMI, ANTI])
def test_exec_host_equals_the_resident_path(gx, jt):
    rng = np.random.default_rng(40 + jt)
    bkeys = np.sort(np.concatenate([bunched(200_000), bunched(200_000)[::4]]))
    bq = rng.integers(0, 10, len(bkeys)).astype(np.int32)
    ok = np.concatenate([rng.choice(bkeys, 300_000), rng.choice(bkeys, 100_000) + 2])
    cols = [rng.permutation(ok), rng.integers(0, 2500, len(ok)).astype(np.int32), rng.standard_normal(len(ok))]
    plan = make_plan(jt, est=2500)
    bpreds = [(1, g.GX_GE, 3)]
    bt = gx.table_from([g.GX_INT8, g.GX_INT4], [bkeys, bq])
    ht = gx.hash_build(bt, 0, [], unique=False, preds=bpreds)
    ot = gx.table_from(OTYPES, cols)
    a = run(gx, ot, plan, ht)[0]
    r = gx.exec_host(OTYPES, cols, len(ok), to_gpu_plan(plan), inner_types=[g.GX_INT8, g.GX_INT4], inner_ptrs=[bkeys, bq],
                     inner_nrows=len(bkeys), inner_key_col=0, inner_preds=bpreds)
    b = r.fetch()
    r.free()
    want = E.expect_exists_groups(plan, jt, cols, OTYPES, bkeys, ikeep=J.quals([bkeys, bq], None, bpreds, len(bkeys)))
    X.check(plan, want, a, [g.GX_INT4])
    X.check(plan, want, b, [g.GX_INT4])
    ka, kb = np.argsort(a[0][:, 0]), np.argsort(b[0][:, 0])
    np.testing.assert_array_equal(a[0][ka], b[0][kb])
    np.testing.assert_array_equal(a[1][ka][:, [0, 3]].view(np.int64), b[1][kb][:, [0, 3]].view(np.int64))
    ot.free(); ht.free(); bt.free()


def test_unsupported_join_types_and_inner_columns_are_arguments_errors(gx):
    """LEFT (its inner group columns would have to turn NULL on a miss) and an unknown join type are GX_ERR_ARG, as is a
    side-1 group column under SEMI / ANTI; the next call on the same context works"""
    bkeys = np.arange(1000, dtype=np.int64)
    bt = gx.table_from([g.GX_INT8, g.GX_INT4], [bkeys, (bkeys % 7).astype(np.int32)])
    ht = gx.hash_build(bt, 0, [1], unique=True)
    cols = [np.arange(-500, 1500, dtype=np.int64), np.zeros(2000, np.int32), np.ones(2000)]
    ot = gx.table_from(OTYPES, cols)
    bad = [make_plan(g.GX_JOIN_LEFT), make_plan(7), make_plan(-1),
           g.make_plan(outer_key_col=0, group_cols=[(1, 0)], aggs=[(g.GX_AGG_COUNT_STAR, [])], join_type=SEMI)]
    for plan in bad:
        with pytest.raises(g.GxError) as ei:
            gx.hash_agg(ot, to_gpu_plan(plan), ht)
        assert ei.value.status == g.GX_ERR_ARG, ei.value
        with pytest.raises(g.GxError) as ei:
            gx.exec_host(OTYPES, cols, len(cols[0]), to_gpu_plan(plan), inner_types=[g.GX_INT8, g.GX_INT4],
                         inner_ptrs=[bkeys, (bkeys % 7).astype(np.int32)], inner_nrows=len(bkeys), inner_key_col=0, payload_cols=[1])
        assert ei.value.status == g.GX_ERR_ARG, ei.value
        check(gx, ot, make_plan(SEMI, est=1), ht, cols, [None] * 3, bkeys)
    ot.free(); ht.free(); bt.free()


# ---------------------------------------------------------------- the provider's executor
HARNESS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "opentenbase_b200", "provider", "harness", "gpuexec_harness")


@pytest.mark.skipif(not os.path.exists(HARNESS), reason="harness binary not built (needs /root/reference at build time)")
@pytest.mark.parametrize("jt", [SEMI, ANTI])
def test_harness_semi_anti_through_begin_exec_end(jt):
    """orders [NOT] EXISTS lineitem[l_shipdate > d] GROUP BY o_orderdate count(*) through the CustomScan's
    Begin / Exec / End, against the oracle's aggregate over ExecHashJoinImpl's SEMI / ANTI arm"""
    from test_provider_harness import INT8OID, run_harness, write_case
    sf, nord = 1, 30000
    o, l = O.gen_orders(sf, 0, nord), O.gen_lineitem(sf, 0, nord)
    otypes = [O.GX_INT8, O.GX_INT4, O.GX_DATE, O.GX_INT4]
    ltypes = [O.GX_INT8, O.GX_FLOAT8, O.GX_FLOAT8, O.GX_FLOAT8, O.GX_FLOAT8, O.GX_DATE, O.ORC_BPCHAR1, O.ORC_BPCHAR1]
    orel, lrel = O.Rel(otypes, o), O.Rel(ltypes, l)
    d = int(np.median(l[g.L_SHIPDATE])) + 400
    plan = g.make_plan(outer_key_col=0, group_cols=[(0, 1)], aggs=[(g.GX_AGG_COUNT_STAR, [])], est_groups=2500, join_type=jt)
    with tempfile.TemporaryDirectory() as td:
        case = os.path.join(td, "exists.case")
        write_case(case, [(otypes, orel), (ltypes, lrel)], {"rti": 1, "attnums": [0, 2]},
                   {"rti": 2, "attnums": [0, 5], "key_col": 0, "payload_cols": [], "unique": False, "preds": [(1, g.GX_GT, d)]},
                   plan, False, [1082, INT8OID])
        rows, err = run_harness(case)
    want = O.exec_agg(orel, O.make_plan(outer_key_col=g.O_ORDERKEY, group_cols=[(0, g.O_ORDERDATE)], aggs=[(g.GX_AGG_COUNT_STAR, [])]),
                      lrel, O.make_join(g.L_ORDERKEY, inner_unique=0, inner_preds=[(g.L_SHIPDATE, g.GX_GT, d)], jointype=jt)).sorted()
    got = sorted((int(r[0]), int(r[1])) for r in rows)
    assert len(got) == want.ngroups > 100
    np.testing.assert_array_equal([x[0] for x in got], want.keys[:, 0])
    np.testing.assert_array_equal([x[1] for x in got], want.aggs[:, 0].view(np.int64))
    assert f"GPU Join Type: {'Semi' if jt == SEMI else 'Anti'}" in err


def test_every_instantiation_ran(request):
    """every (sink, slot format) instantiation of the existence probe answered some case above.  Judged only when the
    whole module was selected."""
    ids = {it.nodeid.split("::")[-1] for it in request.session.items}
    if sum(i.startswith("test_format_and_sink[") for i in ids) < len(FMT) * len(SINK_CASES):
        pytest.skip("not every case of this module was selected")
    want = {(s, f) for s in set(SINK.values()) for f in FMT.values()}
    assert SEEN >= want, f"never ran: {sorted(want - SEEN)}"
