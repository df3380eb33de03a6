"""Aggregates over a chain of unique INNER hash joins (gx_hash_agg_joins): gx_k_agg's chain probe reads step 1's table in
the format its build wrote (wide 16-byte, compact 8-byte, narrow 4-byte slots), steps 2.. in their 16-byte form with keys
from the outer row or from an earlier step's payload, and feeds every sink of the aggregate (lane-private and dense
shared-memory tables, the global table, the records of the radix path).

Every case is compared exactly against tests/star_ref.py (join_ref.join step by step, aggregated by exact_ref): counts and
integer sums bit for bit, float8 within the bounds exact_ref derives for the summation order.  The profile names
probe_agg_chain_wide / _compact / _narrow and agg_smem_lp / agg_smem / agg_records / agg_global show which instantiation
answered."""
import numpy as np
import pytest

import opentenbase_b200 as g
import exact_ref as X
import join_ref as J
import star_ref as S

pytestmark = pytest.mark.gpu

I64, I32 = np.iinfo(np.int64), np.iinfo(np.int32)
FMT = {"wide": "probe_agg_chain_wide", "compact": "probe_agg_chain_compact", "narrow": "probe_agg_chain_narrow"}
SINK = {"lp": "agg_smem_lp", "smem": "agg_smem", "radix": "agg_records", "global": "agg_global", "plain": "agg_smem_lp"}
NAMES = set(FMT.values()) | set(SINK.values()) | {"probe_agg_chain", "probe_agg", "build_narrow", "build_compact"}
SEEN = set()                       # (sink, format) profile-name pairs that answered somewhere in this module
FED = set()                        # test_format_and_sink cases that passed
OTYPES = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8]          # key, group column, value
AGGS = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)]), (g.GX_AGG_MAX_F8, [(g.GX_OP_COL, 2, 0)]),
        (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 1, 0)])]
D_1995_03_15 = -1752                                  # days since 2000-01-01


def bunched(n):
    i = np.arange(n, dtype=np.int64)
    return (i // 8) * 32 + (i % 8) + 1


def absent(rng, lo, hi, present, k):
    """k values in [lo, hi) that are not in present"""
    c = rng.integers(lo, hi, 4 * k + 16)
    return c[~np.isin(c, present)][:k]


def dims(gx, fmt, rng, n1=150_000, n2=5000):
    """d1 [key int8 unique, d2 key int4] in the given slot format, d2 [key int4 unique, segment int4].  The narrow form
    needs d2's keys in a small range; spread over all of int4 they force the compact one; shuffled d1 keys the 16-byte one.
    A tenth of d1's d2 keys find no d2 row."""
    d1k = bunched(n1)
    if fmt == "wide":
        d1k = rng.permutation(d1k)
    if fmt == "narrow":
        d2k = (rng.choice(20_000, n2, replace=False) - 10_000).astype(np.int32)
    else:
        d2k = np.unique(np.concatenate([rng.integers(I32.min, I32.max, n2 - 2), [I32.min, I32.max]])).astype(np.int32)
    d1c = rng.choice(d2k, n1)
    miss = rng.random(n1) < 0.1
    d1c[miss] = absent(rng, int(d2k.min()), int(d2k.max()), d2k, int(miss.sum()))
    d1c = d1c.astype(np.int32)
    d2s = rng.integers(0, 5, len(d2k)).astype(np.int32)
    t1 = gx.table_from([g.GX_INT8, g.GX_INT4], [d1k, d1c])
    gx.profile(True)
    h1 = gx.hash_build(t1, 0, [1], unique=True)
    ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    if fmt == "narrow":
        assert "build_narrow" in ran, sorted(ran)
    elif fmt == "compact":
        assert "build_compact" in ran and "build_narrow" not in ran, sorted(ran)
    t2 = gx.table_from([g.GX_INT4, g.GX_INT4], [d2k, d2s])
    h2 = gx.hash_build(t2, 0, [1], unique=True)
    ref = [S.Step((0, 0), d1k, [d1c], [g.GX_INT4]), S.Step((1, 0), d2k, [d2s], [g.GX_INT4])]
    return [(h1, (0, 0)), (h2, (1, 0))], ref, [t1, t2, h1, h2]


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


def group_types(plan, otypes, ref):
    return [otypes[plan.group_cols[c].col] if plan.group_cols[c].side == 0 else ref[plan.group_cols[c].side - 1].ptypes[plan.group_cols[c].col]
            for c in range(plan.n_group_cols)]


def run(gx, ot, steps, plan):
    gx.profile(True)
    got = gx.hash_agg_joins(ot, steps, plan).fetch()
    ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    return got, ran


def check(gx, ot, steps, plan, cols, nulls, ref, otypes=OTYPES):
    want = S.expect_chain_groups(plan, cols, otypes, ref, outer_nulls=nulls)
    got, ran = run(gx, ot, steps, plan)
    X.check(plan, want, got, group_types(plan, otypes, ref))
    assert "probe_agg_chain" in ran and "probe_agg" not in ran, sorted(ran)
    fmts = [f for f, p in FMT.items() if p in ran]
    sinks = [s for s in set(SINK.values()) if s in ran]
    assert len(fmts) == 1 and len(sinks) == 1, sorted(ran)
    SEEN.add((sinks[0], FMT[fmts[0]]))
    return got, ran, want


def free(*objs):
    for o in objs:
        o.free()


# ---------------------------------------------------------------- every step-1 format x every sink
SINK_CASES = {               # grouped, outer group values (x 5 segments), est_groups, strategy
    "lp": (True, 1, 5, 0),
    "smem": (True, 500, 2500, 1),
    "radix": (True, 8000, 40_000, 2),
    "global": (True, 500, 2500, 3),
    "plain": (False, 7, 0, 0),
}


@pytest.mark.parametrize("sink", list(SINK_CASES))
@pytest.mark.parametrize("fmt", list(FMT))
def test_format_and_sink(gx, fmt, sink):
    grouped, ngroups, est, strategy = SINK_CASES[sink]
    rng = np.random.default_rng(len(fmt) * 10 + len(sink))
    steps, ref, keep = dims(gx, fmt, rng)
    cols, nulls = outer_side(rng, ref[0].bkey, 300_000, ngroups)
    ot = gx.table_from(OTYPES, cols, nulls)
    plan = g.make_plan(preds=[(2, g.GX_LT, 2.5, True)], group_cols=[(0, 1), (2, 0)] if grouped else [], aggs=AGGS,
                       est_groups=est, strategy=strategy)
    _, ran, want = check(gx, ot, steps, plan, cols, nulls, ref)
    assert FMT[fmt] in ran and SINK[sink] in ran, sorted(ran)
    assert sum(e[0].value for e in want.values()) > 50_000
    FED.add((fmt, sink))
    free(ot, *keep)


# ---------------------------------------------------------------- three steps, keys from the outer row and from payloads
def three_dims(gx, rng, how):
    """'payloads': step 2's key is step 1's int8 payload (INT64_MIN among the keys), step 3's key step 2's date payload
    (dates before 2000: negative, sign-extended).  'mixed': step 2's key is an outer int4 column, step 3's key step 1's
    int4 payload (negative values too)."""
    n1, n2, n3 = 40_000, 6000, 900
    d3k = rng.choice(np.arange(-3000, 3000), n3, replace=False).astype(np.int32)
    d3g = rng.integers(0, 4, n3).astype(np.int32)
    if how == "payloads":
        d2k = np.concatenate([rng.choice(np.arange(-2**40, 2**40, 2**20), n2 - 1, replace=False), [I64.min]]).astype(np.int64)
        d2d = np.where(rng.random(n2) < 0.1, 3500, rng.choice(d3k, n2)).astype(np.int32)       # 3500: no d3 row
        d2s = rng.integers(0, 3, n2).astype(np.int32)
        d1k = rng.permutation(np.arange(1, n1 + 1, dtype=np.int64) * 3)
        d1p = np.where(rng.random(n1) < 0.1, 7, rng.choice(d2k, n1)).astype(np.int64)            # 7: no d2 row
        t1 = gx.table_from([g.GX_INT8, g.GX_INT8], [d1k, d1p])
        t2 = gx.table_from([g.GX_INT8, g.GX_DATE, g.GX_INT4], [d2k, d2d, d2s])
        t3 = gx.table_from([g.GX_DATE, g.GX_INT4], [d3k, d3g])
        h1, h2, h3 = gx.hash_build(t1, 0, [1], unique=True), gx.hash_build(t2, 0, [1, 2], unique=True), gx.hash_build(t3, 0, [1], unique=True)
        keys = [(0, 0), (1, 0), (2, 0)]
        ref = [S.Step(keys[0], d1k, [d1p], [g.GX_INT8]), S.Step(keys[1], d2k, [d2d, d2s], [g.GX_DATE, g.GX_INT4]),
               S.Step(keys[2], d3k, [d3g], [g.GX_INT4])]
    else:
        d2k = rng.choice(np.arange(-50_000, 50_000), n2, replace=False).astype(np.int32)
        d2s = rng.integers(0, 3, n2).astype(np.int32)
        d2d = rng.integers(0, 9, n2).astype(np.int32)
        d1k = rng.permutation(np.arange(1, n1 + 1, dtype=np.int64) * 3)
        d1p = np.where(rng.random(n1) < 0.1, 4000, rng.choice(d3k, n1)).astype(np.int32)          # 4000: no d3 row
        t1 = gx.table_from([g.GX_INT8, g.GX_INT4], [d1k, d1p])
        t2 = gx.table_from([g.GX_INT4, g.GX_DATE, g.GX_INT4], [d2k, d2d, d2s])
        t3 = gx.table_from([g.GX_INT4, g.GX_INT4], [d3k, d3g])
        h1, h2, h3 = gx.hash_build(t1, 0, [1], unique=True), gx.hash_build(t2, 0, [1, 2], unique=True), gx.hash_build(t3, 0, [1], unique=True)
        keys = [(0, 0), (0, 3), (1, 0)]
        ref = [S.Step(keys[0], d1k, [d1p], [g.GX_INT4]), S.Step(keys[1], d2k, [d2d, d2s], [g.GX_DATE, g.GX_INT4]),
               S.Step(keys[2], d3k, [d3g], [g.GX_INT4])]
    return [(h1, keys[0]), (h2, keys[1]), (h3, keys[2])], ref, [t1, t2, t3, h1, h2, h3]


@pytest.mark.parametrize("how", ["payloads", "mixed"])
@pytest.mark.parametrize("nsteps", [2, 3])
def test_keys_from_outer_columns_and_payloads(gx, how, nsteps):
    rng = np.random.default_rng(7 + nsteps + len(how))
    steps, ref, keep = three_dims(gx, rng, how)
    steps, ref = steps[:nsteps], ref[:nsteps]
    n = 200_000
    cols, nulls = outer_side(rng, ref[0].bkey, n, 11)
    d2key = rng.choice(keep[1].read(0), n).astype(np.int32) if how == "mixed" else np.zeros(n, np.int32)
    d2null = (rng.random(n) < 0.05).astype(np.uint8)          # a NULL step-2 key drops the row
    otypes = OTYPES + [g.GX_INT4]
    cols, nulls = cols + [d2key], nulls + [d2null]
    ot = gx.table_from(otypes, cols, nulls)
    gcols = [(0, 1), (2, 1)] + ([(3, 0)] if nsteps == 3 else [])
    plan = g.make_plan(preds=[(2, g.GX_LT, 2.5, True)], group_cols=gcols, aggs=AGGS, est_groups=200)
    _, _, want = check(gx, ot, steps, plan, cols, nulls, ref, otypes)
    assert sum(e[0].value for e in want.values()) > 10_000
    free(ot, *keep)


def test_group_columns_from_every_step(gx):
    """GROUP BY an outer column, step 1's int8 payload, step 2's date and int4 payloads and step 3's payload"""
    rng = np.random.default_rng(11)
    steps, ref, keep = three_dims(gx, rng, "payloads")
    # step 1's payload (an int8 key of d2) has few distinct values once the other columns are fixed: group by it too
    cols, nulls = outer_side(rng, ref[0].bkey, 100_000, 3)
    ot = gx.table_from(OTYPES, cols, nulls)
    for gcols in ([(0, 1), (2, 0), (2, 1), (3, 0)], [(1, 0), (3, 0)], [(2, 1), (0, 1)]):
        plan = g.make_plan(group_cols=gcols, aggs=AGGS, est_groups=5000)
        check(gx, ot, steps, plan, cols, nulls, ref)
    free(ot, *keep)


# ---------------------------------------------------------------- empty and fully filtered build sides, shuffled outer side
@pytest.mark.parametrize("where", ["step1", "step2"])
@pytest.mark.parametrize("kind", ["empty", "filtered"])
@pytest.mark.parametrize("grouped", [True, False])
def test_build_side_without_rows(gx, where, kind, grouped):
    rng = np.random.default_rng(3)
    d1k = rng.permutation(np.arange(1, 5001, dtype=np.int64))
    d1c = rng.integers(0, 100, 5000).astype(np.int32)
    d2k, d2s = np.arange(0, 100, dtype=np.int32), rng.integers(0, 4, 100).astype(np.int32)
    if kind == "empty":
        d1k, d1c = (d1k[:0], d1c[:0]) if where == "step1" else (d1k, d1c)
        d2k, d2s = (d2k[:0], d2s[:0]) if where == "step2" else (d2k, d2s)
    p1 = [(0, g.GX_LT, -5)] if kind == "filtered" and where == "step1" else []
    p2 = [(1, g.GX_GT, 10)] if kind == "filtered" and where == "step2" else []
    t1 = gx.table(([g.GX_INT8, g.GX_INT4]), max(len(d1k), 1))
    if len(d1k):
        t1.append([d1k, d1c])
    t2 = gx.table(([g.GX_INT4, g.GX_INT4]), max(len(d2k), 1))
    if len(d2k):
        t2.append([d2k, d2s])
    h1, h2 = gx.hash_build(t1, 0, [1], unique=True, preds=p1), gx.hash_build(t2, 0, [1], unique=True, preds=p2)
    ref = [S.Step((0, 0), d1k, [d1c], [g.GX_INT4], bkeep=J.quals([d1k, d1c], None, p1, len(d1k))),
           S.Step((1, 0), d2k, [d2s], [g.GX_INT4], bkeep=J.quals([d2k, d2s], None, p2, len(d2k)))]
    cols, nulls = outer_side(rng, np.arange(1, 5001), 50_000, 4)
    ot = gx.table_from(OTYPES, cols, nulls)
    plan = g.make_plan(group_cols=[(0, 1), (2, 0)] if grouped else [], aggs=AGGS, est_groups=16)
    got, _, want = check(gx, ot, [(h1, (0, 0)), (h2, (1, 0))], plan, cols, nulls, ref)
    assert sum(e[0].value for e in want.values()) == 0
    assert len(got[0]) == (0 if grouped else 1)
    free(ot, h1, h2, t1, t2)


def test_shuffled_outer_side_gives_the_same_answer(gx):
    rng = np.random.default_rng(21)
    steps, ref, keep = dims(gx, "compact", rng)
    cols, nulls = outer_side(rng, ref[0].bkey, 300_000, 40)
    ot = gx.table_from(OTYPES, cols, nulls)
    pt = ot.permuted(seed=12345)
    pcols, pnulls = [pt.read(0, True)[0], pt.read(1), pt.read(2)], [pt.read(0, True)[1], None, None]
    plan = g.make_plan(group_cols=[(0, 1), (2, 0)], aggs=AGGS, est_groups=200)
    check(gx, ot, steps, plan, cols, nulls, ref)
    check(gx, pt, steps, plan, pcols, pnulls, ref)
    free(ot, pt, *keep)


# ---------------------------------------------------------------- one step, errors
@pytest.mark.parametrize("fmt", list(FMT))
def test_one_step_is_gx_hash_agg(gx, fmt):
    rng = np.random.default_rng(31)
    steps, ref, keep = dims(gx, fmt, rng)
    cols, nulls = outer_side(rng, ref[0].bkey, 200_000, 30)
    ot = gx.table_from(OTYPES, cols, nulls)
    plan = g.make_plan(preds=[(2, g.GX_GT, -1.0, True)], group_cols=[(0, 1), (1, 0)], aggs=AGGS, est_groups=3000)
    got = gx.hash_agg_joins(ot, steps[:1], plan).fetch()
    single = g.make_plan(preds=[(2, g.GX_GT, -1.0, True)], outer_key_col=0, group_cols=[(0, 1), (1, 0)], aggs=AGGS, est_groups=3000)
    base = gx.hash_agg(ot, single, steps[0][0]).fetch()
    o1, o2 = np.lexsort(got[0].T[::-1]), np.lexsort(base[0].T[::-1])
    np.testing.assert_array_equal(got[0][o1], base[0][o2])
    # counts and int4 sums bit for bit (the float8 sums' order of addition may differ between launches)
    np.testing.assert_array_equal(got[1][o1][:, [0, 3]].view(np.int64), base[1][o2][:, [0, 3]].view(np.int64))
    want = S.expect_chain_groups(plan, cols, OTYPES, ref[:1], outer_nulls=nulls)
    X.check(plan, want, got, [g.GX_INT4, g.GX_INT4])
    free(ot, *keep)


def test_argument_errors_leave_the_context_usable(gx):
    rng = np.random.default_rng(41)
    steps, ref, keep = dims(gx, "wide", rng, n1=5000, n2=500)
    (h1, _), (h2, _) = steps
    nonu = gx.hash_build(keep[0], 0, [1], unique=False)
    nopay = gx.hash_build(keep[0], 0, [], unique=True)
    cols, nulls = outer_side(rng, ref[0].bkey, 20_000, 3)
    ot = gx.table_from(OTYPES, cols, nulls)
    good = g.make_plan(group_cols=[(0, 1), (2, 0)], aggs=AGGS, est_groups=20)
    bad_plans = {
        "outer key col set": g.make_plan(outer_key_col=0, group_cols=[(0, 1)], aggs=AGGS),
        "plan join type": g.make_plan(group_cols=[(0, 1)], aggs=AGGS, join_type=g.GX_JOIN_SEMI),
        "group side past the chain": g.make_plan(group_cols=[(0, 1), (3, 0)], aggs=AGGS),
    }
    for what, p in bad_plans.items():
        with pytest.raises(g.GxError) as e:
            gx.hash_agg_joins(ot, [(h1, (0, 0)), (h2, (1, 0))], p)
        assert e.value.status == g.GX_ERR_ARG, what
    bad_steps = {
        "no steps": [],
        "four steps": [(h1, (0, 0)), (h2, (1, 0)), (h2, (1, 0)), (h2, (1, 0))],
        "null table": [(h1, (0, 0)), (None, (1, 0))],
        "not unique": [(nonu, (0, 0)), (h2, (1, 0))],
        "key of its own step": [(h1, (0, 0)), (h2, (2, 0))],
        "key of a later step": [(h1, (1, 0)), (h2, (0, 0))],
        "float8 key column": [(h1, (0, 2)), (h2, (1, 0))],
        "outer key column out of range": [(h1, (0, 9)), (h2, (1, 0))],
        "payload index out of range": [(h1, (0, 0)), (h2, (1, 1))],
        "no payload column": [(nopay, (0, 0)), (h2, (1, 0))],
        "left step": [(h1, (0, 0)), (h2, (1, 0), g.GX_JOIN_LEFT)],
        "semi step": [(h1, (0, 0), g.GX_JOIN_SEMI), (h2, (1, 0))],
    }
    for what, st in bad_steps.items():
        with pytest.raises(g.GxError) as e:
            gx.hash_agg_joins(ot, st, good)
        assert e.value.status == g.GX_ERR_ARG, what
    check(gx, ot, steps, good, cols, nulls, ref)
    free(ot, nonu, nopay, *keep)


# ---------------------------------------------------------------- SF1 star on device-generated tables
@pytest.mark.parametrize("shape", ["seg", "q3f"])
def test_sf1_star(gx, shape):
    """lineitem[l_shipdate > D] -> orders[o_orderdate < D] (o_custkey, o_orderdate) -> customer (c_mktsegment):
    seg groups by c_mktsegment; q3f keeps customer[c_mktsegment = 'B'] and groups by l_orderkey, o_orderdate (Q3)"""
    sf, no, nc = 1, 1_500_000, 150_000
    lt = gx.table(g.SCHEMAS[g.T_LINEITEM], no * 7).generate(g.T_LINEITEM, sf, 0, no)
    ot = gx.table(g.SCHEMAS[g.T_ORDERS], no).generate(g.T_ORDERS, sf, 0, no)
    ct = gx.table(g.SCHEMAS[g.T_CUSTOMER], nc).generate(g.T_CUSTOMER, sf, 0, nc)
    opreds = [(g.O_ORDERDATE, g.GX_LT, D_1995_03_15)]
    cpreds = [(g.C_MKTSEGMENT, g.GX_EQ, ord("B"))] if shape == "q3f" else []
    ho = gx.hash_build(ot, g.O_ORDERKEY, [g.O_CUSTKEY, g.O_ORDERDATE], unique=True, preds=opreds)
    hc = gx.hash_build(ct, g.C_CUSTKEY, [g.C_MKTSEGMENT], unique=True, preds=cpreds)
    revenue = [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0), (g.GX_OP_CONST, 0, 1.0), (g.GX_OP_COL, g.L_DISCOUNT, 0), (g.GX_OP_SUB, 0, 0), (g.GX_OP_MUL, 0, 0)]
    gcols = [(2, 0)] if shape == "seg" else [(0, g.L_ORDERKEY), (1, 1)]
    plan = g.make_plan(preds=[(g.L_SHIPDATE, g.GX_GT, D_1995_03_15)], group_cols=gcols,
                       aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, revenue)], est_groups=5 if shape == "seg" else 40_000)
    lcols = [lt.read(c) for c in range(len(g.SCHEMAS[g.T_LINEITEM]))]
    ocols = [ot.read(c) for c in range(len(g.SCHEMAS[g.T_ORDERS]))]
    ccols = [ct.read(c) for c in range(len(g.SCHEMAS[g.T_CUSTOMER]))]
    ref = [S.Step((0, g.L_ORDERKEY), ocols[g.O_ORDERKEY], [ocols[g.O_CUSTKEY], ocols[g.O_ORDERDATE]], [g.GX_INT4, g.GX_DATE],
                  bkeep=J.quals(ocols, None, opreds, len(ocols[0]))),
           S.Step((1, 0), ccols[g.C_CUSTKEY], [ccols[g.C_MKTSEGMENT]], [g.GX_CHAR], bkeep=J.quals(ccols, None, cpreds, len(ccols[0])))]
    _, _, want = check(gx, lt, [(ho, (0, g.L_ORDERKEY)), (hc, (1, 0))], plan, lcols, None, ref, g.SCHEMAS[g.T_LINEITEM])
    assert sum(e[0].value for e in want.values()) > (100_000 if shape == "seg" else 20_000)
    free(lt, ot, ct, ho, hc)


def test_every_sink_and_format_ran():
    """the 12 (sink, step-1 format) instantiations of the chain probe each answered at least one case above"""
    if len(FED) < len(FMT) * len(SINK_CASES):
        pytest.skip("needs every test_format_and_sink case of this run")
    want = {(s, f) for s in set(SINK.values()) for f in FMT.values()}
    assert want <= SEEN, sorted(want - SEEN)


def test_chain_through_the_executor_harness():
    """the provider's Begin/Exec/End over heap pages on the GPU: lineitem -> orders[o_orderdate < date] (o_custkey) -> customer
    (c_mktsegment), GROUP BY c_mktsegment, against star_ref over the same rows"""
    import os
    import subprocess
    import tempfile
    from test_star_agg_cpu import CASE_ORDER_BEFORE, CASE_SHIP_AFTER, chain_case
    from test_provider_harness import HARNESS
    if not os.path.exists(HARNESS):
        pytest.skip("harness binary not built")
    with tempfile.TemporaryDirectory() as d:
        case, (lc, o, cc) = chain_case(d)
        r = subprocess.run([HARNESS, case], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    rows = [line.split("\t") for line in r.stdout.splitlines() if line]
    plan = g.make_plan(preds=[(2, g.GX_GT, CASE_SHIP_AFTER)], group_cols=[(2, 0)],
                       aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])], est_groups=5)
    ref = [S.Step((0, 0), o[0], [o[1]], [g.GX_INT4], bkeep=o[2] < CASE_ORDER_BEFORE), S.Step((1, 0), cc[0], [cc[1]], [g.GX_INT4])]
    want = S.expect_chain_groups(plan, [lc[0], lc[2], lc[5]], [g.GX_INT8, g.GX_FLOAT8, g.GX_DATE], ref)
    keys = np.array([[int(x[0])] for x in rows], np.int64)
    aggs = np.array([[np.int64(int(x[1])).view(np.float64), float(x[2])] for x in rows])
    X.check(plan, want, (keys, aggs, np.zeros((len(rows), 3), np.uint8)), [g.GX_INT4])
    assert len(rows) == len(want) and sum(e[0].value for e in want.values()) > 1000
