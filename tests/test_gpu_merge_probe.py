"""The merge probe: a unique key-ordered build of an int8 key with one int4/date payload whose narrowest table (4-byte slots)
would not fit L2 defers its fill, and gx_hash_agg of the run-folding plan shape (GROUP BY the payload, count(*) and one
float8 sum, outer side in key order) merges the outer rows with the build rows themselves (gx_k_mergejoin, profile name
probe_agg_merge).  Everything else that reads the handle fills the table first, exactly as an eager build would.

Build sides here are 9 M rows and more: 16 M slots x 4 B = 64 MB, above the H100's 50 MB of L2.  Answers are checked
against the exact references of tests/join_ref.py and tests/exact_ref.py, or against the same handle once ht.info() has
filled it (keys and counts bit-exact, float8 sums within 1e-9 relative)."""
import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import join_ref as J
from helpers import to_gpu_plan

pytestmark = pytest.mark.gpu

I64 = np.iinfo(np.int64)
I32 = np.iinfo(np.int32)
NBUILD = 9_000_000
BUILD_NAMES = ("build", "build_sample", "build_bounds", "build_fill_staged", "build_sorted_search", "build_narrow", "build_compact")


def bunched(n):
    """TPC-H order keys: 8 used of every 32"""
    i = np.arange(n, dtype=np.int64)
    return (i // 8) * 32 + (i % 8) + 1


def dates(rng, n):
    return rng.integers(8036, 8036 + 2406, n).astype(np.int32)


def build(gx, keys, pay, ptype=g.GX_INT4, spare=0):
    t = gx.table([g.GX_INT8, ptype], len(keys) + spare + 1).append([keys, pay])
    return gx.hash_build(t, 0, [1], unique=True), t


def outer_side(rng, keys, n):
    """n rows in key order: mostly build keys (runs of 1..7 rows), some misses between, below and above them"""
    hits = rng.choice(keys, n * 3 // 4)
    miss = np.concatenate([rng.choice(keys, n // 8) + 1, rng.integers(int(keys[0]) - 1000, int(keys[-1]) + 1000, n - n * 3 // 4 - n // 8)])
    return np.sort(np.concatenate([hits, miss]).astype(np.int64))


def plan_of(est=2500):
    return O.make_plan(outer_key_col=0, group_cols=[(1, 0)], aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])],
                       est_groups=est)


def agg(gx, ot, ht, plan):
    """the result and the profile names that ran"""
    gx.profile(True)
    got = gx.hash_agg(ot, to_gpu_plan(plan), ht).fetch()
    ran = {n: gx.profile_get(n)[1] for n in BUILD_NAMES + ("probe_agg_merge", "probe_agg_tma", "probe_agg")}
    gx.profile(False)
    return got, {n for n, c in ran.items() if c}, ran


def exact(gx, ok, x, keys, pay, ht, plan, ptype=g.GX_INT4):
    want = J.expect_groups(plan, J.join(g.GX_JOIN_INNER, ok, keys), [ok, x], [g.GX_INT8, g.GX_FLOAT8], [pay], [ptype])
    ot = gx.table_from([g.GX_INT8, g.GX_FLOAT8], [ok, x])
    got, ran, _ = agg(gx, ot, ht, plan)
    X.check(plan, want, got, [ptype])
    ot.free()
    return ran


def same(a, b, rtol=1e-9):
    ka, aa, _ = a
    kb, ab, _ = b
    oa, ob = np.argsort(ka[:, 0], kind="stable"), np.argsort(kb[:, 0], kind="stable")
    np.testing.assert_array_equal(ka[oa], kb[ob])
    np.testing.assert_array_equal(aa[oa, 0].view(np.int64), ab[ob, 0].view(np.int64))
    np.testing.assert_allclose(aa[oa, 1], ab[ob, 1], rtol=rtol, atol=0)


def test_path_taken_configs2(gx):
    """configs[2] at SF 7: the merge answers, no build kernel runs in either call; once filled, gx_k_runjoin_tma agrees"""
    sf, n = 7, 1_500_000 * 7
    ot = gx.table(g.SCHEMAS[g.T_ORDERS], n + 1000).generate(g.T_ORDERS, sf, 0, n)
    lt = gx.table(g.SCHEMAS[g.T_LINEITEM], n * 7 + 1000).generate(g.T_LINEITEM, sf, 0, n)
    plan = g.GxAggPlan.from_buffer_copy(bytes(O.make_plan(outer_key_col=g.L_ORDERKEY, group_cols=[(1, 0)],
                                                          aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0)])],
                                                          est_groups=2500)))
    gx.profile(True)
    ht = gx.hash_build(ot, g.O_ORDERKEY, [g.O_ORDERDATE], unique=True)
    built = {nm for nm in BUILD_NAMES if nm != "build_sample" and gx.profile_get(nm)[1] > 0}
    merged = gx.hash_agg(lt, plan, ht).fetch()
    ran = {nm for nm in BUILD_NAMES + ("probe_agg_merge", "probe_agg_tma") if gx.profile_get(nm)[1] > 0}
    gx.profile(False)
    assert not built and "probe_agg_merge" in ran and not (ran & set(BUILD_NAMES) - {"build_sample"}), ran
    info = ht.info()
    assert info["slot_mode"] == 2 and ht.nentries == ot.nrows, info
    gx.profile(True)
    filled = gx.hash_agg(lt, plan, ht).fetch()
    assert gx.profile_get("probe_agg_tma")[1] > 0 and gx.profile_get("probe_agg_merge")[1] == 0
    gx.profile(False)
    same(merged, filled)
    assert int(merged[1][:, 0].view(np.int64).sum()) == lt.nrows
    ht.free(); ot.free(); lt.free()


@pytest.mark.parametrize("seed", [1, 2])
def test_keys_and_misses(gx, seed):
    """keys below, above and between the build's, build rows no outer row reaches (with gaps far longer than a warp's
    window), runs across warp boundaries, INT64_MIN / INT64_MAX on both sides, payloads over the whole int4 range"""
    rng = np.random.default_rng(seed)
    keys = bunched(NBUILD)
    keys[NBUILD // 3: NBUILD // 3 + 200_000] += 50_000_000        # a stretch of build keys far above the rest
    keys = np.sort(keys)
    keys[0], keys[-1] = I64.min, I64.max
    # 2000 payload values spread over the whole int4 range, its ends included: 2000 groups
    values = np.concatenate([[I32.min, I32.max, 0], rng.integers(I32.min, I32.max, 1997, endpoint=True)]).astype(np.int32)
    pay = values[rng.integers(0, len(values), NBUILD)]
    ht, t = build(gx, keys, pay)
    ok = outer_side(rng, keys[1:-1], NBUILD + 1000)
    ok = ok[(ok < keys[NBUILD // 3]) | (ok > keys[NBUILD // 3 + 20_000])]       # 20 000 build rows no outer row reaches
    ok = np.sort(np.concatenate([ok, [I64.min] * 3, [I64.max] * 2, rng.choice(keys, NBUILD - len(ok) + 5)]).astype(np.int64))
    x = rng.standard_normal(len(ok)) * 100.0
    ran = exact(gx, ok, x, keys, pay, ht, plan_of())
    assert "probe_agg_merge" in ran and "build_fill_staged" not in ran, ran
    ht.free(); t.free()


@pytest.mark.parametrize("where", ["outer_inside", "outer_boundary", "outer_last", "build_desc", "build_equal"])
def test_order_violation_falls_back(gx, where):
    """one pair out of order: the merge raises its flag, the table is filled (build_fill_staged after the merge) and the
    answer is today's"""
    rng = np.random.default_rng(7)
    keys = bunched(NBUILD)
    pay = dates(rng, NBUILD)
    if where == "build_desc":
        keys[5_000_001], keys[5_000_002] = keys[5_000_002], keys[5_000_001]
    if where == "build_equal":
        keys[5_000_001] = keys[5_000_000]
    ht, t = build(gx, keys, pay)
    ok = outer_side(rng, keys, NBUILD + 1000)
    i = {"outer_inside": len(ok) // 2 + 17, "outer_boundary": 0, "outer_last": len(ok) - 2}.get(where)
    if where == "outer_boundary":
        # the last row of warp 0 and the first of warp 1: one CTA of 32 warps per SM, rows per warp a multiple of 128
        warps = gx.device_info()["sm_count"] * 32
        i = 128 * (((len(ok) + warps - 1) // warps + 127) // 128) - 1
    if i is not None:
        ok[i], ok[i + 1] = ok[i + 1], ok[i] - 1
    x = rng.standard_normal(len(ok))
    plan = plan_of()
    ot = gx.table_from([g.GX_INT8, g.GX_FLOAT8], [ok, x])
    got, ran, _ = agg(gx, ot, ht, plan)
    # the merge ran, saw the pair and the table was filled after it (a build out of key order is filled by the bucketed
    # path, the others by the key-ordered one)
    assert "probe_agg_merge" in ran and "build" in ran, ran
    if where.startswith("outer"):
        assert "build_fill_staged" in ran, ran
    want = J.expect_groups(plan, J.join(g.GX_JOIN_INNER, ok, keys[np.sort(np.unique(keys, return_index=True)[1])]), [ok, x],
                           [g.GX_INT8, g.GX_FLOAT8], [pay[np.sort(np.unique(keys, return_index=True)[1])]], [g.GX_INT4]) \
        if where != "build_equal" else None
    if want is not None:
        X.check(plan, want, got, [g.GX_INT4])
    # the same table filled before any merge answers the same
    ht2, t2 = build(gx, keys, pay)
    ht2.info()
    filled, ran2, _ = agg(gx, ot, ht2, plan)
    assert "probe_agg_merge" not in ran2
    same(got, filled)
    ht.free(); t.free(); ht2.free(); t2.free(); ot.free()


@pytest.mark.parametrize("cover", ["first_quarter", "ends_only"])
def test_outer_covers_part_of_the_build(gx, cover):
    """outer keys over only the first quarter of the build's keys, or over its first and last eighth with the middle
    skipped: a warp would walk a long stretch of build rows alone, so the merge gives up before walking it and the
    filled table answers"""
    rng = np.random.default_rng(13)
    keys = bunched(NBUILD)
    pay = dates(rng, NBUILD)
    ht, t = build(gx, keys, pay)
    part = keys[: NBUILD // 4] if cover == "first_quarter" else np.concatenate([keys[: NBUILD // 8], keys[-NBUILD // 8:]])
    ok = np.sort(rng.choice(part, NBUILD + 100)).astype(np.int64)
    ran = exact(gx, ok, rng.standard_normal(len(ok)), keys, pay, ht, plan_of())
    assert "probe_agg_merge" in ran and "build_fill_staged" in ran, ran
    ht.free(); t.free()


def test_datanode_subset(gx):
    """rank 1 of 4: a pseudo-random quarter of the orders, still ascending, and the lineitem rows of those orders"""
    sf, n = 24, 1_500_000 * 24
    gx.set_shardmap(4)
    try:
        ot = gx.table(g.SCHEMAS[g.T_ORDERS], n // 4 + 1_000_000).generate(g.T_ORDERS, sf, 0, n, 1, 4)
        lt = gx.table(g.SCHEMAS[g.T_LINEITEM], n * 2 + 1_000_000).generate(g.T_LINEITEM, sf, 0, n, 1, 4)
    finally:
        gx.set_shardmap(1)
    plan = to_gpu_plan(O.make_plan(outer_key_col=g.L_ORDERKEY, group_cols=[(1, 0)],
                                   aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0)])], est_groups=2500))
    ht = gx.hash_build(ot, g.O_ORDERKEY, [g.O_ORDERDATE], unique=True)
    gx.profile(True)
    merged = gx.hash_agg(lt, plan, ht).fetch()
    assert gx.profile_get("probe_agg_merge")[1] > 0
    gx.profile(False)
    ht.info()
    same(merged, gx.hash_agg(lt, plan, ht).fetch())
    ht.free(); ot.free(); lt.free()


@pytest.mark.parametrize("extra", [1, 3, 127, 4 * 128 + 5])
def test_tails(gx, extra):
    """outer sides of nbuild + 1, 3, 127 and 517 rows take the merge (the < 4 rows after the last full vector, a last tile
    of a few vectors); outer sides of 1, 3, 127 and 517 rows and an empty one take the filled table"""
    rng = np.random.default_rng(extra)
    keys = bunched(NBUILD)
    pay = dates(rng, NBUILD)
    ht, t = build(gx, keys, pay)
    ok = outer_side(rng, keys, NBUILD + extra)
    ran = exact(gx, ok, rng.standard_normal(len(ok)), keys, pay, ht, plan_of())
    assert "probe_agg_merge" in ran, ran
    ht.free(); t.free()
    for n in (0, extra):
        ht, t = build(gx, keys, pay)
        ok = np.sort(rng.choice(keys, n)).astype(np.int64) if n else np.zeros(0, np.int64)
        ran = exact(gx, ok, rng.standard_normal(n), keys, pay, ht, plan_of())
        assert "probe_agg_merge" not in ran, ran
        ht.free(); t.free()


def test_handle_lifecycle(gx):
    """a deferred handle answers every reader as the eager build of the same table does; its table appended to or
    truncated before the first use still gives the answer of the table at build time; free without use"""
    rng = np.random.default_rng(11)
    keys = bunched(NBUILD)
    pay = dates(rng, NBUILD)
    eager, te = build(gx, keys, pay)
    info = eager.info()                                          # filled now: the reference for every reader
    lazy, tl = build(gx, keys, pay)
    pk = np.sort(np.concatenate([rng.choice(keys, 100_000), rng.integers(0, int(keys[-1]) + 5, 20_000)])).astype(np.int64)
    pt = gx.table_from([g.GX_INT8, g.GX_INT4], [pk, np.arange(len(pk), dtype=np.int32)])
    a = gx.hash_probe(pt, 0, eager, [0, 1])
    b = gx.hash_probe(pt, 0, lazy, [0, 1])
    assert a.nrows == b.nrows
    for c in range(3):
        np.testing.assert_array_equal(np.sort(a.read(c)), np.sort(b.read(c)))
    a.free(); b.free()
    assert lazy.nentries == eager.nentries == NBUILD and lazy.info() == info
    # gx_hash_agg_right rejects a payload-carrying table, deferred or not, with the same error
    plan = to_gpu_plan(O.make_plan(aggs=[(g.GX_AGG_COUNT_STAR, [])]))
    for h, tb in ((eager, te), (lazy, tl)):
        with pytest.raises(g.GxError):
            gx.hash_agg_right(pt, 0, tb, h, g.GX_JOIN_SEMI_RIGHT, plan)
    lazy.free(); tl.free()
    ok = outer_side(rng, keys, NBUILD + 100)
    x = rng.standard_normal(len(ok))
    ot = gx.table_from([g.GX_INT8, g.GX_FLOAT8], [ok, x])
    want, _, _ = agg(gx, ot, eager, plan_of())
    for change in ("append", "truncate"):
        h, tb = build(gx, keys, pay, spare=10)
        if change == "append":
            tb.append([np.array([keys[-1] + 1], np.int64), np.array([1], np.int32)])
        else:
            tb.truncate()
        got, ran, _ = agg(gx, ot, h, plan_of())
        assert "probe_agg_merge" not in ran, ran
        same(got, want)
        h.free(); tb.free()
    h, tb = build(gx, keys, pay)
    h.free()                                                     # never used
    tb.free()
    h, tb = build(gx, keys, pay)
    tb.free()                                                    # the table first: the handle is filled before it goes
    got, _, _ = agg(gx, ot, h, plan_of())
    same(got, want)
    h.free()
    eager.free(); te.free(); pt.free(); ot.free()


def test_group_table_overflow_retries_the_merge(gx):
    """est_groups far too low: the group table overflows and the merge runs again with a larger one"""
    rng = np.random.default_rng(5)
    keys = bunched(NBUILD)
    pay = dates(rng, NBUILD)
    ht, t = build(gx, keys, pay)
    ok = outer_side(rng, keys, NBUILD + 10)
    x = rng.standard_normal(len(ok))
    plan = plan_of(est=200)
    ot = gx.table_from([g.GX_INT8, g.GX_FLOAT8], [ok, x])
    got, ran, counts = agg(gx, ot, ht, plan)
    assert counts["probe_agg_merge"] >= 2 and "build_fill_staged" not in ran, counts
    want = J.expect_groups(plan, J.join(g.GX_JOIN_INNER, ok, keys), [ok, x], [g.GX_INT8, g.GX_FLOAT8], [pay], [g.GX_INT4])
    X.check(plan, want, got, [g.GX_INT4])
    ht.free(); t.free(); ot.free()
