"""The cross-datanode Finalize (gx_result_combine) on one GPU, against the exact reference of tests/exact_ref.py.

gx_debug_combine runs the Finalize's own code for one rank of N, with an in-process transport standing in for NCCL:
it builds on the device what the all-gather of segments, the count exchange and the all-to-all of records would have
delivered.  Each input is cut into N parts, every part is aggregated by gx_hash_agg as a datanode would, and every rank
0..N-1 is combined and fetched.  The union of the ranks' rows must be the exact answer over all rows, with each group on
exactly one rank; a finite union whose finite partials overflow when merged is GX_ERR_OVERFLOW.

Every case runs on both paths of the Finalize: the all-gathered segments (the default below the capacity limit) and
the record exchange (GX_NO_GATHER_COMBINE=1); the profile names combine_merge / combine_partition tell which ran."""
import ctypes

import numpy as np
import pytest

import opentenbase_b200 as g
import exact_ref as X

pytestmark = pytest.mark.gpu

C = g.GX_OP_COL
CNT = (g.GX_AGG_COUNT_STAR, [])


def col(fn, c):
    return (fn, [(C, c, 0)])


I32, I64 = np.iinfo(np.int32), np.iinfo(np.int64)
SEEN = set()                     # (path, what) pairs that ran somewhere in this module
PATHS = ["gathered", "records"]


@pytest.fixture(params=PATHS)
def path(request, monkeypatch):
    if request.param == "records":
        monkeypatch.setenv("GX_NO_GATHER_COMBINE", "1")
    return request.param


class Data:
    """rows of one relation (types, columns, NULL arrays or None) and the part of every row"""

    def __init__(self, types, cols, nulls, part):
        self.types, self.cols, self.part = types, [np.asarray(c) for c in cols], np.asarray(part, np.int64)
        self.nulls = [None if n is None else np.asarray(n, np.uint8) for n in nulls]

    def table(self, gx, p):
        rows = np.flatnonzero(self.part == p)
        cols = [c[rows] for c in self.cols]
        nulls = [None if n is None else n[rows] for n in self.nulls]
        return gx.table_from(self.types, cols, nulls if any(n is not None for n in nulls) else None)


def finalize(gx, nparts, aggregate, families=None):
    """aggregate(p) -> a fresh partial Result of part p.  Combines every rank over the parts; returns (the ranks'
    fetch() outputs or GxError, the profile names that ran per rank).  families: {part: profile name, or a tuple of
    them, that answered its aggregate (the first that ran is noted)}."""
    base = []
    for p in range(nparts):
        gx.profile(True)
        base.append(aggregate(p))
        if families and p in families:
            names = families[p] if isinstance(families[p], tuple) else (families[p],)
            ran = [n for n in names if gx.profile_get(n)[1] > 0]
            assert ran, f"part {p}: none of {names} answered"
            SEEN.add(("part", ran[0]))
        gx.profile(False)
    outs, ran = [], []
    for rank in range(nparts):
        mine = aggregate(rank)
        parts = base[:rank] + [mine] + base[rank + 1:]
        gx.profile(True)
        try:
            gx.debug_combine(parts, rank)
            outs.append(mine.fetch())
        except g.GxError as e:
            outs.append(e)
        ran.append({n for n in ("combine_merge", "combine_partition") if gx.profile_get(n)[1] > 0})
        gx.profile(False)
        mine.free()
    for r in base:
        r.free()
    return outs, ran


def union(outs):
    return tuple(np.concatenate([o[i] for o in outs]) for i in range(3))


def check_union(plan, want, outs, group_types):
    if want == "overflow":
        errs = [o for o in outs if isinstance(o, g.GxError)]
        assert errs, "the reference overflows, no rank did"
        assert all(e.status == g.GX_ERR_OVERFLOW for e in errs), errs
        return
    bad = [o for o in outs if isinstance(o, g.GxError)]
    assert not bad, bad[0]
    X.check(plan, want, union(outs), group_types)


def note_path(path, ran, nparts, big=False):
    """the path every rank took: gathered (merge only), records (partition only), or the fall-through (both)"""
    if nparts == 1:
        return
    want = {"combine_merge", "combine_partition"} if big else {"combine_partition"} if path == "records" else {"combine_merge"}
    for r, names in enumerate(ran):
        assert names == want, f"rank {r}: ran {sorted(names)}, want {sorted(want)}"
    SEEN.add((path, "anybig" if big else "direct"))


def run_scan(gx, path, data, plan, nparts, group_types, big=False, families=None):
    tables = [data.table(gx, p) for p in range(nparts)]
    outs, ran = finalize(gx, nparts, lambda p: gx.hash_agg(tables[p], plan), families)
    for t in tables:
        t.free()
    want = X.expect_groups(plan, data.cols, data.nulls, data.types)
    check_union(plan, want, outs, group_types)
    if want != "overflow":
        note_path(path, ran, nparts, big)
    return outs


# ---- aggregates and partial-state edges -------------------------------------------------------------------------
# columns: 0 key int4, 1 x float8 (nullable), 2 v int4 (nullable)
EVERY_AGG = [CNT, col(g.GX_AGG_COUNT, 1), col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_AVG_F8, 1), col(g.GX_AGG_MIN_F8, 1),
             col(g.GX_AGG_MAX_F8, 1), col(g.GX_AGG_SUM_I4, 2), col(g.GX_AGG_COUNT, 2)]
NAN, INF = float("nan"), float("inf")
N_ = None                        # a NULL input
# per group, per part: the x inputs of that part (None = NULL); parts beyond the list get nothing
STATE_GROUPS = [
    [[1.5, 2.25, -7.0]],                               # on one part only
    [[N_, N_], [3.0, 4.0]],                            # all NULL on one part, not on another
    [[N_], [N_, N_], [N_]],                            # all NULL everywhere: count 0, the rest NULL
    [[NAN, 1.0], [-5.0]],                              # NaN next to finite: max NaN, min finite
    [[NAN], [NAN, NAN]],                               # NaN-only partials
    [[-0.0, -0.0], [0.0]],                             # -0 only next to +0: sum +0
    [[-0.0], [-0.0, -0.0], [-0.0]],                    # -0 everywhere: sum -0
    [[INF, 1.0], [2.0]],                               # +inf in one partial: inf, not an error
    [[INF], [-INF]],                                   # +inf and -inf partials: NaN
    [[-INF, 3.0], [N_], [7.0]],
    [[1e150, 5.0], [-1e150]],                          # cancellation across parts
    [[0.1] * 40, [0.2] * 33, [0.3] * 7],
    [[], [], [6.0]],                                   # only on the last part
]


def state_data(nparts, rng):
    keys, xs, xn, part = [], [], [], []
    for gi, per_part in enumerate(STATE_GROUPS):
        for p, vals in enumerate(per_part):
            for v in vals:
                keys.append(gi * 7 - 3)
                xs.append(0.0 if v is None else v)
                xn.append(v is None)
                part.append(p % nparts)
    n = len(keys)
    v = rng.choice(np.array([I32.min, I32.max, -1, 0, 1], np.int32), n)
    vn = rng.random(n) < 0.2
    vn[np.array(keys) == 3 * 7 - 3] = True                # one group whose int4 inputs are all NULL
    o = rng.permutation(n)
    return Data([g.GX_INT4, g.GX_FLOAT8, g.GX_INT4],
                [np.array(keys, np.int32)[o], np.array(xs)[o], v[o]],
                [None, np.array(xn)[o], vn[o]], np.array(part)[o])


@pytest.mark.parametrize("nparts", [2, 3])
def test_partial_state_edges(gx, path, nparts):
    data = state_data(nparts, np.random.default_rng(nparts))
    for aggs in (EVERY_AGG, [col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_AVG_F8, 1)]):     # twins: sum and avg of one argument
        for est in (16, 1000):
            plan = g.make_plan(group_cols=[(0, 0)], aggs=aggs, est_groups=est)
            run_scan(gx, path, data, plan, nparts, [g.GX_INT4])


def test_combine_overflow_rule(gx, path):
    """two finite partial sums overflowing in the merge: GX_ERR_OVERFLOW on the rank that owns the group; an infinite
    partial merged with a finite one is infinite, and the other ranks answer"""
    types = [g.GX_INT4, g.GX_FLOAT8]
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[col(g.GX_AGG_SUM_F8, 1), CNT], est_groups=100)
    data = Data(types, [np.array([1, 1, 2, 2, 3], np.int32), np.array([1e308, 1e308, INF, 1e308, 1.0])], [None, None], [0, 1, 0, 1, 1])
    outs = run_scan(gx, path, data, plan, 2, [g.GX_INT4])
    assert sum(isinstance(o, g.GxError) for o in outs) == 1
    for aggs in ([col(g.GX_AGG_AVG_F8, 1)], [col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_AVG_F8, 1)]):
        run_scan(gx, path, data, g.make_plan(group_cols=[(0, 0)], aggs=aggs, est_groups=100), 2, [g.GX_INT4])
    # the same merge without the finite overflow: every rank answers, group 2 is +inf
    ok = Data(types, [np.array([1, 1, 2, 2, 3], np.int32), np.array([1e307, 1e307, INF, 1e308, 1.0])], [None, None], [0, 1, 0, 1, 1])
    run_scan(gx, path, ok, plan, 2, [g.GX_INT4])


# ---- group keys ---------------------------------------------------------------------------------------------------
def key_data(kind, n, rng):
    """(types, cols, nulls, group columns) for one kind of group key; x float8 and v int4 follow the key columns"""
    nan = np.float64(np.nan)
    if kind == "int4":
        k = [rng.choice(np.array([I32.min, -1, 0, 1, I32.max], np.int32), n)]
    elif kind == "int8":
        k = [rng.choice(np.array([I64.min, -1, 0, I64.max], np.int64), n)]
    elif kind == "date":
        k = [rng.choice(np.array([-2451545, -1, 0, 10957, 2147483494], np.int32), n)]
    elif kind == "char":
        k = [rng.choice(np.array([-128, -1, 0, 65, 127], np.int8), n)]
    elif kind == "float8":
        k = [rng.choice(np.array([0.0, -0.0, nan, -nan, 1.5, -INF]), n)]
    elif kind in ("nulls", "two_words"):
        k = [rng.choice(np.array([I32.min, 0, 5], np.int32), n), rng.choice(np.array([I64.min, -1, 7], np.int64), n),
             rng.choice(np.array([-3, 0, 9], np.int32), n)]
        if kind == "two_words":
            k = [rng.choice(np.array([I64.min, -1, 3], np.int64), n), rng.choice(np.array([I64.max, 0, -9], np.int64), n)]
    else:
        k = []
    types = {"int4": [g.GX_INT4], "int8": [g.GX_INT8], "date": [g.GX_DATE], "char": [g.GX_CHAR], "float8": [g.GX_FLOAT8],
             "nulls": [g.GX_INT4, g.GX_INT8, g.GX_DATE], "two_words": [g.GX_INT8, g.GX_INT8], "none": []}[kind]
    nulls = [None] * len(k)
    if kind == "nulls":
        nulls = [rng.random(n) < 0.3 for _ in k]               # a NULL in every group column position
    x = rng.random(n) * 100 - 50
    v = rng.integers(-1000, 1000, n).astype(np.int32)
    return types + [g.GX_FLOAT8, g.GX_INT4], k + [x, v], nulls + [None, None], list(range(len(k)))


KEY_KINDS = ["int4", "int8", "date", "char", "float8", "nulls", "two_words", "none"]


@pytest.mark.parametrize("kind", KEY_KINDS)
def test_group_keys(gx, path, kind):
    rng = np.random.default_rng(KEY_KINDS.index(kind))
    n, nparts = 3001, 3
    types, cols, nulls, gcols = key_data(kind, n, rng)
    nk = len(gcols)
    aggs = [CNT, col(g.GX_AGG_SUM_F8, nk), col(g.GX_AGG_SUM_I4, nk + 1), col(g.GX_AGG_MAX_F8, nk)]
    plan = g.make_plan(group_cols=[(0, c) for c in gcols], aggs=aggs, est_groups=64)
    data = Data(types, cols, nulls, rng.integers(0, nparts, n))
    outs = run_scan(gx, path, data, plan, nparts, [types[c] for c in gcols])
    if kind == "none":
        assert [o[0].shape[0] for o in outs] == [1, 0, 0], "a plain aggregate's one row comes from rank 0 only"


def test_group_key_from_a_join_payload(gx, path):
    """GROUP BY a payload column of the join's build side (side 1), int4 edge values, over an INNER join"""
    rng = np.random.default_rng(11)
    M, n, nparts = 500, 4000, 3
    pay = rng.choice(np.array([I32.min, -1, 0, 42, I32.max], np.int32), M)
    inner = gx.table_from([g.GX_INT8, g.GX_INT4], [np.arange(1, M + 1, dtype=np.int64), pay])
    ht = gx.hash_build(inner, 0, [1], unique=True)
    okey = rng.integers(1, M + 1, n).astype(np.int64)
    x = rng.random(n) - 0.5
    part = rng.integers(0, nparts, n)
    data = Data([g.GX_INT8, g.GX_FLOAT8], [okey, x], [None, None], part)
    aggs = [CNT, col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_MIN_F8, 1)]
    plan = g.make_plan(group_cols=[(1, 0)], aggs=aggs, est_groups=8)
    tables = [data.table(gx, p) for p in range(nparts)]
    outs, ran = finalize(gx, nparts, lambda p: gx.hash_agg_joins(tables[p], [(ht, (0, 0))], plan))
    for t in tables:
        t.free()
    ref_plan = g.make_plan(group_cols=[(0, 0)], aggs=aggs)
    want = X.expect_groups(ref_plan, [pay[okey - 1], x], None, [g.GX_INT4, g.GX_FLOAT8])
    check_union(plan, want, outs, [g.GX_INT4])
    note_path(path, ran, nparts)
    ht.free(); inner.free()


# ---- part shapes --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nparts", [1, 2, 3, 8, 64])
def test_part_counts(gx, path, nparts):
    rng = np.random.default_rng(nparts)
    n = 2000
    types, cols, nulls, _ = key_data("int4", n, rng)
    cols[0] = rng.integers(-300, 300, n).astype(np.int32)
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_AVG_F8, 1), col(g.GX_AGG_SUM_I4, 2)], est_groups=600)
    run_scan(gx, path, Data(types, cols, nulls, rng.integers(0, nparts, n)), plan, nparts, [g.GX_INT4])


@pytest.mark.parametrize("shape", ["one_empty", "all_empty", "one_holds_all"])
@pytest.mark.parametrize("grouped", [True, False], ids=["grouped", "plain"])
def test_part_shapes(gx, path, shape, grouped):
    """an empty table has no NULL arrays, and a result's record layout follows them: no NULL arrays here"""
    rng = np.random.default_rng(5)
    n, nparts = 0 if shape == "all_empty" else 1500, 3
    types = [g.GX_INT4, g.GX_FLOAT8, g.GX_INT4]
    cols = [rng.integers(0, 50, n).astype(np.int32), rng.random(n), rng.integers(-5, 5, n).astype(np.int32)]
    part = {"one_empty": rng.integers(1, nparts, n), "all_empty": np.zeros(0, np.int64), "one_holds_all": np.full(n, 1)}[shape]
    aggs = EVERY_AGG
    plan = g.make_plan(group_cols=[(0, 0)] if grouped else [], aggs=aggs, est_groups=64)
    outs = run_scan(gx, path, Data(types, cols, [None, None, None], part), plan, nparts, [g.GX_INT4])
    if not grouped:
        assert [o[0].shape[0] for o in outs] == [1, 0, 0]


# ---- the capacity switch -------------------------------------------------------------------------------------------
def groups_data(counts, rng, key_scale=3):
    """one row per (group, part) for counts[p] groups on part p, groups overlapping between parts"""
    keys, part = [], []
    for p, c in enumerate(counts):
        ks = rng.permutation(max(counts) + 16)[:c]
        keys.append(ks * key_scale - 1000); part.append(np.full(c, p))
    k = np.concatenate(keys).astype(np.int32)
    n = len(k)
    return Data([g.GX_INT4, g.GX_FLOAT8, g.GX_INT4], [k, rng.random(n), rng.integers(-9, 9, n).astype(np.int32)],
                [None, None, None], np.concatenate(part))


@pytest.mark.parametrize("most", [1024, 1025])
def test_segment_capacity(gx, path, most):
    """est_groups 512 gives segments of 1024 records: a part of exactly 1024 groups fits, one of 1025 makes every rank
    fall through to the record exchange"""
    data = groups_data([300, most, 0], np.random.default_rng(most))
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_SUM_I4, 2)], est_groups=512)
    run_scan(gx, path, data, plan, 3, [g.GX_INT4], big=path == "gathered" and most > 1024)


@pytest.mark.parametrize("est", [32768, 32769])
def test_capacity_limit(gx, path, est):
    """est_groups 32768 gives segments of 65536 records, the limit; 32769 goes to the record exchange directly"""
    data = groups_data([2000, 1500], np.random.default_rng(est))
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(g.GX_AGG_SUM_F8, 1)], est_groups=est)
    tables = [data.table(gx, p) for p in range(2)]
    outs, ran = finalize(gx, 2, lambda p: gx.hash_agg(tables[p], plan))
    for t in tables:
        t.free()
    check_union(plan, X.expect_groups(plan, data.cols, data.nulls, data.types), outs, [g.GX_INT4])
    gathered = path == "gathered" and est == 32768
    assert all(r == ({"combine_merge"} if gathered else {"combine_partition"}) for r in ran), ran


def test_estimate_far_below_the_truth(gx, path):
    """est_groups 4 against 6000 groups per part: the parts' own aggregates retry, the segments do not fit"""
    data = groups_data([6000, 5000, 100], np.random.default_rng(9))
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_MIN_F8, 1)], est_groups=4)
    run_scan(gx, path, data, plan, 3, [g.GX_INT4], big=path == "gathered")


def test_a_million_groups_over_four_parts(gx, path):
    """the record exchange at size: about 1 M groups, so the radix merge takes several partitions; checked against an
    exact integer reference (float8 values are small integers, so every order of summation is exact)"""
    rng = np.random.default_rng(12)
    G, nparts = 1_000_000, 4
    rows = np.concatenate([np.arange(G), rng.integers(0, G, G // 2)])
    keys = (rows * 2654435761 % (1 << 40) - (1 << 39)).astype(np.int64)
    x = rng.integers(-1000, 1000, len(rows)).astype(np.float64)
    part = rng.integers(0, nparts, len(rows))
    tables = [gx.table_from([g.GX_INT8, g.GX_FLOAT8], [keys[part == p], x[part == p]]) for p in range(nparts)]
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_MAX_F8, 1)], est_groups=G)
    outs, ran = finalize(gx, nparts, lambda p: gx.hash_agg(tables[p], plan))
    for t in tables:
        t.free()
    assert all(r == {"combine_partition"} for r in ran), ran
    k, a, nl = union(outs)
    assert len(k) == G and len(np.unique(k[:, 0])) == G and not nl.any()
    o = np.argsort(k[:, 0])
    uk, inv = np.unique(keys, return_inverse=True)
    assert np.array_equal(k[o, 0], uk)
    assert np.array_equal(a[o, 0].view(np.int64), np.bincount(inv, minlength=G))
    assert np.array_equal(a[o, 1], np.bincount(inv, weights=x, minlength=G))
    mx = np.full(G, -np.inf); np.maximum.at(mx, inv, x)
    assert np.array_equal(a[o, 2], mx)
    SEEN.add((path, "size"))


def test_fetch_paths(gx, path):
    """8192 combined groups are finalized on the host, 8193 on the device (gx_k_finalize).  16385 groups over two
    ranks put one rank on each side of that split."""
    rng = np.random.default_rng(17)
    G = 16385
    gi = np.concatenate([np.arange(G), rng.integers(0, G, 4000)])
    gkeys = [(int(k),) for k in np.arange(G) * 5 - 40000]
    x = rng.choice(np.array([1.0, -0.0, 0.0, INF, NAN, 2.5]), len(gi))
    xn = rng.random(len(gi)) < 0.2
    data = Data([g.GX_INT4, g.GX_FLOAT8], [(gi * 5 - 40000).astype(np.int32), x], [None, xn], rng.integers(0, 2, len(gi)))
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(g.GX_AGG_COUNT, 1), col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_MAX_F8, 1)], est_groups=G)
    tables = [data.table(gx, p) for p in range(2)]
    outs, ran = finalize(gx, 2, lambda p: gx.hash_agg(tables[p], plan))
    for t in tables:
        t.free()
    sizes = sorted(o[0].shape[0] for o in outs)
    assert sizes[0] <= 8192 < sizes[1], sizes
    check_union(plan, X.expect_groups(plan, data.cols, data.nulls, data.types, gindex=gi, gkeys=gkeys), outs, [g.GX_INT4])
    note_path(path, ran, 2)


# ---- parts answered by different kernel families (one plan) -------------------------------------------------------
GENERAL = ("agg_smem", "agg_lptile8", "agg_lptile4", "agg_smem_lp", "agg_fast", "agg_global", "scan_records")


def test_run_aggregate_next_to_the_general_kernel(gx, path):
    """sum(x) GROUP BY the join key with x NOT NULL keeps no row count (need_w0 = 0).  Part 0 has its outer side in key
    order (gx_k_runagg), part 1 the same kind of rows permuted (gx_k_agg); groups seen only by part 1 must keep their
    sums on whichever rank owns them"""
    rng = np.random.default_rng(13)
    M = 3000
    inner = gx.table_from([g.GX_INT8, g.GX_INT4], [np.arange(1, M + 1, dtype=np.int64), np.zeros(M, np.int32)])
    ht = gx.hash_build(inner, 0, [1], unique=True)
    k0 = np.sort(rng.integers(1, 1500, 20000)).astype(np.int64)
    k1 = rng.permutation(np.concatenate([np.arange(1000, M + 1), rng.integers(1, M + 1, 5000)])).astype(np.int64)
    keys = np.concatenate([k0, k1])
    x = rng.random(len(keys)) * 10
    data = Data([g.GX_INT8, g.GX_FLOAT8], [keys, x], [None, None], np.r_[np.zeros(len(k0)), np.ones(len(k1))])
    tables = [data.table(gx, p) for p in range(2)]
    for aggs in ([col(g.GX_AGG_SUM_F8, 1)], [col(g.GX_AGG_SUM_F8, 1), CNT]):
        plan = g.make_plan(outer_key_col=0, group_cols=[(0, 0)], aggs=aggs, est_groups=1500)
        outs, ran = finalize(gx, 2, lambda p: gx.hash_agg(tables[p], plan, ht), {0: "runagg_dense", 1: "agg_smem"})
        check_union(plan, X.expect_groups(plan, data.cols, data.nulls, data.types), outs, [g.GX_INT8])
        note_path(path, ran, 2)
    for t in tables:
        t.free()
    ht.free(); inner.free()


def test_strategy_1_next_to_strategy_2(gx, path):
    """one plan, est_groups 1000: a part of 300 groups stays in the shared-memory table, a part of 40000 groups
    outgrows it and is aggregated by the radix path"""
    rng = np.random.default_rng(14)
    data = groups_data([300, 40000], rng, key_scale=1)
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_AVG_F8, 1), col(g.GX_AGG_MIN_F8, 1)], est_groups=1000)
    tables = [data.table(gx, p) for p in range(2)]
    outs, ran = finalize(gx, 2, lambda p: gx.hash_agg(tables[p], plan), {0: "agg_smem", 1: "scan_records"})
    for t in tables:
        t.free()
    check_union(plan, X.expect_groups(plan, data.cols, data.nulls, data.types), outs, [g.GX_INT4])
    note_path(path, ran, 2, big=path == "gathered")


def test_few_group_kernel_next_to_the_general_one(gx, path):
    """one plan, est_groups 4: a part of 3 groups is answered by the register kernel (gx_k_fewgroups), a part of 60
    groups by a general kernel after the register kernel gave up"""
    rng = np.random.default_rng(15)
    data = groups_data([3, 60], rng, key_scale=1)
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[col(g.GX_AGG_SUM_F8, 1), col(g.GX_AGG_AVG_F8, 1), CNT], est_groups=4)
    tables = [data.table(gx, p) for p in range(2)]
    outs, ran = finalize(gx, 2, lambda p: gx.hash_agg(tables[p], plan), {0: "agg_fewgroups", 1: GENERAL})
    for t in tables:
        t.free()
    check_union(plan, X.expect_groups(plan, data.cols, data.nulls, data.types), outs, [g.GX_INT4])
    note_path(path, ran, 2)


# ---- errors -------------------------------------------------------------------------------------------------------
def test_errors_leave_the_context_usable(gx):
    rng = np.random.default_rng(16)
    t = gx.table_from([g.GX_INT4, g.GX_FLOAT8, g.GX_INT4], [rng.integers(0, 9, 100).astype(np.int32), rng.random(100), np.ones(100, np.int32)])
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(g.GX_AGG_SUM_F8, 1)], est_groups=16)

    def arg_error(parts, rank):
        with pytest.raises(g.GxError) as ei:
            gx.debug_combine(parts, rank)
        assert ei.value.status == g.GX_ERR_ARG, ei.value

    for fn, c in ((g.GX_AGG_COUNT_DISTINCT, 2), (g.GX_AGG_VAR_SAMP_F8, 1), (g.GX_AGG_STDDEV_POP_F8, 1)):
        p = g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(fn, c)], est_groups=16)
        parts = [gx.hash_agg(t, p) for _ in range(2)]
        arg_error(parts, 0)
        gx.debug_combine(parts[:1], 0)                     # one rank: nothing to combine
        for r in parts:
            r.free()
    a, b = gx.hash_agg(t, plan), gx.hash_agg(t, g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(g.GX_AGG_SUM_F8, 1)], est_groups=17))
    arg_error([a, b], 0)                                   # the plans differ
    c = gx.hash_agg(t, g.make_plan(group_cols=[(0, 0)], aggs=[CNT, col(g.GX_AGG_SUM_F8, 1)], est_groups=16))
    for rank in (-1, 2):
        arg_error([a, c], rank)
    arg_error([a] * 65, 0)
    assert g.lib().gx_debug_combine(gx.h, 0, (ctypes.c_void_p * 1)(a.h), 0) == g.GX_ERR_ARG
    gx.debug_combine([a, c], 1)
    arg_error([a, c], 0)                                   # c was combined already
    for r in (a, b, c):
        r.free()
    # still usable: a clean combine
    parts = [gx.hash_agg(t, plan) for _ in range(2)]
    outs = []
    for rank in range(2):
        mine = gx.hash_agg(t, plan)
        gx.debug_combine([mine if i == rank else parts[i] for i in range(2)], rank)
        outs.append(mine.fetch())
        mine.free()
    data = Data(t.types, [t.read(0), t.read(1), t.read(2)], [None] * 3, np.zeros(100))
    both = Data(t.types, [np.concatenate([c, c]) for c in data.cols], [None] * 3, np.zeros(200))
    X.check(plan, X.expect_groups(plan, both.cols, both.nulls, both.types), union(outs), [g.GX_INT4])
    for r in parts:
        r.free()
    t.free()


def test_zz_every_path_and_family_ran(request):
    """runs last: every path of the Finalize and every kernel family of the mixed cases answered somewhere.  Judged
    only when the whole module was selected."""
    ids = {it.nodeid.split("::")[-1] for it in request.session.items}
    need = ["test_segment_capacity[gathered-1025]", "test_a_million_groups_over_four_parts[records]",
            "test_run_aggregate_next_to_the_general_kernel[gathered]", "test_few_group_kernel_next_to_the_general_one[records]"]
    if not all(n in ids for n in need):
        pytest.skip("not every test of the module was selected")
    want = {("gathered", "direct"), ("gathered", "anybig"), ("records", "direct"), ("gathered", "size"), ("records", "size")}
    want |= {("part", f) for f in ("runagg_dense", "agg_smem", "scan_records", "agg_fewgroups")}
    assert SEEN >= want, f"never ran: {sorted(want - SEEN)}"
