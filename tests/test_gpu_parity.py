"""Parity of the CUDA path (through the C ABI of libgpuexec.so) against the CPU
oracle on the same seeded inputs.  Integer/byte/index work is bit-exact; float8
aggregates are held to 1e-9 relative (the north-star tolerance)."""
import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
from helpers import assert_agg_equal, to_gpu_plan, lineitem_rel, orders_rel

pytestmark = pytest.mark.gpu

SF = 1
NORD = 20000          # orders generated for the small parity cases (~80k lineitem rows)


@pytest.fixture(scope="module")
def data(gx):
    o = O.gen_orders(SF, 0, NORD)
    l = O.gen_lineitem(SF, 0, NORD)
    return {
        "o": o, "l": l,
        "orel": orders_rel(o), "lrel": lineitem_rel(l),
        "ot": gx.table_from(g.SCHEMAS[g.T_ORDERS], o),
        "lt": gx.table_from(g.SCHEMAS[g.T_LINEITEM], l),
    }


# ---------------------------------------------------------------- hashes
def test_device_hashes_match_oracle(gx):
    L = O.lib()
    rng = np.random.default_rng(7)
    v4 = np.concatenate([np.array([0, 1, 17, 42, 550273, 207112489, -1, -2**31, 2**31 - 1]),
                         rng.integers(-2**31, 2**31, 2000)]).astype(np.int64)
    v8 = np.concatenate([np.array([0, 1, 2**32 + 1, -1, -2**63, 2**63 - 1, -2**32]),
                         rng.integers(-2**63, 2**63 - 1, 2000)]).astype(np.int64)
    np.testing.assert_array_equal(gx.debug_hash(1, v4), [L.orc_hashint4(int(x)) for x in v4])
    np.testing.assert_array_equal(gx.debug_hash(2, v8), [L.orc_hashint8(int(x)) for x in v8])
    np.testing.assert_array_equal(gx.debug_hash(3, v4), [L.orc_hashint4new(int(x)) for x in v4])
    np.testing.assert_array_equal(gx.debug_hash(4, v8), [L.orc_hashint8new(int(x)) for x in v8])
    u = (v4 & 0xFFFFFFFF)
    np.testing.assert_array_equal(gx.debug_hash(5, u), [L.orc_murmurhash32(int(x)) for x in u])
    # the upstream KAT hashint4(1) = -1905060026
    assert int(gx.debug_hash(1, [1])[0]) - (1 << 32) == -1905060026


# ------------------------------------------------------------- generator
@pytest.mark.parametrize("node,nnodes", [(0, 1), (1, 4), (3, 4)])
def test_device_generator_matches_host(gx, node, nnodes):
    gx.set_shardmap(nnodes)
    for tid, gen in ((g.T_ORDERS, O.gen_orders), (g.T_LINEITEM, O.gen_lineitem), (g.T_CUSTOMER, O.gen_customer)):
        want = gen(SF, 100, 5100, node, nnodes)
        t = gx.table(g.SCHEMAS[tid], max(len(want[0]), 1) + 16)
        t.generate(tid, SF, 100, 5100, node, nnodes)
        assert t.nrows == len(want[0])
        for c, w in enumerate(want):
            got = t.read(c)
            if got.dtype == np.float64:
                np.testing.assert_array_equal(got.view(np.int64), w.view(np.int64))   # bit-identical doubles
            else:
                np.testing.assert_array_equal(got, w)
        t.free()
    gx.set_shardmap(1)


# --------------------------------------------------- configs 1, 2 (no join)
@pytest.mark.parametrize("strategy", [1, 2, 3])
def test_config1_count_by_returnflag(gx, data, strategy):
    plan = O.make_plan(group_cols=[(0, g.L_RETURNFLAG)], aggs=[(g.GX_AGG_COUNT_STAR, [])], est_groups=3, strategy=strategy)
    want = O.exec_agg(data["lrel"], plan)
    res = gx.hash_agg(data["lt"], to_gpu_plan(plan))
    assert_agg_equal(plan, res.fetch(), want)
    assert res.fetch()[1].view(np.int64).sum() == data["lt"].nrows


@pytest.mark.parametrize("strategy", [1, 2, 3])
def test_config2_sum_by_shipdate(gx, data, strategy):
    plan = O.make_plan(group_cols=[(0, g.L_SHIPDATE)],
                       aggs=[(g.GX_AGG_SUM_F8, [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0)])], est_groups=2600, strategy=strategy)
    want = O.exec_agg(data["lrel"], plan)
    assert_agg_equal(plan, gx.hash_agg(data["lt"], to_gpu_plan(plan)).fetch(), want)


def test_q1_shape(gx, data):
    """TPC-H Q1: filter, two "char" group columns, eight aggregates with expressions."""
    C, K, A, S, M = g.GX_OP_COL, g.GX_OP_CONST, g.GX_OP_ADD, g.GX_OP_SUB, g.GX_OP_MUL
    disc_price = [(C, g.L_EXTENDEDPRICE, 0), (K, 0, 1.0), (C, g.L_DISCOUNT, 0), (S, 0, 0), (M, 0, 0)]
    charge = disc_price + [(K, 0, 1.0), (C, g.L_TAX, 0), (A, 0, 0), (M, 0, 0)]
    plan = O.make_plan(
        preds=[(g.L_SHIPDATE, g.GX_LE, -517 - 90)],
        group_cols=[(0, g.L_RETURNFLAG), (0, g.L_LINESTATUS)],
        aggs=[(g.GX_AGG_SUM_F8, [(C, g.L_QUANTITY, 0)]), (g.GX_AGG_SUM_F8, [(C, g.L_EXTENDEDPRICE, 0)]),
              (g.GX_AGG_SUM_F8, disc_price), (g.GX_AGG_SUM_F8, charge),
              (g.GX_AGG_AVG_F8, [(C, g.L_QUANTITY, 0)]), (g.GX_AGG_AVG_F8, [(C, g.L_EXTENDEDPRICE, 0)]),
              (g.GX_AGG_AVG_F8, [(C, g.L_DISCOUNT, 0)]), (g.GX_AGG_COUNT_STAR, [])],
        est_groups=6)
    want = O.exec_agg(data["lrel"], plan)
    assert want.ngroups == 4
    for strategy in (1, 2):
        plan.strategy = strategy
        assert_agg_equal(plan, gx.hash_agg(data["lt"], to_gpu_plan(plan)).fetch(), want)


def test_plain_aggregate_and_minmax(gx, data):
    plan = O.make_plan(aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, g.L_QUANTITY, 0)]),
                             (g.GX_AGG_MIN_F8, [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0)]),
                             (g.GX_AGG_MAX_F8, [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0)]),
                             (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, g.L_SHIPDATE, 0)])])
    # SUM_I4 wants an int4 column: use a table with one
    cols = [data["l"][g.L_QUANTITY], data["l"][g.L_EXTENDEDPRICE], (data["l"][g.L_SHIPDATE] % 1000).astype(np.int32)]
    types = [g.GX_FLOAT8, g.GX_FLOAT8, g.GX_INT4]
    plan = O.make_plan(aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 0, 0)]),
                             (g.GX_AGG_MIN_F8, [(g.GX_OP_COL, 1, 0)]), (g.GX_AGG_MAX_F8, [(g.GX_OP_COL, 1, 0)]),
                             (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 2, 0)])])
    want = O.exec_agg(O.Rel(types, cols), plan)
    assert_agg_equal(plan, gx.hash_agg(gx.table_from(types, cols), to_gpu_plan(plan)).fetch(), want)


# --------------------------------------------------------- config 3 (join)
@pytest.mark.parametrize("strategy", [1, 2, 3])
def test_config3_join_groupby(gx, data, strategy):
    """lineitem JOIN orders ON l_orderkey = o_orderkey GROUP BY o_orderdate: count(*), sum(l_extendedprice)"""
    plan = O.make_plan(outer_key_col=g.L_ORDERKEY, group_cols=[(1, 0)],
                       aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0)])],
                       est_groups=2500, strategy=strategy)
    join = O.make_join(g.O_ORDERKEY, payload_cols=[g.O_ORDERDATE], inner_unique=1)
    want = O.exec_agg(data["lrel"], plan, data["orel"], join)
    ht = gx.hash_build(data["ot"], g.O_ORDERKEY, [g.O_ORDERDATE], unique=True)
    assert ht.nentries == NORD
    got = gx.hash_agg(data["lt"], to_gpu_plan(plan), ht).fetch()
    assert_agg_equal(plan, got, want)
    assert got[1][:, 0].view(np.int64).sum() == data["lt"].nrows      # every line finds its order


@pytest.mark.parametrize("layout", ["key_order", "shuffled", "key_order_filtered", "clustered", "key_order_no_payload",
                                    "key_order_wide_span", "shuffled_wide_span", "key_order_no_payload_wide_span",
                                    "key_order_grouped_twice"])
def test_big_build_paths_agree_with_oracle(gx, layout, monkeypatch):
    """Build sides large enough for the sub-table builders (>= 64 sub-tables): the
    partition-free path for a build side stored in key order, the two-level bucketing
    path for an unordered one, and the fall-back to the mixing hash when the keys are
    clustered — all three must give the oracle's join (nodeHash.c:1828, nodeHashjoin.c:446)."""
    nord = 200_000
    if layout.endswith("_wide_span"):
        # what a key span above 2^32 selects (8 datanodes at SF100 each): 64-bit interpolation
        # arithmetic and 16-byte slots instead of the 32-bit / compact forms
        monkeypatch.setenv("GX_SLOT_WIDE", "1")
        layout = layout[:-len("_wide_span")]
    o, l = O.gen_orders(SF, 0, nord), O.gen_lineitem(SF, 0, nord)
    o = [c.copy() for c in o]; l = [c.copy() for c in l]
    inner_preds = []
    if layout == "shuffled":
        perm = np.random.default_rng(7).permutation(nord)
        o = [c[perm] for c in o]
        lperm = np.random.default_rng(8).permutation(len(l[0]))      # outer side without key runs as well
        l = [c[lperm] for c in l]
    elif layout == "key_order_filtered":
        inner_preds = [(g.O_ORDERDATE, g.GX_LT, -1752)]
    elif layout == "clustered":                       # ascending but bunched: half the keys in a narrow band
        k = o[g.O_ORDERKEY]
        remap = np.where(k % 2 == 0, k // 64, k)
        o[g.O_ORDERKEY] = np.sort(remap)
        l[g.L_ORDERKEY] = np.where(l[g.L_ORDERKEY] % 2 == 0, l[g.L_ORDERKEY] // 64, l[g.L_ORDERKEY])
    payload = [g.O_ORDERDATE]
    group_cols = [(1, 0)]
    if layout == "key_order_no_payload":              # the join only filters: half the orders are kept out of the build side
        payload, group_cols = [], [(0, g.L_SHIPDATE)]
        o = [c[::2].copy() for c in o]
    elif layout == "key_order_grouped_twice":         # GROUP BY o_orderdate, o_orderdate: two group columns, one payload slot
        group_cols = [(1, 0), (1, 0)]
    plan = O.make_plan(outer_key_col=g.L_ORDERKEY, group_cols=group_cols,
                       aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0)])],
                       est_groups=2600)
    uniq = layout != "clustered"                     # unique build keys take the specialised probe kernels
    join = O.make_join(g.O_ORDERKEY, payload_cols=payload, inner_unique=int(uniq), inner_preds=inner_preds)
    want = O.exec_agg(lineitem_rel(l), plan, orders_rel(o), join)
    ot = gx.table_from(g.SCHEMAS[g.T_ORDERS], o); lt = gx.table_from(g.SCHEMAS[g.T_LINEITEM], l)
    ht = gx.hash_build(ot, g.O_ORDERKEY, payload, unique=uniq, preds=inner_preds)
    info = ht.info()
    if layout in ("key_order", "key_order_filtered", "key_order_no_payload", "key_order_grouped_twice"):
        assert info["slot_mode"] == 2, info          # partition-free key-ordered build
    elif layout == "shuffled":
        assert info["slot_mode"] == 1, info          # interpolation slots, bucketed build
    got = gx.hash_agg(lt, to_gpu_plan(plan), ht).fetch()
    assert_agg_equal(plan, got, want)


def test_q3_shape_two_word_key(gx, data):
    """GROUP BY l_orderkey, o_orderdate, o_shippriority: 16-byte key, many groups -> radix."""
    C, K, S, M = g.GX_OP_COL, g.GX_OP_CONST, g.GX_OP_SUB, g.GX_OP_MUL
    rev = [(C, g.L_EXTENDEDPRICE, 0), (K, 0, 1.0), (C, g.L_DISCOUNT, 0), (S, 0, 0), (M, 0, 0)]
    plan = O.make_plan(preds=[(g.L_SHIPDATE, g.GX_GT, -1752)], outer_key_col=g.L_ORDERKEY,
                       group_cols=[(0, g.L_ORDERKEY), (1, 0), (1, 1)],
                       aggs=[(g.GX_AGG_SUM_F8, rev)], est_groups=NORD)
    join = O.make_join(g.O_ORDERKEY, payload_cols=[g.O_ORDERDATE, g.O_SHIPPRIORITY], inner_unique=1,
                       inner_preds=[(g.O_ORDERDATE, g.GX_LT, -1752)])
    want = O.exec_agg(data["lrel"], plan, data["orel"], join)
    assert want.ngroups > 500
    ht = gx.hash_build(data["ot"], g.O_ORDERKEY, [g.O_ORDERDATE, g.O_SHIPPRIORITY], unique=True,
                       preds=[(g.O_ORDERDATE, g.GX_LT, -1752)])
    for strategy in (0, 2, 3):
        plan.strategy = strategy
        assert_agg_equal(plan, gx.hash_agg(data["lt"], to_gpu_plan(plan), ht).fetch(), want)


def test_join_materialised(gx, data):
    join = O.make_join(g.O_ORDERKEY, payload_cols=[g.O_ORDERDATE, g.O_SHIPPRIORITY], inner_unique=1)
    want = O.exec_join(data["lrel"], g.L_ORDERKEY, data["orel"], join, [g.L_ORDERKEY, g.L_SHIPDATE],
                       outer_preds=[(g.L_QUANTITY, g.GX_LT, 10.0, True)])
    ht = gx.hash_build(data["ot"], g.O_ORDERKEY, [g.O_ORDERDATE, g.O_SHIPPRIORITY], unique=True)
    t = gx.hash_probe(data["lt"], g.L_ORDERKEY, ht, [g.L_ORDERKEY, g.L_SHIPDATE],
                      preds=[(g.L_QUANTITY, g.GX_LT, 10.0, True)])
    got = [t.read(c).astype(np.int64) for c in range(4)]
    assert t.nrows == len(want[0])
    order_w = np.lexsort(want[::-1]); order_g = np.lexsort(got[::-1])
    for w, x in zip(want, got):
        np.testing.assert_array_equal(x[order_g], w[order_w])


def test_join_duplicates_and_special_key(gx):
    """N:M join: duplicate build keys, unmatched probes, and the key INT64_MIN
    (the empty-slot marker of the table) on both sides."""
    rng = np.random.default_rng(3)
    I64MIN = -2**63
    bkeys = np.concatenate([rng.integers(0, 500, 3000), [I64MIN, I64MIN, 7, 7, 7]]).astype(np.int64)
    bval = np.arange(len(bkeys), dtype=np.int32)
    pkeys = np.concatenate([rng.integers(-50, 700, 5000), [I64MIN, 7]]).astype(np.int64)
    pval = np.arange(len(pkeys), dtype=np.int32)
    bt, pt = [g.GX_INT8, g.GX_INT4], [g.GX_INT8, g.GX_INT4]
    join = O.make_join(0, payload_cols=[1], inner_unique=0)
    want = O.exec_join(O.Rel(pt, [pkeys, pval]), 0, O.Rel(bt, [bkeys, bval]), join, [0, 1])
    ht = gx.hash_build(gx.table_from(bt, [bkeys, bval]), 0, [1], unique=False)
    assert ht.nentries == len(bkeys)
    t = gx.hash_probe(gx.table_from(pt, [pkeys, pval]), 0, ht, [0, 1])
    got = [t.read(c).astype(np.int64) for c in range(3)]
    assert t.nrows == len(want[0])
    ow, og = np.lexsort(want[::-1]), np.lexsort(got[::-1])
    for w, x in zip(want, got):
        np.testing.assert_array_equal(x[og], w[ow])
    # and fused into an aggregate
    plan = O.make_plan(outer_key_col=0, group_cols=[(0, 0)], aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 1, 0)])],
                       est_groups=600)
    wagg = O.exec_agg(O.Rel(pt, [pkeys, pval]), plan, O.Rel(bt, [bkeys, bval]), join)
    for strategy in (1, 2):
        plan.strategy = strategy
        assert_agg_equal(plan, gx.hash_agg(gx.table_from(pt, [pkeys, pval]), to_gpu_plan(plan), ht).fetch(), wagg)


# ------------------------------------------------------------------ NULLs
def test_null_semantics(gx):
    """NULL join keys never match (hashStrict); NULL group keys form one group;
    strict transition functions skip NULL inputs; sum over only-NULLs is NULL."""
    rng = np.random.default_rng(11)
    n = 6000
    key = rng.integers(0, 40, n).astype(np.int64)
    grp = rng.integers(0, 7, n).astype(np.int32)
    val = rng.normal(100, 30, n)
    ival = rng.integers(-1000, 1000, n).astype(np.int32)
    nulls = [rng.random(n) < 0.1, rng.random(n) < 0.15, rng.random(n) < 0.2, rng.random(n) < 0.2]
    nulls[2][grp == 3] = True                     # group 3: every float input NULL -> SUM NULL, COUNT(col) 0
    nulls = [x.astype(np.uint8) for x in nulls]
    types = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8, g.GX_INT4]
    bkey = np.arange(0, 30, dtype=np.int64); bpay = (bkey * 3).astype(np.int32)
    bnull = [(bkey % 11 == 5).astype(np.uint8), None]
    aggs = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_COUNT, [(g.GX_OP_COL, 2, 0)]),
            (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)]), (g.GX_AGG_AVG_F8, [(g.GX_OP_COL, 2, 0)]),
            (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 3, 0)]), (g.GX_AGG_MIN_F8, [(g.GX_OP_COL, 2, 0)]),
            (g.GX_AGG_MAX_F8, [(g.GX_OP_COL, 2, 0)])]
    orel = O.Rel(types, [key, grp, val, ival], nulls)
    gt = gx.table_from(types, [key, grp, val, ival], nulls)
    # no join
    plan = O.make_plan(group_cols=[(0, 1)], aggs=aggs, est_groups=16)
    want = O.exec_agg(orel, plan)
    assert want.nulls[:, 0].sum() == 1            # one NULL group
    for strategy in (1, 2, 3):
        plan.strategy = strategy
        assert_agg_equal(plan, gx.hash_agg(gt, to_gpu_plan(plan)).fetch(), want)
    # with a join whose keys carry NULLs on both sides
    plan = O.make_plan(outer_key_col=0, group_cols=[(0, 1), (1, 0)], aggs=aggs, est_groups=300)
    join = O.make_join(0, payload_cols=[1], inner_unique=1)
    irel = O.Rel([g.GX_INT8, g.GX_INT4], [bkey, bpay], bnull)
    want = O.exec_agg(orel, plan, irel, join)
    ht = gx.hash_build(gx.table_from([g.GX_INT8, g.GX_INT4], [bkey, bpay], bnull), 0, [1], unique=True)
    assert ht.nentries == int((bnull[0] == 0).sum())
    for strategy in (1, 2):
        plan.strategy = strategy
        assert_agg_equal(plan, gx.hash_agg(gt, to_gpu_plan(plan), ht).fetch(), want)


def test_empty_and_ragged_inputs(gx):
    types = [g.GX_INT8, g.GX_FLOAT8]
    empty = gx.table(types, 4)
    plan = O.make_plan(aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])])
    want = O.exec_agg(O.Rel(types, [np.zeros(0, np.int64), np.zeros(0)]), plan)
    assert want.ngroups == 1 and want.nulls[0, 1] == 1          # count 0, sum NULL
    assert_agg_equal(plan, gx.hash_agg(empty, to_gpu_plan(plan)).fetch(), want)
    plan = O.make_plan(group_cols=[(0, 0)], aggs=[(g.GX_AGG_COUNT_STAR, [])], est_groups=4)
    res = gx.hash_agg(empty, to_gpu_plan(plan))
    assert res.ngroups == 0
    ht = gx.hash_build(empty, 0, [], unique=True)
    assert ht.nentries == 0
    # ragged sizes around the vector / block boundaries
    for n in (1, 31, 33, 511, 513, 2049):
        k = (np.arange(n) % 5).astype(np.int64); v = np.arange(n, dtype=np.float64) * 0.25
        plan = O.make_plan(group_cols=[(0, 0)], aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])], est_groups=5)
        want = O.exec_agg(O.Rel(types, [k, v]), plan)
        for strategy in (1, 2):
            plan.strategy = strategy
            assert_agg_equal(plan, gx.hash_agg(gx.table_from(types, [k, v]), to_gpu_plan(plan)).fetch(), want)


def test_group_estimate_too_low_is_survived(gx, data):
    """The planner's numGroups can be badly wrong; the result must not depend on it."""
    plan = O.make_plan(group_cols=[(0, g.L_ORDERKEY)], aggs=[(g.GX_AGG_COUNT_STAR, [])], est_groups=2)
    want = O.exec_agg(data["lrel"], plan)
    assert want.ngroups == NORD
    assert_agg_equal(plan, gx.hash_agg(data["lt"], to_gpu_plan(plan)).fetch(), want)


# ---------------------------------------------------------------- scan (K1)
def test_scan_filter(gx, data):
    t = gx.scan_filter(data["lt"], [(g.L_SHIPDATE, g.GX_GT, -1000), (g.L_DISCOUNT, g.GX_LE, 0.05, True)],
                       [g.L_ORDERKEY, g.L_EXTENDEDPRICE, g.L_RETURNFLAG])
    l = data["l"]
    m = (l[g.L_SHIPDATE] > -1000) & (l[g.L_DISCOUNT] <= 0.05)
    assert t.nrows == int(m.sum())
    np.testing.assert_array_equal(t.read(0), l[g.L_ORDERKEY][m])        # K1 keeps scan order
    np.testing.assert_array_equal(t.read(1).view(np.int64), l[g.L_EXTENDEDPRICE][m].view(np.int64))
    np.testing.assert_array_equal(t.read(2), l[g.L_RETURNFLAG][m])


# ------------------------------------------------------------ routing (K5)
@pytest.mark.parametrize("nnodes", [2, 4, 8])
def test_route_bit_exact_with_reference_rule(gx, data, nnodes):
    gx.set_shardmap(nnodes)
    got = gx.route(data["ot"], g.O_ORDERKEY)
    np.testing.assert_array_equal(got, O.route_nodes(data["o"][0], O.GX_INT8, nnodes))
    got4 = gx.route(data["ot"], g.O_CUSTKEY)
    np.testing.assert_array_equal(got4, O.route_nodes(data["o"][1], O.GX_INT4, nnodes))
    part, counts = gx.partition_by_node(data["ot"], g.O_CUSTKEY, nnodes)
    assert counts.sum() == NORD
    np.testing.assert_array_equal(counts, np.bincount(got4, minlength=nnodes))
    # each destination's slice holds exactly that destination's rows (as a multiset)
    ck, ok = part.read(g.O_CUSTKEY), part.read(g.O_ORDERKEY)
    off = 0
    for n in range(nnodes):
        sl = slice(off, off + counts[n]); off += counts[n]
        assert (O.route_nodes(ck[sl], O.GX_INT4, nnodes) == n).all()
        np.testing.assert_array_equal(np.sort(ok[sl]), np.sort(data["o"][0][got4 == n]))
    # single-process redistribute degenerates to the local partition
    gx.set_shardmap(1)
    r = gx.redistribute(data["ot"], g.O_CUSTKEY)
    np.testing.assert_array_equal(np.sort(r.read(0)), np.sort(data["o"][0]))


def test_sf100_full_size_properties(gx):
    """BASELINE config 3 at its full size (150 M orders, ~600 M lineitem rows, the tables bench.py
    runs on).  The oracle cannot follow here; size-independent properties must hold instead:
    every lineitem row finds exactly one order (count(*) sums to the row count), the groups are the
    2406 order dates, the per-group sums add up to the plain sum of the column (1e-9), and three
    independent paths agree group by group: the run-folding kernel on the compact table, the
    row-per-lane kernel on 16-byte slots with the mixing hash, and the radix strategy.
    The radix leg keeps three record buffers of ~0.72 GB per unit of scale factor beside the ~0.11 GB of
    columns: SF100 needs ~84 GB, so a GPU with less than 120 GB (an 80 GB H100) runs SF50."""
    import os
    free_b = gx.device_info()["hbm_bytes"]
    if free_b < 60e9:
        pytest.skip("needs a GPU with room for the SF50 columns and radix records")
    sf = 100 if free_b >= 120e9 else 50
    no = 1_500_000 * sf
    ot = gx.table([g.GX_INT8, g.GX_DATE], no); ot.generate(g.T_ORDERS, sf, 0, no, colmap=[g.O_ORDERKEY, g.O_ORDERDATE])
    lt = gx.table([g.GX_INT8, g.GX_FLOAT8], no * 4 + no // 8); lt.generate(g.T_LINEITEM, sf, 0, no, colmap=[g.L_ORDERKEY, g.L_EXTENDEDPRICE])
    nl = lt.nrows
    assert 3.99 * no < nl < 4.01 * no
    aggs = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])]
    total = gx.hash_agg(lt, g.make_plan(aggs=aggs)).fetch()[1]
    assert total[0, 0].view(np.int64) == nl
    results = {}
    for name, env, strategy in (("runjoin_compact", {}, 1),
                                ("row_per_lane_mixhash", {"GX_NO_RUNJOIN": "1", "GX_SLOT_MODE": "0"}, 1),
                                ("radix", {}, 2)):
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            ht = gx.hash_build(ot, 0, [1], unique=True)
            assert ht.nentries == no
            if name == "runjoin_compact":
                assert ht.info()["slot_mode"] == 2
            k, a, _ = gx.hash_agg(lt, g.make_plan(outer_key_col=0, group_cols=[(1, 0)], aggs=aggs, est_groups=2500, strategy=strategy), ht).fetch()
            ht.free()
        finally:
            for kk, v in old.items():
                if v is None:
                    os.environ.pop(kk, None)
                else:
                    os.environ[kk] = v
        assert len(k) == 2406
        assert a[:, 0].view(np.int64).sum() == nl
        np.testing.assert_allclose(a[:, 1].sum(), total[0, 1], rtol=1e-9)
        o = np.argsort(k[:, 0])
        results[name] = (k[o, 0], a[o, 0].view(np.int64).copy(), a[o, 1].copy())
    ref = results["runjoin_compact"]
    for name in ("row_per_lane_mixhash", "radix"):
        np.testing.assert_array_equal(results[name][0], ref[0])
        np.testing.assert_array_equal(results[name][1], ref[1], err_msg=f"{name}: counts differ from the run-folding kernel")
        np.testing.assert_allclose(results[name][2], ref[2], rtol=1e-9, atol=0)
    ot.free(); lt.free()


# ----------------------------------------------------- heap pages (K0)
def test_heap_page_deform_matches_oracle(gx):
    """Raw 8 KB OpenTenBase heap pages -> columns on the device, against the
    oracle's heapgetpage + slot_deform_tuple; with NULLs, short varlenas
    (bpchar(1)) in front of the wanted attributes, and deleted tuples."""
    rng = np.random.default_rng(5)
    n = 5000
    types = [O.GX_INT8, O.GX_INT4, O.GX_FLOAT8, O.ORC_BPCHAR1, O.ORC_BPCHAR1, O.GX_DATE, O.GX_CHAR, O.GX_FLOAT8]
    cols = [rng.integers(-2**62, 2**62, n), rng.integers(-2**31, 2**31, n).astype(np.int32), rng.normal(0, 1e6, n),
            rng.choice(np.frombuffer(b"RAN", np.int8), n), rng.choice(np.frombuffer(b"OF", np.int8), n),
            rng.integers(-3000, 0, n).astype(np.int32), rng.integers(32, 127, n).astype(np.int8), rng.random(n)]
    nulls = [None, (rng.random(n) < 0.1).astype(np.uint8), (rng.random(n) < 0.1).astype(np.uint8),
             (rng.random(n) < 0.2).astype(np.uint8), None, (rng.random(n) < 0.1).astype(np.uint8), None, None]
    rel = O.Rel(types, cols, nulls)
    for p, off in [(0, 1), (0, 7), (3, 2), (rel.npages - 1, 1)]:
        assert rel.delete(p, off) == 0
    attnums = [0, 2, 3, 5, 6, 7]
    want_cols, want_nulls = rel.scan(attnums)
    assert len(want_cols[0]) == n - 4
    gtypes = [g.GX_INT8, g.GX_FLOAT8, g.GX_CHAR, g.GX_DATE, g.GX_CHAR, g.GX_FLOAT8]
    att_len = [8, 4, 8, -1, -1, 4, 1, 8]; att_align = [8, 4, 8, 4, 4, 4, 1, 8]
    # (a) visibility lists as heapgetpage would hand them over
    pages = rel.pages()
    import ctypes as C
    vis = np.zeros((rel.npages, 300), np.uint16); cnt = np.zeros(rel.npages, np.int32)
    L = O.lib()
    L.orc_heapgetpage.restype = C.c_int
    L.orc_heapgetpage.argtypes = [C.c_void_p, C.c_void_p]
    for p in range(rel.npages):
        cnt[p] = L.orc_heapgetpage(pages[p * 8192:].ctypes.data, vis[p].ctypes.data)
    t = gx.table(gtypes, n)
    t.append_heap_pages(pages, att_len, att_align, attnums, vis, cnt)
    assert t.nrows == n - 4
    for c in range(len(attnums)):
        got, gn = t.read(c, with_nulls=True)
        np.testing.assert_array_equal(gn, want_nulls[c])
        keep = want_nulls[c] == 0
        if got.dtype == np.float64:
            np.testing.assert_array_equal(got.view(np.int64)[keep], want_cols[c].view(np.int64)[keep])
        else:
            np.testing.assert_array_equal(got[keep], want_cols[c][keep])
    # (b) no visibility list: every LP_NORMAL item (deleted tuples come back too)
    t2 = gx.table(gtypes, n)
    t2.append_heap_pages(pages, att_len, att_align, attnums)
    assert t2.nrows == n


def test_heap_page_deform_throughput(gx, capsys):
    """K0 at a size where the kernel time is visible: ~25 k pages (200 MB) of lineitem-shaped
    tuples.  Checks the columns again and reports GB/s of page bytes (kernel only and from host
    pages); the floor is deliberately loose — the number itself goes to DESIGN.md."""
    n_orders = 300_000
    cols = list(O.gen_lineitem(1, 0, n_orders))
    use = [g.L_ORDERKEY, g.L_QUANTITY, g.L_EXTENDEDPRICE, g.L_DISCOUNT, g.L_TAX, g.L_RETURNFLAG, g.L_LINESTATUS, g.L_SHIPDATE]
    cols = [cols[c] for c in use]
    types = [g.SCHEMAS[g.T_LINEITEM][c] for c in use]
    rel = O.Rel(types, cols)
    pages = rel.pages()
    n = len(cols[0])
    att_len = [8, 8, 8, 8, 8, 1, 1, 4]; att_align = [8, 8, 8, 8, 8, 1, 1, 4]
    t = gx.table(types, n); t.append_heap_pages(pages, att_len, att_align, list(range(8)))
    assert t.nrows == n
    np.testing.assert_array_equal(t.read(0), cols[0])
    np.testing.assert_array_equal(t.read(7), cols[7])
    np.testing.assert_array_equal(t.read(2).view(np.int64), cols[2].view(np.int64))
    t.free()
    iters = 5
    gx.profile(True)
    gx.sync(); gx.timer_start()
    for _ in range(iters):
        t = gx.table(types, n); t.append_heap_pages(pages, att_len, att_align, list(range(8))); t.free()
    ms = gx.timer_stop() / iters
    kms, kn = gx.profile_get("deform")
    gx.profile(False)
    page_gb = rel.npages * 8192 / 1e9
    with capsys.disabled():
        print(f"\nK0: {rel.npages} pages, {n} tuples: {ms:.2f} ms from host pages ({page_gb / ms * 1e3:.1f} GB/s of pages); "
              f"deform kernels {kms / iters:.3f} ms per call ({page_gb / (kms / iters) * 1e3:.0f} GB/s of pages, {kn // iters} launches)")
    assert page_gb / (kms / iters) * 1e3 > 200.0           # the kernels stream pages well above PCIe speed


# ----------------------------------------------------- host-buffer entry
def test_exec_host_matches_resident_path(gx, data):
    plan = O.make_plan(outer_key_col=g.L_ORDERKEY, group_cols=[(1, 0)],
                       aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0)])], est_groups=2500)
    join = O.make_join(g.O_ORDERKEY, payload_cols=[g.O_ORDERDATE], inner_unique=1)
    want = O.exec_agg(data["lrel"], plan, data["orel"], join)
    lc = [np.ascontiguousarray(c) for c in data["l"]]; oc = [np.ascontiguousarray(c) for c in data["o"]]
    res = gx.exec_host(g.SCHEMAS[g.T_LINEITEM], lc, len(lc[0]), to_gpu_plan(plan), g.SCHEMAS[g.T_ORDERS], oc, len(oc[0]),
                       inner_key_col=g.O_ORDERKEY, payload_cols=[g.O_ORDERDATE], inner_unique=True)
    assert_agg_equal(plan, res.fetch(), want)


# --------------------------------------- full-size, size-independent checks
def test_sf10_properties(gx):
    """At BASELINE config-2/3 shapes the oracle is too slow; check invariants:
    counts sum to the row count, every lineitem finds its order, per-group sums
    add up to the plain sum, and the radix and shared-memory strategies agree."""
    sf = 10
    no = 1_500_000 * sf // 10                     # a tenth of SF10's orders keeps the test short
    ot = gx.table([g.GX_INT8, g.GX_DATE], no); ot.generate(g.T_ORDERS, sf, 0, no, colmap=[g.O_ORDERKEY, g.O_ORDERDATE])
    lt = gx.table([g.GX_INT8, g.GX_FLOAT8, g.GX_DATE], no * 7); lt.generate(g.T_LINEITEM, sf, 0, no, colmap=[g.L_ORDERKEY, g.L_EXTENDEDPRICE, g.L_SHIPDATE])
    nl = lt.nrows
    assert 3.9 * no < nl < 4.1 * no
    ht = gx.hash_build(ot, 0, [1], unique=True)
    assert ht.nentries == no
    aggs = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])]
    total = gx.hash_agg(lt, g.make_plan(aggs=aggs)).fetch()[1]
    assert total[0, 0].view(np.int64) == nl
    byjoin = {}
    for strategy in (1, 2):
        k, a, _ = gx.hash_agg(lt, g.make_plan(outer_key_col=0, group_cols=[(1, 0)], aggs=aggs, est_groups=2500, strategy=strategy), ht).fetch()
        assert a[:, 0].view(np.int64).sum() == nl
        assert len(k) == 2406
        np.testing.assert_allclose(a[:, 1].sum(), total[0, 1], rtol=1e-9)
        byjoin[strategy] = (k, a)
    o1, o2 = np.argsort(byjoin[1][0][:, 0]), np.argsort(byjoin[2][0][:, 0])
    np.testing.assert_array_equal(byjoin[1][1][o1, 0].view(np.int64), byjoin[2][1][o2, 0].view(np.int64))
    np.testing.assert_allclose(byjoin[1][1][o1, 1], byjoin[2][1][o2, 1], rtol=1e-9)
    k, a, _ = gx.hash_agg(lt, g.make_plan(group_cols=[(0, 2)], aggs=aggs, est_groups=2600)).fetch()
    assert a[:, 0].view(np.int64).sum() == nl
    np.testing.assert_allclose(a[:, 1].sum(), total[0, 1], rtol=1e-9)
