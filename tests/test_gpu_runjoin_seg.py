"""The two cp.async.bulk + mbarrier variants of the config-3 probe against the oracle's HashJoin + HashAggregate
(nodeHashjoin.c:186-742, nodeAgg.c:2609-2648):

* gx_k_runjoin_seg (GX_RUNJOIN_SEG=1) streams the JOIN TABLE through a shared-memory ring instead of gathering it,
* gx_k_runjoin_tma (GX_RUNJOIN_TMA=1) has the copy engine deliver the OUTER ROWS of every warp's next tile,

on the layouts that decide which of their code paths run:

* both sides in key order              every probe answered from the staged window
* outer side shuffled                  chunk key ranges far wider than the ring: nothing staged, global probes
* outer side descending                first key > last key of every chunk: empty windows
* build side with holes / narrow span  misses, keys below and above the build side's key span (clamped windows)
* tiny outer sides                     fewer rows than one chunk, a tail that is not a multiple of four

and with every ring depth.  The switches force a variant on or off; the profile names `probe_agg_seg` /
`probe_agg_tma` prove which kernel ran."""
import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
from helpers import assert_agg_equal, to_gpu_plan, lineitem_rel, orders_rel

pytestmark = pytest.mark.gpu

NORD = 200_000        # >= 64 sub-tables: interpolation slots + compact table, what the seg variant needs
VARIANTS = {"seg": ("GX_RUNJOIN_SEG", "1", "probe_agg_seg"), "tma": ("GX_RUNJOIN_TMA", "1", "probe_agg_tma"),
            "tma2": ("GX_RUNJOIN_TMA", "2", "probe_agg_tma"),          # tma2: gx_k_runjoin_tma with the branch-free fold
            "tma3": ("GX_RUNJOIN_TMA", "3", "probe_agg_tma")}          # tma3: + probe rounds of 32 lanes only (runs wait in the list)


@pytest.fixture(params=list(VARIANTS))
def variant(request, monkeypatch):
    for env, _, _ in VARIANTS.values():
        monkeypatch.setenv(env, "0")
    monkeypatch.setenv(VARIANTS[request.param][0], VARIANTS[request.param][1])
    monkeypatch.setenv("GX_DEBUG_AGG", "1")
    return VARIANTS[request.param][2]


def _plan(count=True, total=True):
    aggs = []
    if count:
        aggs.append((g.GX_AGG_COUNT_STAR, []))
    if total:
        aggs.append((g.GX_AGG_SUM_F8, [(g.GX_OP_COL, g.L_EXTENDEDPRICE, 0)]))
    return O.make_plan(outer_key_col=g.L_ORDERKEY, group_cols=[(1, 0)], aggs=aggs, est_groups=2600)


def _run(gx, o, l, plan, expect_seg=True, prof="probe_agg_seg"):
    join = O.make_join(g.O_ORDERKEY, payload_cols=[g.O_ORDERDATE], inner_unique=1)
    want = O.exec_agg(lineitem_rel(l), plan, orders_rel(o), join)
    ot = gx.table_from(g.SCHEMAS[g.T_ORDERS], o)
    lt = gx.table_from(g.SCHEMAS[g.T_LINEITEM], l)
    ht = gx.hash_build(ot, g.O_ORDERKEY, [g.O_ORDERDATE], unique=True)
    if expect_seg:
        assert ht.info()["slot_mode"] == 2, ht.info()        # key-ordered build: compact slots, order-preserving
    gx.profile(True)
    try:
        got = gx.hash_agg(lt, to_gpu_plan(plan), ht).fetch()
        _, nseg = gx.profile_get(prof)
    finally:
        gx.profile(False)
    if expect_seg is not None:
        assert (nseg > 0) == expect_seg, f"{prof} launches: {nseg}"
    assert_agg_equal(plan, got, want)
    for t in (ht, lt, ot):
        t.free()
    return got


@pytest.fixture(scope="module")
def base():
    o = [c.copy() for c in O.gen_orders(1, 0, NORD)]
    l = [c.copy() for c in O.gen_lineitem(1, 0, NORD)]
    return o, l


@pytest.mark.parametrize("bufs", ["2", "3", "4"])
def test_key_ordered_both_sides(gx, base, monkeypatch, variant, bufs):
    """Every ring depth of the seg variant; the copy-engine variants have no ring and must give the same
    answer whatever depth is set for it."""
    monkeypatch.setenv("GX_RUNJOIN_SEG_BUFS", bufs)
    o, l = base
    got = _run(gx, o, l, _plan(), prof=variant)
    assert got[1][:, 0].view(np.int64).sum() == len(l[0])     # every line finds its order


@pytest.mark.parametrize("aggs", ["count", "sum"])
def test_single_aggregate_instantiations(gx, base, variant, aggs):
    o, l = base
    _run(gx, o, l, _plan(count=aggs == "count", total=aggs == "sum"), prof=variant)


@pytest.mark.parametrize("layout", ["shuffled", "descending", "block_shuffled"])
def test_outer_side_not_in_key_order(gx, base, variant, layout):
    """The windows are a guess from the first and last key of a chunk; the answer may not depend on it."""
    o, l = base
    n = len(l[0])
    if layout == "shuffled":
        perm = np.random.default_rng(3).permutation(n)
    elif layout == "descending":
        perm = np.arange(n)[::-1].copy()
    else:                                   # key order inside blocks of 1000 rows, the blocks in random order:
        nb = (n + 999) // 1000              # chunks straddle unrelated key ranges, some windows hold part of the keys
        order = np.random.default_rng(4).permutation(nb)
        perm = np.concatenate([np.arange(b * 1000, min((b + 1) * 1000, n)) for b in order])
    _run(gx, o, [c[perm] for c in l], _plan(), prof=variant)


def test_misses_and_keys_outside_the_build_span(gx, base, variant):
    """Build side = the middle half of the orders with every third order removed: lines of the first and
    last quarter carry keys below / above the build side's span (windows clamped to the span or empty),
    lines of removed orders miss inside it."""
    o, l = base
    keep = np.zeros(NORD, bool)
    keep[NORD // 4: 3 * NORD // 4] = True
    keep[::3] = False
    got = _run(gx, [c[keep] for c in o], l, _plan(), expect_seg=None, prof=variant)     # a 67 k-row build side is at the edge of the interpolation rule
    assert 0 < got[1][:, 0].view(np.int64).sum() < len(l[0])


@pytest.mark.parametrize("nrows", [1, 3, 4, 127, 130, 3967, 3968, 3971, 4 * 3968 + 5])
def test_short_outer_sides(gx, base, variant, nrows):
    """Fewer rows than one chunk (31 tiles of 128 rows), one chunk exactly, tails of 1-3 rows."""
    o, l = base
    start = 123_457                          # somewhere inside the table, mid-run
    _run(gx, o, [c[start:start + nrows] for c in l], _plan(), prof=variant)


def test_switch_off_keeps_the_gathering_kernel(gx, base, monkeypatch):
    monkeypatch.setenv("GX_RUNJOIN_SEG", "0")
    monkeypatch.setenv("GX_RUNJOIN_TMA", "0")
    o, l = base
    _run(gx, o, l, _plan(), expect_seg=False)
    _run(gx, o, l, _plan(), expect_seg=False, prof="probe_agg_tma")


def test_default_is_the_copy_engine_kernel(gx, base, monkeypatch):
    """No switch set: gx_k_runjoin_tma (GX_RUNJOIN_TMA_DEFAULT in csrc/gx_agg.cu) answers config 3."""
    monkeypatch.delenv("GX_RUNJOIN_TMA", raising=False)
    monkeypatch.delenv("GX_RUNJOIN_SEG", raising=False)
    o, l = base
    _run(gx, o, l, _plan(), expect_seg=True, prof="probe_agg_tma")


def test_same_answer_as_the_gathering_kernel_at_sf10_slice(gx, monkeypatch):
    """10 M orders generated on the device (no oracle at this size): all variants must agree bit for bit
    on the counts and to 1e-9 on the sums, and count(*) must equal the lineitem rows."""
    nord = 10_000_000
    ot = gx.table(g.SCHEMAS[g.T_ORDERS], nord).generate(g.T_ORDERS, 10, 0, nord)
    lt = gx.table(g.SCHEMAS[g.T_LINEITEM], nord * 7).generate(g.T_LINEITEM, 10, 0, nord)
    ht = gx.hash_build(ot, g.O_ORDERKEY, [g.O_ORDERDATE], unique=True)
    plan = to_gpu_plan(_plan())
    res = {}
    for sw, (seg, tma) in {"0": ("0", "0"), "seg": ("1", "0"), "tma": ("0", "1"), "tma2": ("0", "2"), "tma3": ("0", "3")}.items():
        monkeypatch.setenv("GX_RUNJOIN_SEG", seg)
        monkeypatch.setenv("GX_RUNJOIN_TMA", tma)
        k, a, _ = gx.hash_agg(lt, plan, ht).fetch()
        order = np.argsort(k[:, 0])
        res[sw] = (k[order], a[order])
    for sw in ("seg", "tma", "tma2", "tma3"):
        np.testing.assert_array_equal(res["0"][0], res[sw][0])
        np.testing.assert_array_equal(res["0"][1][:, 0].view(np.int64), res[sw][1][:, 0].view(np.int64))
        np.testing.assert_allclose(res["0"][1][:, 1], res[sw][1][:, 1], rtol=1e-9, atol=0)
        assert res[sw][1][:, 0].view(np.int64).sum() == lt.nrows
    for t in (ht, lt, ot):
        t.free()


@pytest.mark.parametrize("layout", ["all", "blocks"])
def test_one_row_per_key(gx, base, variant, layout):
    """Every probe row its own run (128 runs per tile): the run list is full after every tile.  In blocks of 300 orders
    alternating with ordinary ones, tiles of 128 runs follow tiles that left runs waiting at the front of the list, and the
    variant that keeps them there has to make room first."""
    o, l = base
    first = np.concatenate([[True], l[g.L_ORDERKEY][1:] != l[g.L_ORDERKEY][:-1]])
    if layout == "blocks":
        order_no = np.cumsum(first) - 1
        first = first | ((order_no // 300) % 2 == 0)
    _run(gx, o, [c[first] for c in l], _plan(), prof=variant)
