"""tests/star_ref.py, the exact reference of an aggregate over a chain of INNER hash joins, pinned to the oracle without a
GPU: the oracle joins the fact table to the first dimension (orc_exec_join, the reference's ExecHashJoinImpl) and then
aggregates that join's output over a hash join with the second dimension (orc_exec_agg), quals on every side."""
import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import join_ref as J
import star_ref as S

I64 = np.iinfo(np.int64)


def _data(rng, n_outer, n_d1, n_d2):
    """fact [key int8 (NULLs, INT64_MIN, misses), value float8, group int4]; d1 [key int8 unique, d2 key int4, date];
    d2 [key int4 unique, segment int4]"""
    d1k = rng.permutation(np.concatenate([rng.choice(np.arange(-3000, 3000), n_d1 - 1, replace=False), [I64.min]])).astype(np.int64)
    d2k = rng.choice(np.arange(-400, 400), n_d2, replace=False).astype(np.int32)
    d1c = rng.integers(-450, 450, n_d1).astype(np.int32)                 # some find no d2 row
    d1d = rng.integers(-100, 100, n_d1).astype(np.int32)
    d2s = rng.integers(0, 5, n_d2).astype(np.int32)
    ok = np.concatenate([rng.choice(d1k, n_outer - 40), rng.integers(-4000, 4000, 36), [I64.min, I64.max, 2**32, -2**31]])
    ok = rng.permutation(ok).astype(np.int64)
    onull = (rng.random(n_outer) < 0.06).astype(np.uint8)
    ox = rng.standard_normal(n_outer) * 10.0 ** rng.integers(-3, 4, n_outer)
    og = rng.integers(0, 6, n_outer).astype(np.int32)
    return [ok, ox, og], [onull, None, None], [d1k, d1c, d1d], [d2k, d2s]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_star_ref_matches_the_oracle_join_then_aggregate(seed):
    rng = np.random.default_rng(seed)
    ocols, onulls, d1, d2 = _data(rng, 1500, 600, 300)
    otypes, d1types, d2types = [g.GX_INT8, g.GX_FLOAT8, g.GX_INT4], [g.GX_INT8, g.GX_INT4, g.GX_DATE], [g.GX_INT4, g.GX_INT4]
    opreds, d1preds, d2preds = [(1, g.GX_LT, 3.0, True)], [(2, g.GX_GE, -60)], [(1, g.GX_NE, 3)]
    aggs = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 2, 0)]), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)]),
            (g.GX_AGG_MAX_F8, [(g.GX_OP_COL, 1, 0)])]

    # oracle: fact JOIN d1 (payload d2 key, date), then aggregate over that JOIN d2 (payload segment)
    j1 = O.exec_join(O.Rel(otypes, ocols, onulls), 0, O.Rel(d1types, d1),
                     O.make_join(0, payload_cols=[1, 2], inner_unique=1, inner_preds=d1preds), [0, 1, 2], outer_preds=opreds)
    jcols = [j1[0], j1[1].view(np.float64), j1[2].astype(np.int32), j1[3].astype(np.int32), j1[4].astype(np.int32)]
    jtypes = [g.GX_INT8, g.GX_FLOAT8, g.GX_INT4, g.GX_INT4, g.GX_DATE]
    oplan = O.make_plan(outer_key_col=3, group_cols=[(0, 2), (0, 4), (1, 0)], aggs=aggs, est_groups=64)
    r = O.exec_agg(O.Rel(jtypes, jcols), oplan, O.Rel(d2types, d2), O.make_join(0, payload_cols=[1], inner_unique=1, inner_preds=d2preds))

    plan = g.make_plan(preds=opreds, group_cols=[(0, 2), (1, 1), (2, 0)], aggs=aggs, est_groups=64)
    steps = [S.Step((0, 0), d1[0], [d1[1], d1[2]], [g.GX_INT4, g.GX_DATE], bkeep=J.quals(d1, None, d1preds, len(d1[0]))),
             S.Step((1, 0), d2[0], [d2[1]], [g.GX_INT4], bkeep=J.quals(d2, None, d2preds, len(d2[0])))]
    want = S.expect_chain_groups(plan, ocols, otypes, steps, outer_nulls=onulls)
    X.check(plan, want, (r.keys, r.aggs, r.nulls), [g.GX_INT4, g.GX_DATE, g.GX_INT4])
    assert sum(e[0].value for e in want.values()) > 100


def test_a_row_reaches_the_aggregate_only_through_every_step():
    """hand-sized: a miss at either step drops the row, a NULL key drops it, a step-2 key comes from step 1's payload"""
    ok = np.array([1, 2, 3, 4, 1, 0], np.int64)
    onull = np.array([0, 0, 0, 0, 0, 1], np.uint8)
    og = np.array([10, 20, 30, 40, 10, 50], np.int32)
    d1k, d1c = np.array([1, 2, 4, 0], np.int64), np.array([7, 8, 9, 7], np.int32)       # key 3 misses step 1
    d2k, d2s = np.array([7, 9], np.int32), np.array([100, 300], np.int32)               # d2 key 8 misses step 2
    p = g.make_plan(group_cols=[(0, 1), (2, 0)], aggs=[(g.GX_AGG_COUNT_STAR, [])])
    steps = [S.Step((0, 0), d1k, [d1c], [g.GX_INT4]), S.Step((1, 0), d2k, [d2s], [g.GX_INT4])]
    want = S.expect_chain_groups(p, [ok, og], [g.GX_INT8, g.GX_INT4], steps, outer_nulls=[onull, None])
    assert {k: v[0].value for k, v in want.items()} == {(10, 100): 2, (40, 300): 1}


# ---------------------------------------------------------------- the provider: planner, descriptor, shipping, host logic
import os                                                                  # noqa: E402
import struct                                                              # noqa: E402
import subprocess                                                          # noqa: E402
import tempfile                                                            # noqa: E402

from test_provider_harness import HARNESS, write_case                      # noqa: E402
from test_provider_planner_cpu import LINEITEM, ORDERS, parse_desc, plan   # noqa: E402

needs_harness = pytest.mark.skipif(not os.path.exists(HARNESS), reason="harness binary not built (needs /root/reference at build time)")
CUSTOMER = "rel 3 tuples 150000 pages 1100 cols int4! bpchar1! int4! int4"       # custkey, mktsegment, nationkey, a nullable int4
NATION = "rel 4 tuples 25 pages 1 cols int4! int4!"                              # nationkey, regionkey
REGION = "rel 5 tuples 5 pages 1 cols int4! int4!"                               # regionkey, a code
SEG = ["qual 2 3 date_lt date -1752", "qual 1 6 date_gt date -1752", "group 3.2", "target var 3.2", "target agg count_star",
       "target agg sum_f8 v1.3 k1 v1.4 - *", "dist none", "groups 5"]
CHAIN_WORD = 100


def parse_chain_desc(d):
    """the wire layout of gpuexec_serialise for a join chain: the single join's layout with steps 2.. after its block"""
    it = iter(d)
    nx = lambda: next(it)
    out = {"abi": nx(), "word": nx()}

    def rel():
        rti, n = nx(), nx()
        return {"rti": rti, "cols": [(nx(), nx()) for _ in range(n)]}
    out["outer"] = rel()
    out["inner"] = rel()
    out["inner_key_col"] = nx()
    out["payload"] = [nx() for _ in range(nx())]
    out["inner_unique"] = nx()
    out["inner_preds"] = [(nx(), nx(), nx(), nx()) for _ in range(nx())]
    out["more"] = []
    for _ in range(nx()):
        m = {"rel": rel(), "key_col": nx(), "probe": (nx(), nx())}
        m["payload"] = [nx() for _ in range(nx())]
        m["preds"] = [(nx(), nx(), nx(), nx()) for _ in range(nx())]
        out["more"].append(m)
    out["partial"] = nx()
    npred = nx()
    out["outer_key_col"] = nx()
    out["preds"] = [(nx(), nx(), nx(), nx()) for _ in range(npred)]
    out["group_cols"] = [(nx(), nx()) for _ in range(nx())]
    out["aggs"] = [(lambda fn, n: (fn, [(nx(), nx(), nx()) for _ in range(n)]))(nx(), nx()) for _ in range(nx())]
    out["est_groups"] = nx()
    assert next(it, None) is None
    return out


@needs_harness
def test_planner_takes_a_two_step_chain():
    """lineitem -> orders[o_orderdate < D] (o_custkey carried) -> customer, GROUP BY c_mktsegment"""
    r = plan(LINEITEM, ORDERS, CUSTOMER, "join 1.1 2.1 unique 1", "join 2.2 3.1 unique 1", *SEG)
    assert r is not None and r["path"] == "path pushdown: CustomScan"
    d = parse_chain_desc(r["desc"])
    assert d["word"] == CHAIN_WORD and d["inner_unique"] == 1 and len(d["more"]) == 1
    ocols, icols = [c for c, _ in d["outer"]["cols"]], [c for c, _ in d["inner"]["cols"]]
    assert ocols[d["outer_key_col"]] == 0 and icols[d["inner_key_col"]] == 0
    assert [icols[c] for c in d["payload"]] == [1]                                  # o_custkey: step 2's key
    assert d["inner_preds"] == [(icols.index(2), g.GX_LT, -1752, 0)]
    m = d["more"][0]
    mcols = [c for c, _ in m["rel"]["cols"]]
    assert m["rel"]["rti"] == 3 and mcols[m["key_col"]] == 0 and m["probe"] == (1, 0)
    assert [mcols[c] for c in m["payload"]] == [1] and d["group_cols"] == [(2, 0)]   # c_mktsegment: step 2's payload
    assert d["preds"] == [(ocols.index(5), g.GX_GT, -1752, 0)]


@needs_harness
def test_planner_takes_a_three_step_chain_and_shares_payload_slots():
    """... -> customer (c_nationkey) -> nation; GROUP BY c_nationkey shares the slot step 3's key uses, n_regionkey from step 3"""
    r = plan(LINEITEM, ORDERS, CUSTOMER, NATION, "join 1.1 2.1 unique 1", "join 2.2 3.1 unique 1", "join 3.3 4.1 unique 1",
             "group 3.3", "group 4.2", "target var 3.3", "target var 4.2", "target agg count_star", "dist none", "groups 25")
    assert r is not None
    d = parse_chain_desc(r["desc"])
    assert d["word"] == CHAIN_WORD and len(d["more"]) == 2
    m2, m3 = d["more"]
    assert m2["probe"] == (1, 0) and m3["probe"] == (2, 0) and len(m2["payload"]) == 1
    assert d["group_cols"] == [(2, 0), (3, 0)]


@needs_harness
def test_single_join_descriptor_is_unchanged():
    r = plan(LINEITEM, ORDERS, "join 1.1 2.1 unique 1", "group 2.3", "target var 2.3", "target agg count_star", "dist none", "groups 2526")
    d = parse_desc(r["desc"])
    assert r["desc"][1] == 1 and d["has_join"] == 1 and d["payload"] == [1] and d["group_cols"] == [(1, 0)]


DECLINES = {
    "non-unique step 2": (["join 1.1 2.1 unique 1", "join 2.2 3.1 unique 0"], SEG),
    "non-unique step 1": (["join 1.1 2.1 unique 0", "join 2.2 3.1 unique 1"], SEG),
    "left step 1": (["join 1.1 2.1 unique 1 left", "join 2.2 3.1 unique 1"], SEG),
    "left step 2": (["join 1.1 2.1 unique 1", "join 2.2 3.1 unique 1 left"], SEG),
    "semi step 2": (["join 1.1 2.1 unique 1", "join 2.2 3.1 unique 1 semi"], SEG),
    "anti step 1": (["join 1.1 2.1 unique 1 anti", "join 2.2 3.1 unique 1"], SEG),
    "remote scan step 1": (["join 1.1 2.1 unique 1 remote_inner", "join 2.2 3.1 unique 1"], SEG),
    "remote scan step 2": (["join 1.1 2.1 unique 1", "join 2.2 3.1 unique 1 remote_inner"], SEG),
    "nullable key column": (["join 1.1 2.1 unique 1", "join 3.4 4.1 unique 1"], ["group 4.2", "target var 4.2", "target agg count_star", "dist none"]),
    "aggregate over a dimension column": (["join 1.1 2.1 unique 1", "join 2.2 3.1 unique 1"],
                                          ["group 3.2", "target var 3.2", "target agg sum_f8 v2.5", "dist none"]),
    "payload overflow": (["join 1.1 2.1 unique 1", "join 2.2 3.1 unique 1"],
                         ["group 2.3", "group 2.4", "group 3.2", "target var 3.2", "target agg count_star", "dist none"]),
    "four levels": (["join 1.1 2.1 unique 1", "join 2.2 3.1 unique 1", "join 3.3 4.1 unique 1", "join 4.2 5.1 unique 1"],
                    ["group 5.2", "target var 5.2", "target agg count_star", "dist none"]),
}


@needs_harness
@pytest.mark.parametrize("what", list(DECLINES))
def test_planner_declines(what):
    joins, tail = DECLINES[what]
    assert plan(LINEITEM, ORDERS, CUSTOMER, NATION, REGION, *joins, *tail) is None


@needs_harness
def test_the_decline_cases_are_accepted_once_the_one_fault_is_removed():
    """the DECLINES scenarios are one change away from an accepted plan: the harness really builds what they describe"""
    assert plan(LINEITEM, ORDERS, CUSTOMER, NATION, "join 1.1 2.1 unique 1", "join 3.3 4.1 unique 1",
                "group 4.2", "target var 4.2", "target agg count_star", "dist none") is None      # 3.3 is not in the chain
    assert plan(LINEITEM, ORDERS, CUSTOMER, NATION, "join 1.1 2.1 unique 1", "join 2.2 3.1 unique 1", "join 3.3 4.1 unique 1",
                "group 4.2", "target var 4.2", "target agg count_star", "dist none") is not None


# ---- the executor side: case files of a chain (gpuexec_harness / gpuexec_harness_double)
def write_chain_case(path, rels, outer, steps, plan_, partial, out_types):
    """write_case's format with the join count in the has_join word and steps 2.. after the first join's block;
    steps: dict(rti, attnums, key_col, payload_cols, preds[, probe=(side, col)]) in chain order"""
    write_case(path, rels, outer, dict(steps[0], unique=True), plan_, partial, out_types)
    with open(path, "rb") as f:
        blob = f.read()
    head = 4 + 4
    for types, rel in rels:
        head += 4 + 16 * len(types) + 8 + 4 + rel.npages * 8192
    more = bytearray()
    for st in steps[1:]:
        types = rels[st["rti"] - 1][0]
        more += struct.pack("<ii", st["rti"], len(st["attnums"]))
        for a in st["attnums"]:
            more += struct.pack("<ii", a, {O.GX_INT8: g.GX_INT8, O.GX_INT4: g.GX_INT4, O.GX_DATE: g.GX_DATE, O.GX_FLOAT8: g.GX_FLOAT8}.get(types[a], g.GX_CHAR))
        more += struct.pack("<iiii", st["key_col"], st["probe"][0], st["probe"][1], len(st["payload_cols"]))
        for c in st["payload_cols"]:
            more += struct.pack("<i", c)
        more += struct.pack("<i", len(st.get("preds", [])))
        for pr in st.get("preds", []):
            more += bytes(g.mk_pred(*pr))
    # the tail: partial, the plan, the output types
    tail = 4 + len(bytes(plan_)) + 4 + 4 * len(out_types)
    body = blob[head + 4:len(blob) - tail]
    with open(path, "wb") as f:
        f.write(blob[:head] + struct.pack("<i", len(steps)) + body + bytes(more) + blob[len(blob) - tail:])


CASE_ORDER_BEFORE, CASE_SHIP_AFTER = -1000, -2000          # o_orderdate < 1997-04-06, l_shipdate > 1994-07-11


def chain_case(d):
    """lineitem (l_orderkey, l_extendedprice, l_shipdate) -> orders (o_orderkey; o_custkey carried) -> customer
    (c_custkey; c_mktsegment carried), GROUP BY c_mktsegment: count(*), sum(l_extendedprice)"""
    o, l, c = O.gen_orders(1, 0, 2000), O.gen_lineitem(1, 0, 2000), O.gen_customer(1, 0, 150_000)
    otypes, ctypes = [O.GX_INT8, O.GX_INT4, O.GX_DATE, O.GX_INT4], [O.GX_INT4, O.GX_INT4]
    ltypes = [O.GX_INT8, O.GX_FLOAT8, O.GX_FLOAT8, O.GX_FLOAT8, O.GX_FLOAT8, O.GX_DATE, O.GX_INT4, O.GX_INT4]
    lc = [l[0], l[1], l[2], l[3], l[4], l[5], l[6].astype(np.int32), l[7].astype(np.int32)]
    cc = [c[0], c[1].astype(np.int32)]
    rels = [(ltypes, O.Rel(ltypes, lc)), (otypes, O.Rel(otypes, o)), (ctypes, O.Rel(ctypes, cc))]
    p = g.make_plan(preds=[(2, g.GX_GT, CASE_SHIP_AFTER)], outer_key_col=0, group_cols=[(2, 0)],
                    aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])], est_groups=5)
    steps = [{"rti": 2, "attnums": [0, 1, 2], "key_col": 0, "payload_cols": [1], "preds": [(2, g.GX_LT, CASE_ORDER_BEFORE)]},
             {"rti": 3, "attnums": [0, 1], "key_col": 0, "payload_cols": [1], "preds": [], "probe": (1, 0)}]
    case = os.path.join(d, "chain.case")
    write_chain_case(case, rels, {"rti": 1, "attnums": [0, 2, 5]}, steps, p, False, [23, 20, 701])
    return case, (lc, o, cc)


@needs_harness
def test_chain_descriptor_survives_plan_shipping():
    from test_provider_ship_cpu import ship
    with tempfile.TemporaryDirectory() as d:
        case, _ = chain_case(d)
        toks = ship(case).strip("()").split(" ")
    assert toks[1] == str(CHAIN_WORD)
    dd = parse_chain_desc([int(t) for t in toks])
    assert dd["more"][0]["probe"] == (1, 0) and dd["group_cols"] == [(2, 0)] and dd["outer_key_col"] == 0


DOUBLE = HARNESS + "_double"


def _canned(path):
    with open(path, "wb") as f:
        f.write(struct.pack("<qii", 1, 1, 2))
        f.write(np.array([3], np.int64).tobytes()); f.write(np.array([np.int64(7).view(np.float64), 1.5]).tobytes())     # count(*) bit-cast
        f.write(np.array([7, 7], np.int64).tobytes()); f.write(np.zeros(3, np.uint8).tobytes())


@pytest.mark.skipif(not os.path.exists(DOUBLE), reason="harness binary not built (needs /root/reference at build time)")
@pytest.mark.parametrize("fail", [False, True])
def test_chain_host_logic_load_and_build_order_and_every_handle_freed(fail):
    """Begin/Exec/End against the ABI double: every inner relation loads (chain order) before the outer one, the tables
    are built in chain order, gx_hash_agg_joins gets the steps' keys; on an ERROR every table and handle is freed"""
    with tempfile.TemporaryDirectory() as d:
        case, _ = chain_case(d)
        res = os.path.join(d, "r.res")
        _canned(res)
        env = dict(os.environ, GX_DOUBLE_RESULT=res, **({"GX_DOUBLE_FAIL_AGG": "1"} if fail else {}))
        r = subprocess.run([DOUBLE, case], capture_output=True, text=True, timeout=120, env=env)
    err = r.stderr.splitlines()
    creates = [l for l in err if l.startswith("double: table_create")]
    assert [l.split()[3] for l in creates] == ["3", "2", "3"]                 # orders (3 cols), customer (2), lineitem (3)
    builds = [l for l in err if l.startswith("double: hash_build")]
    assert len(builds) == 2 and all("unique 1" in b for b in builds)
    assert f"payload 1 preds (2 1 {CASE_ORDER_BEFORE})" in builds[0] and "payload 1 preds" in builds[1]
    assert any(l.startswith("double: hash_agg_joins steps 2 (key 0.0 table key 0) (key 1.0 table key 0)") for l in err), err
    if fail:
        assert r.returncode == 3 and "ereport(ERROR)" in r.stderr
    else:
        assert r.returncode == 0, r.stderr[-2000:]
        assert r.stdout.split() == ["3", "7", "1.5"]
    assert "double: shutdown live tables 0 hashes 0 results 0" in err
