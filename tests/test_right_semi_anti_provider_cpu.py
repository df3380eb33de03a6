"""The provider's right semi / right anti joins (JOIN_SEMI_RIGHT / JOIN_ANTI_RIGHT), without a GPU: what the planner
takes and declines, the descriptor it ships (the hashed relation in the outer slot, the probing one in the join step,
word 1 + GX_JOIN_* after the version) through the reference's own nodes/read.c, the cost term, and the executor's host
calls against the ABI double (a build with no payload, then gx_hash_agg_right)."""
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
from test_provider_harness import HARNESS, write_case
from test_provider_planner_cpu import LINEITEM, ORDERS, parse_desc, plan

needs_harness = pytest.mark.skipif(not os.path.exists(HARNESS), reason="harness binary not built (needs /root/reference at build time)")
DOUBLE = HARNESS + "_double"
WORDS = {"semi_right": g.GX_JOIN_SEMI_RIGHT, "anti_right": g.GX_JOIN_ANTI_RIGHT}
DATE_Q3 = -1752
# lineitem (rel 1) probes orders (rel 2): GROUP BY o_orderdate count(*), l_shipdate > 1995-03-15
Q4 = ["qual 1 6 date_gt date -1752", "group 2.3", "target var 2.3", "target agg count_star", "dist none", "groups 2406"]


def right(word, *tail, unique=1, lineitem=LINEITEM):
    return plan(lineitem, ORDERS, f"join 1.1 2.1 unique {unique} {word}", *tail)


@needs_harness
@pytest.mark.parametrize("word", list(WORDS))
def test_planner_takes_the_right_forms_and_swaps_the_sides(word):
    """the hashed relation (orders) takes the outer slot with its key and GROUP BY column, the probing one (lineitem)
    the join step with its key and its qual"""
    r = right(word, *Q4)
    assert r is not None and r["path"].startswith("path pushdown")
    d = r["desc"]
    assert d[1] == 1 + WORDS[word]                     # 9 / 10
    d = parse_desc([d[0], 1] + d[2:])                  # otherwise the layout of a single join
    ocols, icols = [c for c, _ in d["outer"]["cols"]], [c for c, _ in d["inner"]["cols"]]
    assert d["outer"]["rti"] == 2 and d["inner"]["rti"] == 1
    assert ocols[d["outer_key_col"]] == 0 and d["group_cols"] == [(0, ocols.index(2))] and d["preds"] == []
    assert icols[d["inner_key_col"]] == 0 and d["payload"] == [] and d["inner_unique"] == 1
    assert d["inner_preds"] == [(icols.index(5), g.GX_GT, DATE_Q3, 0)]
    assert sorted(icols) == [0, 5]                     # the probe side is loaded with its key and qual columns only


@needs_harness
@pytest.mark.parametrize("word", list(WORDS))
def test_build_side_quals_and_arguments(word):
    r = right(word, "qual 2 3 date_lt date -1000", "group 2.3", "target var 2.3", "target agg sum_f8 v2.5", "target agg count_star",
              "dist none", "groups 2406")
    d = parse_desc([r["desc"][0], 1] + r["desc"][2:])
    ocols = [c for c, _ in d["outer"]["cols"]]
    assert d["preds"] == [(ocols.index(2), g.GX_LT, -1000, 0)] and d["inner_preds"] == []
    assert d["aggs"][0] == (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, ocols.index(4), 0)])


@needs_harness
@pytest.mark.parametrize("word", list(WORDS))
def test_right_forms_decline(word):
    assert right(word, "group 1.6", "target var 1.6", "target agg count_star", "dist none") is None                 # probe-side GROUP BY
    assert right(word, "group 2.3", "target var 2.3", "target agg sum_f8 v1.3", "dist none") is None               # probe-side argument
    assert plan(LINEITEM, ORDERS, f"join 1.1 2.1 unique 1 {word} remote_inner", *Q4) is None                      # remote build side
    assert plan(LINEITEM, ORDERS, f"join 1.1 2.1 unique 1 {word} extra_clause", *Q4) is None                      # another join clause
    chain = ["rel 3 tuples 150000 pages 3000 cols int4! int4!", "join 1.1 2.1 unique 1", f"join 2.2 3.1 unique 1 {word}",
             "group 2.3", "target var 2.3", "target agg count_star", "dist none"]
    assert plan(LINEITEM, ORDERS, *chain) is None                                                                 # in a chain
    assert plan(LINEITEM, ORDERS, *chain[:2], f"join 2.2 3.1 unique 1", *chain[3:]) is not None                    # the INNER chain is taken


@needs_harness
def test_other_words_keep_their_meaning():
    """"right" and "semi" are still RIGHT (declined) and SEMI (taken, with the probing side as the outer slot)"""
    assert right("right", *Q4) is None
    r = plan(ORDERS, LINEITEM, "join 2.1 1.1 unique 0 semi", "qual 1 6 date_gt date -1752", "group 2.3", "target var 2.3",
             "target agg count_star", "dist none", "groups 2406")
    assert r is not None and r["desc"][1] == 1 + g.GX_JOIN_SEMI


@needs_harness
def test_cost_term():
    """the build is priced over the hashed relation, the probe side once over its key and qual columns: a larger probe
    side costs more, and so does a larger build side"""
    base = right("semi_right", *Q4)["total"]
    more_probe = right("semi_right", *Q4, lineitem=LINEITEM.replace("tuples 6000000", "tuples 60000000"))["total"]
    more_build = plan(LINEITEM, ORDERS.replace("tuples 1500000", "tuples 15000000"), "join 1.1 2.1 unique 1 semi_right", *Q4)["total"]
    assert base < more_probe and base < more_build
    # gpuexec_right_join_bytes, restated: 3 passes over the build row, 32 B of table and one bit per build row, the probe row once
    import ctypes
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "opentenbase_b200", "provider", "gpuexec_cost.h")
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "c.c")
        with open(c, "w") as f:
            f.write(f'#include "{src}"\ndouble f(double a, double b, double c, double d) {{ return gpuexec_right_join_bytes(a, b, c, d); }}\n')
        so = os.path.join(d, "c.so")
        subprocess.check_call(["cc", "-shared", "-fPIC", "-O1", "-o", so, c])
        fn = ctypes.CDLL(so).f
        fn.restype, fn.argtypes = ctypes.c_double, [ctypes.c_double] * 4
        assert fn(1e6, 12.0, 6e6, 12.0) == pytest.approx(1e6 * (36 + 32 + 0.125) + 6e6 * 12)


def _case(d, jt):
    """lineitem (key, shipdate) probes orders (key, orderdate), GROUP BY o_orderdate count(*), l_shipdate > d"""
    o, l = O.gen_orders(1, 0, 3000), O.gen_lineitem(1, 0, 3000)
    otypes = [O.GX_INT8, O.GX_INT4, O.GX_DATE, O.GX_INT4]
    ltypes = [O.GX_INT8, O.GX_FLOAT8, O.GX_FLOAT8, O.GX_FLOAT8, O.GX_FLOAT8, O.GX_DATE, O.ORC_BPCHAR1, O.ORC_BPCHAR1]
    orel, lrel = O.Rel(otypes, o), O.Rel(ltypes, l)
    sd = int(np.median(l[g.L_SHIPDATE]))
    p = g.make_plan(outer_key_col=0, group_cols=[(0, 1)], aggs=[(g.GX_AGG_COUNT_STAR, [])], est_groups=2406, join_type=jt)
    case = os.path.join(d, "right.case")
    write_case(case, [(ltypes, lrel), (otypes, orel)], {"rti": 2, "attnums": [0, 2]},
               {"rti": 1, "attnums": [0, 5], "key_col": 0, "payload_cols": [], "unique": True, "preds": [(1, g.GX_GT, sd)]},
               p, False, [1082, 20])
    return case, sd, (orel, lrel)


@needs_harness
@pytest.mark.parametrize("jt", list(WORDS.values()))
def test_descriptor_survives_plan_shipping(jt):
    from test_provider_ship_cpu import ship
    with tempfile.TemporaryDirectory() as d:
        case, sd, _ = _case(d, jt)
        toks = ship(case).strip("()").split(" ")
    assert toks[1] == str(1 + jt) and toks[-1] == "2406"


@pytest.mark.skipif(not os.path.exists(DOUBLE), reason="harness binary not built (needs /root/reference at build time)")
@pytest.mark.parametrize("jt", list(WORDS.values()))
def test_host_calls_build_without_payload_then_hash_agg_right(jt):
    with tempfile.TemporaryDirectory() as d:
        case, sd, _ = _case(d, jt)
        res = os.path.join(d, "r.res")
        with open(res, "wb") as f:
            f.write(struct.pack("<qii", 1, 1, 1))
            f.write(np.array([-1500], np.int64).tobytes()); f.write(np.array([np.int64(4).view(np.float64)]).tobytes())
            f.write(np.array([4], np.int64).tobytes()); f.write(np.zeros(2, np.uint8).tobytes())
        r = subprocess.run([DOUBLE, case], capture_output=True, text=True, timeout=120, env=dict(os.environ, GX_DOUBLE_RESULT=res))
    assert r.returncode == 0, r.stderr[-2000:]
    err = r.stderr.splitlines()
    calls = [l for l in err if l.startswith(("double: hash_build", "double: hash_agg"))]
    assert calls[0] == "double: hash_build key 0 unique 1 payload preds", calls           # the hashed relation, no payload
    assert calls[1].startswith(f"double: hash_agg_right type {jt} probe rows ") and \
        calls[1].endswith(f"key 0 table key 0 preds (1 5 {sd})"), calls                      # the probing relation, its qual
    assert calls[2].startswith("double: hash_agg outer rows") and "join 0" in calls[2] and "outer_key -1" in calls[2], calls
    assert len(calls) == 3
    assert r.stdout.split() == ["-1500", "4"]
    assert f"GPU Join Type: {'Right Semi' if jt == g.GX_JOIN_SEMI_RIGHT else 'Right Anti'}" in r.stderr
    assert "double: shutdown live tables 0 hashes 0 results 0" in err
