"""Aggregates over a chain of unique INNER hash joins at TPC-H scale on one GPU: gx_hash_agg_joins' single probe pass
against the device-side alternative without it, on device-generated tables.

    python scripts/star_agg_probe.py [--sf 100] [--steps 20] [--warmup 3] [--out DIR]

Shapes (D = 1995-03-15):
  seg   lineitem[l_shipdate > D] -> orders[o_orderdate < D] (payload o_custkey, o_orderdate) -> customer (payload
        c_mktsegment), GROUP BY c_mktsegment: count(*), sum(l_extendedprice * (1 - l_discount))
  q3f   the same chain with customer[c_mktsegment = 'BUILDING'], GROUP BY l_orderkey, o_orderdate (TPC-H Q3; the
        generator's o_shippriority is always 0)
Each shape runs fused (gx_hash_agg_joins) and materialised (gx_hash_probe writes lineitem JOIN orders, gx_hash_agg joins
customer over it); q3f also runs plans.q3_datanode at N = 1.  A step builds the join tables, runs the plan and fetches
the groups.  Reported per run: the median step time over --steps steps after --warmup, the per-kernel profile of one
more pass, and for the fused probe the bytes it must read (lineitem's four columns, the orders table in the form step 1
reads and customer's 16-byte table, each once) over its kernel time against the H100 SXM's 3.35 TB/s.  Built-in checks:
the same group sets, equal counts, sums within 1e-9 relative.  Prints the card's name and power limit and one JSON line;
--out also writes it to DIR/star_agg_probe.json."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import opentenbase_b200 as g                                     # noqa: E402
from opentenbase_b200 import plans                               # noqa: E402

D = plans.DATE_Q3
HBM_TBPS = 3.35
KERNELS = ("probe_agg_chain", "probe_agg_chain_wide", "probe_agg_chain_compact", "probe_agg_chain_narrow", "probe_agg",
           "probe_records", "probe", "build", "build_expand", "agg_smem", "agg_smem_lp", "agg_global", "agg_records",
           "runagg", "agg_inf_scan", "scan_filter", "partition")
SLOT_BYTES = {"probe_agg_chain_wide": 16, "probe_agg_chain_compact": 8, "probe_agg_chain_narrow": 4}
# lineitem as generated here: l_orderkey, l_extendedprice, l_discount, l_shipdate
LK, LP, LD, LS = 0, 1, 2, 3


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def groups(res, nkeys):
    keys, aggs, _ = res
    return {tuple(int(v) for v in k[:nkeys]): (int(a[0:1].view(np.int64)[0]), float(a[1])) for k, a in zip(keys, aggs)}


def agree(a, b):
    assert set(a) == set(b), f"group sets differ: {len(a)} vs {len(b)}"
    for k in a:
        assert a[k][0] == b[k][0], f"count of {k}: {a[k][0]} vs {b[k][0]}"
        assert abs(a[k][1] - b[k][1]) <= 1e-9 * max(abs(a[k][1]), abs(b[k][1])), f"sum of {k}: {a[k][1]} vs {b[k][1]}"
    return len(a)


def measure(ctx, name, step, steps, warmup):
    """median step ms and the kernel profile (ms per step) of one more pass; returns (summary, last result)"""
    for _ in range(warmup):
        step()
    times = []
    for _ in range(steps):
        ctx.sync()
        t0 = time.perf_counter()
        out = step()
        ctx.sync()
        times.append((time.perf_counter() - t0) * 1e3)
    ctx.profile(True)
    for _ in range(steps):
        out = step()
    ctx.sync()
    prof = {k: round(ctx.profile_get(k)[0] / steps, 3) for k in KERNELS if ctx.profile_get(k)[1] > 0}
    ctx.profile(False)
    s = {"name": name, "median_ms": round(float(np.median(times)), 3), "min_ms": round(min(times), 3), "kernels_ms": prof}
    print(json.dumps(s), flush=True)
    return s, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sf = args.sf
    no, nc = 1_500_000 * sf, 150_000 * sf
    gpu = card()
    print(f"card: {gpu}", flush=True)
    ctx = g.Context(0)
    t0 = time.time()
    orders = ctx.table(g.SCHEMAS[g.T_ORDERS], no).generate(g.T_ORDERS, sf, 0, no)
    line = ctx.table([g.GX_INT8, g.GX_FLOAT8, g.GX_FLOAT8, g.GX_DATE], no * 4 + no // 8).generate(
        g.T_LINEITEM, sf, 0, no, colmap=[g.L_ORDERKEY, g.L_EXTENDEDPRICE, g.L_DISCOUNT, g.L_SHIPDATE])
    cust = ctx.table(g.SCHEMAS[g.T_CUSTOMER], nc).generate(g.T_CUSTOMER, sf, 0, nc)
    print(f"generated {orders.nrows} orders, {line.nrows} lineitem, {cust.nrows} customer rows in {time.time() - t0:.1f} s", flush=True)
    rev = plans.revenue_expr(LP, LD)
    oq = [(g.O_ORDERDATE, g.GX_LT, D)]
    res = {"card": gpu, "sf": sf, "steps": args.steps, "runs": []}
    run = lambda name, step: measure(ctx, name, step, args.steps, args.warmup)

    def fused(cpreds, gcols, est):
        plan = g.make_plan(preds=[(LS, g.GX_GT, D)], group_cols=gcols, aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, rev)],
                           est_groups=est)
        info = {}

        def step():
            ho = ctx.hash_build(orders, g.O_ORDERKEY, [g.O_CUSTKEY, g.O_ORDERDATE], unique=True, preds=oq)
            hc = ctx.hash_build(cust, g.C_CUSTKEY, [g.C_MKTSEGMENT], unique=True, preds=cpreds)
            info.update(o_slots=ho.nslots, c_slots=hc.nslots)
            r = ctx.hash_agg_joins(line, [(ho, (0, LK)), (hc, (1, 0))], plan)
            out = r.fetch()
            r.free(); hc.free(); ho.free()
            return out
        return step, info

    def materialised(cpreds, outer_cols, gcols, est):
        """lineitem JOIN orders written out (outer_cols + o_custkey, o_orderdate), then aggregated over JOIN customer"""
        nout = len(outer_cols)
        p, d = outer_cols.index(LP), outer_cols.index(LD)
        plan = g.make_plan(outer_key_col=nout, group_cols=gcols, aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, plans.revenue_expr(p, d))],
                           est_groups=est)

        def step():
            ho = ctx.hash_build(orders, g.O_ORDERKEY, [g.O_CUSTKEY, g.O_ORDERDATE], unique=True, preds=oq)
            hc = ctx.hash_build(cust, g.C_CUSTKEY, [g.C_MKTSEGMENT], unique=True, preds=cpreds)
            j = ctx.hash_probe(line, LK, ho, outer_cols, preds=[(LS, g.GX_GT, D)])
            r = ctx.hash_agg(j, plan, hc)
            out = r.fetch()
            r.free(); j.free(); hc.free(); ho.free()
            return out
        return step

    def probe_share(s, info):
        """bytes the fused probe must read over its kernel time: lineitem's four columns (28 B a row), step 1's table in the
        format it read, customer's 16-byte table"""
        fmt = [k for k in SLOT_BYTES if k in s["kernels_ms"]]
        nbytes = line.nrows * 28 + info["o_slots"] * SLOT_BYTES[fmt[0]] + info["c_slots"] * 16
        ms = s["kernels_ms"]["probe_agg_chain"]
        s.update(probe_format=fmt[0], probe_bytes=nbytes, probe_tbps=round(nbytes / ms / 1e9, 3),
                 probe_share_of_hbm=round(nbytes / ms / 1e9 / HBM_TBPS, 3))

    # seg: GROUP BY c_mktsegment
    step, info = fused([], [(2, 0)], 5)
    s, seg_f = run("seg_fused", step)
    probe_share(s, info)
    res["runs"].append(s)
    s, seg_m = run("seg_materialised", materialised([], [LP, LD], [(1, 0)], 5))
    res["runs"].append(s)
    res["seg_groups_checked"] = agree(groups(seg_f, 1), groups(seg_m, 1))

    # q3f: customer[c_mktsegment = 'BUILDING'], GROUP BY l_orderkey, o_orderdate
    seg = [(g.C_MKTSEGMENT, g.GX_EQ, plans.SEGMENT_Q3)]
    est = no // 100
    step, info = fused(seg, [(0, LK), (1, 1)], est)
    s, q3_f = run("q3f_fused", step)
    probe_share(s, info)
    res["runs"].append(s)
    s, q3_m = run("q3f_materialised", materialised(seg, [LK, LP, LD], [(0, 0), (0, 4)], est))
    res["runs"].append(s)

    def q3dn():
        r = plans.q3_datanode(ctx, cust, orders, line, {"custkey": g.C_CUSTKEY, "mktsegment": g.C_MKTSEGMENT},
                              {"orderkey": g.O_ORDERKEY, "custkey": g.O_CUSTKEY, "orderdate": g.O_ORDERDATE, "shippriority": g.O_SHIPPRIORITY},
                              {"orderkey": LK, "extendedprice": LP, "discount": LD, "shipdate": LS})
        out = r.fetch()
        r.free()
        return out
    s, q3_d = run("q3f_q3_datanode", q3dn)
    res["runs"].append(s)
    res["q3f_groups_checked"] = agree(groups(q3_f, 2), groups(q3_m, 2))
    # q3_datanode has sum(revenue) only, and a third group column (o_shippriority, always 0)
    dn = {(int(k[0]), int(k[1])): float(a[0]) for k, a in zip(q3_d[0], q3_d[1])}
    assert all(int(k[2]) == 0 for k in q3_d[0]), "o_shippriority is not 0"
    fq = groups(q3_f, 2)
    assert set(dn) == set(fq), f"q3_datanode groups differ: {len(dn)} vs {len(fq)}"
    assert all(abs(dn[k] - fq[k][1]) <= 1e-9 * max(abs(dn[k]), abs(fq[k][1])) for k in fq), "q3_datanode sums differ"
    res["q3f_datanode_groups_checked"] = len(dn)
    res["checks"] = True
    print(json.dumps({k: v for k, v in res.items()}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "star_agg_probe.json"), "w") as f:
            json.dump(res, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
