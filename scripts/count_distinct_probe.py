"""count(DISTINCT col) at TPC-H scale on one GPU: what stage 1 (the plan grouped by its key plus col) and the fold
(agg_distinct_fold: pairs back to the plan's groups) each cost, on device-generated tables.

    python scripts/count_distinct_probe.py [--sf 100] [--steps 20] [--warmup 3] [--out DIR]

Shapes:
  orders    count(DISTINCT o_custkey) GROUP BY o_orderdate
  lineitem  count(DISTINCT l_orderkey) GROUP BY l_shipdate (close to one pair per row)
  join      lineitem JOIN orders ON l_orderkey = o_orderkey (unique, payload o_orderdate),
            count(DISTINCT l_orderkey) GROUP BY o_orderdate (stage 1 takes the run-aggregate kernel)
A step is one gx_hash_agg call and its group count; the join table is built once, outside the steps.  Reported per
shape: the median step time of the DISTINCT plan (total_ms), the median step time of its stage-1 plan run alone
(stage1_ms: the same plan with col as a group column and count(*)), the fold's profiled time per step (fold_ms), the
number of (group, value) pairs, and the stage-1 kernels that ran.  Built-in check: the distinct counts add up to the
pair count (no argument is NULL here).  Prints the card's name and power limit and one JSON line; --out also writes
it to DIR/count_distinct_probe.json."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import opentenbase_b200 as g                                     # noqa: E402

KERNELS = ("agg", "probe_agg", "agg_smem", "agg_smem_lp", "agg_global", "agg_records", "agg_fewgroups", "runagg",
           "radix_partition", "radix_agg", "agg_distinct_fold")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def median_ms(ctx, step, steps, warmup):
    for _ in range(warmup):
        step()
    times = []
    for _ in range(steps):
        ctx.sync()
        t0 = time.perf_counter()
        step()
        ctx.sync()
        times.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(times)), 3)


def shape(ctx, name, t, gcol, arg, steps, warmup, ht=None, okey=-1):
    """one shape's numbers, or its error (a stage-1 table of one record per pair may not fit HBM: GX_ERR_NOMEM)"""
    try:
        return measure(ctx, name, t, gcol, arg, steps, warmup, ht, okey)
    except g.GxError as e:
        out = {"name": name, "rows": int(t.nrows), "error": str(e)}
        print(json.dumps(out), flush=True)
        return out


def measure(ctx, name, t, gcol, arg, steps, warmup, ht, okey):
    est = t.nrows
    dplan = g.make_plan(outer_key_col=okey, group_cols=[gcol], aggs=[(g.GX_AGG_COUNT_DISTINCT, [(g.GX_OP_COL, arg, 0)])],
                        est_groups=est)
    splan = g.make_plan(outer_key_col=okey, group_cols=[gcol, (0, arg)], aggs=[(g.GX_AGG_COUNT_STAR, [])], est_groups=est)

    def run(plan):
        r = ctx.hash_agg(t, plan, ht)
        n = r.ngroups
        r.free()
        return n

    total = median_ms(ctx, lambda: run(dplan), steps, warmup)
    stage1 = median_ms(ctx, lambda: run(splan), steps, warmup)
    ctx.profile(True)
    for _ in range(steps):
        run(dplan)
    ctx.sync()
    prof = {k: round(ctx.profile_get(k)[0] / steps, 3) for k in KERNELS if ctx.profile_get(k)[1] > 0}
    ctx.profile(False)
    r = ctx.hash_agg(t, dplan, ht)
    _, aggs, _ = r.fetch()
    r.free()
    s = ctx.hash_agg(t, splan, ht)
    pairs = s.ngroups
    s.free()
    assert int(aggs[:, 0].view(np.int64).sum()) == pairs, "distinct counts do not add up to the pair count"
    out = {"name": name, "total_ms": total, "stage1_ms": stage1, "fold_ms": prof.get("agg_distinct_fold"), "pairs": int(pairs),
           "groups": int(aggs.shape[0]), "rows": int(t.nrows), "kernels_ms": prof}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sf, no = args.sf, 1_500_000 * args.sf
    gpu = card()
    print(f"card: {gpu}", flush=True)
    ctx = g.Context(0)
    res = {"card": gpu, "sf": sf, "steps": args.steps, "runs": []}
    orders = ctx.table(g.SCHEMAS[g.T_ORDERS], no).generate(g.T_ORDERS, sf, 0, no)
    res["runs"].append(shape(ctx, "orders", orders, (0, g.O_ORDERDATE), g.O_CUSTKEY, args.steps, args.warmup))
    line = ctx.table([g.GX_INT8, g.GX_DATE], no * 4 + no // 8).generate(g.T_LINEITEM, sf, 0, no, colmap=[g.L_ORDERKEY, g.L_SHIPDATE])
    res["runs"].append(shape(ctx, "lineitem", line, (0, 1), 0, args.steps, args.warmup))
    ht = ctx.hash_build(orders, g.O_ORDERKEY, [g.O_ORDERDATE], unique=True)
    res["runs"].append(shape(ctx, "join", line, (1, 0), 0, args.steps, args.warmup, ht=ht, okey=0))
    ht.free(); line.free(); orders.free()
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "count_distinct_probe.json"), "w") as f:
            json.dump(res, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
