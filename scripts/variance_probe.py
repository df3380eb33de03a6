"""Variance and standard deviation over float8 at TPC-H scale on one GPU, next to the same plans without them, on
device-generated lineitem.

    python scripts/variance_probe.py [--sf 100] [--steps 20] [--warmup 3] [--out DIR] [--baseline-tree DIR]

Shapes:
  shipdate      stddev_samp(l_extendedprice) GROUP BY l_shipdate, against avg(l_extendedprice) GROUP BY l_shipdate
  q1            the Q1 shape (4 groups, 8 aggregates, shipdate qual), against the same with stddev_samp(l_extendedprice)
                in place of avg(l_discount) (a plan has 8 aggregates at most)
A step is one gx_hash_agg call and its fetch.  Reported per plan: the median step time and the per-kernel profile of
the variance plan (agg_smem / agg_smem_lp are the sinks of gx_k_agg it takes; agg_compact, agg_inf_scan and finalize
follow it).  The avg plan takes the specialised kernels a variance plan leaves, so the difference is the price of the
variance state.  --baseline-tree DIR: a built tree of an earlier version of this project; the plans without a variance
are timed there and here in alternation, with the general kernel forced by GX_NO_LPTILE=1 GX_NO_FEWGROUPS=1 for one
more Q1 run, so that a change of the shared kernels shows.  Prints the card's name and power limit and one JSON line;
--out also writes it to DIR/variance_probe.json."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = ("agg", "agg_smem", "agg_smem_lp", "agg_global", "agg_records", "agg_fewgroups", "agg_lptile8", "agg_lptile4",
           "agg_fast", "agg_compact", "agg_inf_scan", "finalize")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def plans(g):
    kQ, kP, kD, kT, kF, kS, kSH = range(7)
    C, K, A, S, M = g.GX_OP_COL, g.GX_OP_CONST, g.GX_OP_ADD, g.GX_OP_SUB, g.GX_OP_MUL
    disc_price = [(C, kP, 0), (K, 0, 1.0), (C, kD, 0), (S, 0, 0), (M, 0, 0)]
    charge = disc_price + [(K, 0, 1.0), (C, kT, 0), (A, 0, 0), (M, 0, 0)]
    q1 = [(g.GX_AGG_SUM_F8, [(C, kQ, 0)]), (g.GX_AGG_SUM_F8, [(C, kP, 0)]), (g.GX_AGG_SUM_F8, disc_price),
          (g.GX_AGG_SUM_F8, charge), (g.GX_AGG_AVG_F8, [(C, kQ, 0)]), (g.GX_AGG_AVG_F8, [(C, kP, 0)]),
          (g.GX_AGG_AVG_F8, [(C, kD, 0)]), (g.GX_AGG_COUNT_STAR, [])]
    q1_plan = lambda aggs: g.make_plan(preds=[(kSH, g.GX_LE, -517 - 90)], group_cols=[(0, kF), (0, kS)], aggs=aggs, est_groups=6)
    out = {"shipdate_avg": g.make_plan(group_cols=[(0, kSH)], aggs=[(g.GX_AGG_AVG_F8, [(C, kP, 0)])], est_groups=2600), "q1": q1_plan(q1)}
    sd = getattr(g, "GX_AGG_STDDEV_SAMP_F8", None)          # absent in a baseline tree from before the variances
    if sd is not None:
        out["shipdate_stddev"] = g.make_plan(group_cols=[(0, kSH)], aggs=[(sd, [(C, kP, 0)])], est_groups=2600)
        out["q1_stddev"] = q1_plan(q1[:6] + [(sd, [(C, kP, 0)])] + q1[7:])     # GX_MAX_AGGS: in place of avg(l_discount)
    return out


def lineitem(g, ctx, sf):
    no = 1_500_000 * sf
    cols = [g.L_QUANTITY, g.L_EXTENDEDPRICE, g.L_DISCOUNT, g.L_TAX, g.L_RETURNFLAG, g.L_LINESTATUS, g.L_SHIPDATE]
    return ctx.table([g.SCHEMAS[g.T_LINEITEM][c] for c in cols], no * 4 + no // 8).generate(g.T_LINEITEM, sf, 0, no, colmap=cols)


def step_ms(ctx, t, plan, steps, warmup):
    def step():
        r = ctx.hash_agg(t, plan)
        r.fetch()
        r.free()
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


def profile(ctx, t, plan, steps):
    ctx.profile(True)
    for _ in range(steps):
        r = ctx.hash_agg(t, plan)
        r.fetch()
        r.free()
    ctx.sync()
    prof = {k: round(ctx.profile_get(k)[0] / steps, 3) for k in KERNELS if ctx.profile_get(k)[1] > 0}
    ctx.profile(False)
    return prof


# one tree's plans without a variance, run in a child process with that tree's package first on sys.path
CHILD = r"""
import json, os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(1, os.path.dirname(sys.argv[2]))
import opentenbase_b200 as g
import variance_probe as P
ctx = g.Context(0)
t = P.lineitem(g, ctx, int(sys.argv[3]))
pl = P.plans(g)
print(json.dumps({k: P.step_ms(ctx, t, pl[k], int(sys.argv[4]), 3) for k in ("shipdate_avg", "q1")}))
ctx.close()
"""


def baseline_ab(tree, sf, steps, rounds=2):
    out = {"baseline": [], "this": [], "baseline_general": [], "this_general": []}
    for _ in range(rounds):
        for name, root in (("baseline", tree), ("this", HERE)):
            for env, suffix in (({}, ""), ({"GX_NO_LPTILE": "1", "GX_NO_FEWGROUPS": "1"}, "_general")):
                r = subprocess.run([sys.executable, "-c", CHILD, root, os.path.abspath(__file__), str(sf), str(steps)],
                                   capture_output=True, text=True, timeout=1800, env=dict(os.environ, **env))
                if r.returncode != 0:
                    raise RuntimeError(r.stderr[-2000:])
                out[name + suffix].append(json.loads(r.stdout.strip().splitlines()[-1]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--baseline-tree", default=None)
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import opentenbase_b200 as g
    gpu = card()
    print(f"card: {gpu}", flush=True)
    res = {"card": gpu, "sf": args.sf, "steps": args.steps, "plans": {}}
    ctx = g.Context(0)
    t = lineitem(g, ctx, args.sf)
    res["rows"] = int(t.nrows)
    pl = plans(g)
    for name, plan in pl.items():
        res["plans"][name] = {"ms": step_ms(ctx, t, plan, args.steps, args.warmup), "kernels_ms": profile(ctx, t, plan, args.steps)}
        print(json.dumps({name: res["plans"][name]}), flush=True)
    for a, b in (("shipdate_stddev", "shipdate_avg"), ("q1_stddev", "q1")):
        res[f"{a}_over_{b}"] = round(res["plans"][a]["ms"] / res["plans"][b]["ms"], 3)
    t.free()
    ctx.close()
    if args.baseline_tree:
        res["ab"] = baseline_ab(args.baseline_tree, args.sf, args.steps)
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "variance_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
