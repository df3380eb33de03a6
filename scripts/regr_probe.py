"""The SQL:2003 binary aggregates (corr, regr_slope, ...) at TPC-H scale on one GPU, next to the same plans without
them, on device-generated lineitem and orders.

    python scripts/regr_probe.py [--sf 100] [--steps 20] [--warmup 3] [--out DIR] [--baseline-tree DIR]

Shapes:
  shipdate   corr, regr_slope and regr_intercept(l_extendedprice, l_discount) GROUP BY l_shipdate, against its avg twin
             avg(l_extendedprice) GROUP BY l_shipdate
  q1         the Q1 shape (4 groups, 8 aggregates, shipdate qual), against the same with
             covar_samp(l_extendedprice, l_discount) in place of avg(l_discount)
A step is one gx_hash_agg call and its fetch; reported: the median step time and the per-kernel profile.
--baseline-tree DIR: a built tree of an earlier version of this project.  Plans without a regression aggregate are timed
there and here in alternation, two rounds, so that a change of the shared kernels shows: bench.py's headline, the
variance_probe.py shapes (avg and stddev GROUP BY l_shipdate, Q1 and Q1 with a stddev, and Q1 forced onto the
lane-private gx_k_agg by GX_NO_LPTILE=1 GX_NO_FEWGROUPS=1), and lineitem SEMI orders[o_orderdate < 1995-03-15] GROUP BY
l_returnflag, l_linestatus, which the lane-private existence probe of gx_k_agg runs (the Q4 / Q21 kind of plan).
Prints the card's name and power limit and one JSON line; --out also writes it to DIR/regr_probe.json."""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(HERE, "scripts"))
import variance_probe as VP                                    # noqa: E402  (card, lineitem, step_ms, profile)

KERNELS = VP.KERNELS + ("probe_agg_exist_wide", "probe_agg_exist_compact", "probe_agg_exist_narrow")


def plans(g):
    kQ, kP, kD, kT, kF, kS, kSH = range(7)                      # the columns VP.lineitem generates
    C, ARG2 = g.GX_OP_COL, g.GX_OP_ARG2
    pair = [(C, kP, 0), (ARG2, 0, 0), (C, kD, 0)]
    vp = VP.plans(g)
    q1 = [(a.fn, [(o.op, o.col, o.k) for o in a.arg.ops[:a.arg.nops]]) for a in vp["q1"].aggs[:vp["q1"].n_aggs]]
    return {
        "shipdate_avg": vp["shipdate_avg"],
        "shipdate_regr": g.make_plan(group_cols=[(0, kSH)], est_groups=2600,
                                     aggs=[(g.GX_AGG_CORR_F8, pair), (g.GX_AGG_REGR_SLOPE_F8, pair), (g.GX_AGG_REGR_INTERCEPT_F8, pair)]),
        "q1": vp["q1"],
        "q1_covar": g.make_plan(preds=[(kSH, g.GX_LE, -517 - 90)], group_cols=[(0, kF), (0, kS)], est_groups=6,
                                aggs=q1[:6] + [(g.GX_AGG_COVAR_SAMP_F8, pair)] + q1[7:]),
    }


# one tree's plans without a regression aggregate, in a child process with that tree's package first on sys.path
CHILD = r"""
import json, os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(1, os.path.join(sys.argv[1], "scripts")); sys.path.insert(2, sys.argv[2])
import opentenbase_b200 as g
import variance_probe as P
sf, steps = int(sys.argv[3]), int(sys.argv[4])
ctx = g.Context(0)
t = P.lineitem(g, ctx, sf)
pl = P.plans(g)
out = {k: P.step_ms(ctx, t, pl[k], steps, 3) for k in ("shipdate_avg", "shipdate_stddev", "q1", "q1_stddev")}
os.environ["GX_NO_LPTILE"] = os.environ["GX_NO_FEWGROUPS"] = "1"     # read per call: Q1 on the lane-private gx_k_agg
out["q1_general"] = P.step_ms(ctx, t, pl["q1"], steps, 3)
del os.environ["GX_NO_LPTILE"], os.environ["GX_NO_FEWGROUPS"]
t.free()
# lineitem SEMI orders[o_orderdate < 1995-03-15] GROUP BY l_returnflag, l_linestatus: the lane-private existence probe
no = 1_500_000 * sf
ocols = [g.O_ORDERKEY, g.O_ORDERDATE]
o = ctx.table([g.SCHEMAS[g.T_ORDERS][c] for c in ocols], no).generate(g.T_ORDERS, sf, 0, no, colmap=ocols)
h = ctx.hash_build(o, 0, [], unique=True, preds=[(1, g.GX_LT, -1752)])   # semi_anti_probe.DATE_Q3
lcols = [g.L_ORDERKEY, g.L_EXTENDEDPRICE, g.L_RETURNFLAG, g.L_LINESTATUS]
l = ctx.table([g.SCHEMAS[g.T_LINEITEM][c] for c in lcols], no * 4 + no // 8).generate(g.T_LINEITEM, sf, 0, no, colmap=lcols)
semi = g.make_plan(outer_key_col=0, group_cols=[(0, 2), (0, 3)], est_groups=6, strategy=1, join_type=g.GX_JOIN_SEMI,
                   aggs=[(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])])
def step():
    r = ctx.hash_agg(l, semi, h); r.fetch(); r.free()
import time, numpy as np
for _ in range(3): step()
ts = []
for _ in range(steps):
    ctx.sync(); t0 = time.perf_counter(); step(); ctx.sync(); ts.append((time.perf_counter() - t0) * 1e3)
out["semi_lp"] = round(float(np.median(ts)), 3)
print(json.dumps(out))
ctx.close()
"""


def bench_ms(root, steps):
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", "3"],
                       capture_output=True, text=True, timeout=1800, cwd=root)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-2000:])
    return round(json.loads(r.stdout.strip().splitlines()[-1])["ms_per_step"], 3)


def baseline_ab(tree, sf, steps, rounds=2):
    out = {"baseline": [], "this": []}
    for _ in range(rounds):
        for name, root in (("baseline", tree), ("this", HERE)):
            row = {"bench_ms_per_step": bench_ms(root, steps)}
            r = subprocess.run([sys.executable, "-c", CHILD, root, os.path.join(HERE, "scripts"), str(sf), str(steps)],
                               capture_output=True, text=True, timeout=1800)
            if r.returncode != 0:
                raise RuntimeError(r.stderr[-2000:])
            row.update(json.loads(r.stdout.strip().splitlines()[-1]))
            out[name].append(row)
            print(json.dumps({name: row}), flush=True)
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
    gpu = VP.card()
    print(f"card: {gpu}", flush=True)
    res = {"card": gpu, "sf": args.sf, "steps": args.steps, "plans": {}}
    ctx = g.Context(0)
    t = VP.lineitem(g, ctx, args.sf)
    res["rows"] = int(t.nrows)
    for name, plan in plans(g).items():
        ms = VP.step_ms(ctx, t, plan, args.steps, args.warmup)
        ctx.profile(True)
        for _ in range(args.steps):
            r = ctx.hash_agg(t, plan)
            r.fetch()
            r.free()
        ctx.sync()
        prof = {k: round(ctx.profile_get(k)[0] / args.steps, 3) for k in KERNELS if ctx.profile_get(k)[1] > 0}
        ctx.profile(False)
        res["plans"][name] = {"ms": ms, "kernels_ms": prof}
        print(json.dumps({name: res["plans"][name]}), flush=True)
    for a, b in (("shipdate_regr", "shipdate_avg"), ("q1_covar", "q1")):
        res[f"{a}_over_{b}"] = round(res["plans"][a]["ms"] / res["plans"][b]["ms"], 3)
    t.free()
    ctx.close()
    if args.baseline_tree:
        res["ab"] = baseline_ab(os.path.abspath(args.baseline_tree), args.sf, args.steps)
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "regr_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
