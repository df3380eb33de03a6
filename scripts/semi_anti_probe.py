"""Aggregates over SEMI and ANTI hash joins at TPC-H scale on one GPU: the existence probe of gx_k_agg against the
aggregate with no join and against the INNER plan, on device-generated tables.

    python scripts/semi_anti_probe.py [--sf 100] [--steps 20] [--warmup 3] [--out DIR]

Shapes (DATE_Q3 = 1995-03-15):
  q4     orders SEMI lineitem[l_shipdate > DATE_Q3] on the order key, GROUP BY o_orderdate count(*)
         (lineitem: a key-ordered, non-unique build side, about 4 rows per key)
  q22    customer ANTI orders on c_custkey = o_custkey, GROUP BY c_mktsegment count(*)
         (orders: an unordered, non-unique build side, about 10 rows per key)
  semi   lineitem SEMI orders[o_orderdate < DATE_Q3], GROUP BY l_shipdate count(*), sum(l_extendedprice), against the INNER
         plan with the same outer-only GROUP BY; both on the unique build
  q4_right_semi / q4_right_anti   the right form of q4 (gx_hash_agg_right): orders hashed (unique, key-ordered),
         lineitem[l_shipdate > DATE_Q3] probing it, GROUP BY o_orderdate count(*)
  q22_right_anti                  the right form of q22: customer hashed (unique), orders probing it, GROUP BY c_mktsegment
Per shape: the median step time over --steps steps (table build + probe/aggregate + fetch), the per-kernel profile of
one more pass over the same steps, and the bytes the probe must read (outer columns + the join table once) over its
kernel time against the H100 SXM's 3.35 TB/s.  Built-in checks: on the unique build the SEMI counts equal the INNER
counts exactly, and per group count(SEMI) + count(ANTI) equals the count with no join exactly (sums within 1e-9
relative); each right form's counts equal its left form's, group for group.  For a right form the kernel time is the
marking probe's (probe_mark), its bytes the probe side's key and qual columns plus the join table and the bitmap once.
Prints the card's name and power limit and one JSON line; --out also writes it to DIR/semi_anti_probe.json."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import opentenbase_b200 as g                                     # noqa: E402

DATE_Q3 = -1752
HBM_TBPS = 3.35
KERNELS = ("probe_mark", "probe_mark_wide", "probe_mark_compact", "probe_mark_walk", "filter", "probe_agg", "agg", "probe_agg_exist_wide", "probe_agg_exist_compact", "probe_agg_exist_narrow", "build",
           "build_expand", "agg_smem", "agg_smem_lp", "agg_global", "agg_records", "agg_compact", "agg_inf_scan")
SLOT_BYTES = {"probe_agg_exist_wide": 16, "probe_agg_exist_compact": 8, "probe_agg_exist_narrow": 4}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def by_key(keys, aggs):
    return {tuple(int(v) for v in k): a for k, a in zip(keys.tolist(), aggs)}


def measure(ctx, name, inner, ikey, ipreds, unique, outer, plan, outer_bytes_per_row, steps, warmup):
    """median step ms, kernel profile (ms per step), bytes / probe time; returns (summary, last result)"""
    def step():
        ht = ctx.hash_build(inner, ikey, [], unique=unique, preds=ipreds) if inner is not None else None
        r = ctx.hash_agg(outer, plan, ht)
        out = r.fetch()
        slots = ht.nslots if ht is not None else 0
        r.free()
        if ht is not None:
            ht.free()
        return out, slots
    for _ in range(warmup):
        step()
    times = []
    for _ in range(steps):
        ctx.timer_start()
        out, slots = step()
        times.append(ctx.timer_stop())
    ctx.profile(True)
    for _ in range(steps):
        step()
    prof = {k: ctx.profile_get(k) for k in KERNELS}
    ctx.profile(False)
    prof = {k: {"ms_per_step": round(ms / steps, 4), "launches_per_step": n / steps} for k, (ms, n) in prof.items() if n}
    kname = "probe_agg" if inner is not None else "agg"
    kms = prof[kname]["ms_per_step"]
    fmt = [k for k in SLOT_BYTES if k in prof]
    table_bytes = slots * (SLOT_BYTES[fmt[0]] if fmt else 16)
    nbytes = outer.nrows * outer_bytes_per_row + table_bytes
    s = {"shape": name, "median_step_ms": round(float(np.median(times)), 4), "min_step_ms": round(float(np.min(times)), 4),
         "steps": steps, "kernel": kname, "kernel_ms": kms, "format": fmt[0] if fmt else None, "outer_rows": outer.nrows,
         "bytes": nbytes, "gb_per_s": round(nbytes / (kms * 1e-3) / 1e9, 1), "frac_of_3.35TBps": round(nbytes / (kms * 1e-3) / (HBM_TBPS * 1e12), 3),
         "profile": prof}
    print(json.dumps(s), flush=True)
    return s, out


def measure_right(ctx, name, build, bkey, probe, pkey, ppreds, jt, plan, probe_bytes_per_row, steps, warmup):
    """measure() for gx_hash_agg_right: the build (no payload: the row number) is timed with every step"""
    def step():
        ht = ctx.hash_build(build, bkey, [], unique=True)
        r = ctx.hash_agg_right(probe, pkey, build, ht, jt, plan, probe_preds=ppreds)
        out = r.fetch()
        slots = ht.nslots
        r.free()
        ht.free()
        return out, slots
    for _ in range(warmup):
        step()
    times = []
    for _ in range(steps):
        ctx.timer_start()
        out, slots = step()
        times.append(ctx.timer_stop())
    ctx.profile(True)
    for _ in range(steps):
        step()
    prof = {k: ctx.profile_get(k) for k in KERNELS}
    ctx.profile(False)
    prof = {k: {"ms_per_step": round(ms / steps, 4), "launches_per_step": n / steps} for k, (ms, n) in prof.items() if n}
    kms = prof["probe_mark"]["ms_per_step"]
    fmt = [k for k in ("probe_mark_compact", "probe_mark_wide", "probe_mark_walk") if k in prof]
    nbytes = probe.nrows * probe_bytes_per_row + slots * (8 if fmt == ["probe_mark_compact"] else 16) + build.nrows // 8
    s = {"shape": name, "median_step_ms": round(float(np.median(times)), 4), "min_step_ms": round(float(np.min(times)), 4),
         "steps": steps, "kernel": "probe_mark", "kernel_ms": kms, "format": fmt[0] if fmt else None, "outer_rows": probe.nrows,
         "bytes": nbytes, "gb_per_s": round(nbytes / (kms * 1e-3) / 1e9, 1), "frac_of_3.35TBps": round(nbytes / (kms * 1e-3) / (HBM_TBPS * 1e12), 3),
         "profile": prof}
    print(json.dumps(s), flush=True)
    return s, out


def same_counts(right, left):
    """per group: the right form's count equals the left form's exactly"""
    kr, kl = by_key(right[0], right[1]), by_key(left[0], left[1])
    assert set(kr) == set(kl), "group keys differ"
    for k in kl:
        assert int(kr[k][0:1].view(np.int64)[0]) == int(kl[k][0:1].view(np.int64)[0]), k
    return len(kl)


def counts_add_up(semi, anti, none, sum_col=None):
    """per group: count(SEMI) + count(ANTI) == count(no join) exactly; sums within 1e-9 relative"""
    ks, ka, kn = by_key(semi[0], semi[1]), by_key(anti[0], anti[1]), by_key(none[0], none[1])
    assert set(ks) | set(ka) == set(kn), "group keys differ"
    for k, a in kn.items():
        c = lambda d: int(d[k][0:1].view(np.int64)[0]) if k in d else 0
        assert c(ks) + c(ka) == int(a[0:1].view(np.int64)[0]), k
        if sum_col is not None:
            s = lambda d: float(d[k][sum_col]) if k in d else 0.0
            assert abs(s(ks) + s(ka) - float(a[sum_col])) <= 1e-9 * abs(float(a[sum_col])), k
    return len(kn)


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
    orders = ctx.table([g.GX_INT8, g.GX_INT4, g.GX_DATE], no).generate(g.T_ORDERS, sf, 0, no, colmap=[g.O_ORDERKEY, g.O_CUSTKEY, g.O_ORDERDATE])
    lineitem = ctx.table([g.GX_INT8, g.GX_FLOAT8, g.GX_DATE], no * 4 + no // 8).generate(
        g.T_LINEITEM, sf, 0, no, colmap=[g.L_ORDERKEY, g.L_EXTENDEDPRICE, g.L_SHIPDATE])
    customer = ctx.table([g.GX_INT4, g.GX_CHAR], nc).generate(g.T_CUSTOMER, sf, 0, nc)
    print(f"generated {orders.nrows} orders, {lineitem.nrows} lineitem, {customer.nrows} customer rows in {time.time() - t0:.1f} s", flush=True)
    cnt = [(g.GX_AGG_COUNT_STAR, [])]
    res = {"card": gpu, "sf": sf, "shapes": []}

    def plan(key, gcol, aggs, est, jt):
        return g.make_plan(outer_key_col=key, group_cols=[(0, gcol)], aggs=aggs, est_groups=est, join_type=jt)

    run = lambda *a: measure(ctx, *a, steps=args.steps, warmup=args.warmup)
    # Q4: orders SEMI lineitem[l_shipdate > DATE_Q3]; the outer side reads o_orderkey (8 B) and o_orderdate (4 B)
    lq = [(2, g.GX_GT, DATE_Q3)]
    s, q4s = run("q4_semi", lineitem, 0, lq, False, orders, plan(0, 2, cnt, 2406, g.GX_JOIN_SEMI), 12)
    res["shapes"].append(s)
    s, q4a = run("q4_anti", lineitem, 0, lq, False, orders, plan(0, 2, cnt, 2406, g.GX_JOIN_ANTI), 12)
    res["shapes"].append(s)
    s, q4n = run("q4_nojoin", None, 0, (), False, orders, g.make_plan(group_cols=[(0, 2)], aggs=cnt, est_groups=2406), 4)
    res["shapes"].append(s)
    res["q4_groups_checked"] = counts_add_up(q4s, q4a, q4n)
    # the right forms of Q4: lineitem[l_shipdate > DATE_Q3] probes orders (l_orderkey 8 B + l_shipdate 4 B per probe row)
    rrun = lambda *a: measure_right(ctx, *a, steps=args.steps, warmup=args.warmup)
    rplan = g.make_plan(group_cols=[(0, 2)], aggs=cnt, est_groups=2406)
    s, q4rs = rrun("q4_right_semi", orders, 0, lineitem, 0, lq, g.GX_JOIN_SEMI_RIGHT, rplan, 12)
    res["shapes"].append(s)
    s, q4ra = rrun("q4_right_anti", orders, 0, lineitem, 0, lq, g.GX_JOIN_ANTI_RIGHT, rplan, 12)
    res["shapes"].append(s)
    res["q4_right_equals_left_groups"] = same_counts(q4rs, q4s) + same_counts(q4ra, q4a)
    # Q22: customer ANTI orders on c_custkey = o_custkey (c_custkey 4 B, c_mktsegment 1 B)
    s, q22a = run("q22_anti", orders, 1, (), False, customer, plan(0, 1, cnt, 5, g.GX_JOIN_ANTI), 5)
    res["shapes"].append(s)
    s, q22s = run("q22_semi", orders, 1, (), False, customer, plan(0, 1, cnt, 5, g.GX_JOIN_SEMI), 5)
    res["shapes"].append(s)
    s, q22n = run("q22_nojoin", None, 0, (), False, customer, g.make_plan(group_cols=[(0, 1)], aggs=cnt, est_groups=5), 1)
    res["shapes"].append(s)
    res["q22_groups_checked"] = counts_add_up(q22s, q22a, q22n)
    # the right form of Q22: orders probes customer (o_custkey 4 B per probe row)
    s, q22ra = rrun("q22_right_anti", customer, 0, orders, 1, (), g.GX_JOIN_ANTI_RIGHT,
                    g.make_plan(group_cols=[(0, 1)], aggs=cnt, est_groups=5), 4)
    res["shapes"].append(s)
    res["q22_right_equals_left_groups"] = same_counts(q22ra, q22a)
    # lineitem SEMI orders[o_orderdate < DATE_Q3] against INNER, GROUP BY l_shipdate (8 + 4 + 8 B per outer row)
    oq = [(2, g.GX_LT, DATE_Q3)]
    aggs = cnt + [(g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)])]
    s, ls = run("li_semi", orders, 0, oq, True, lineitem, plan(0, 2, aggs, 2526, g.GX_JOIN_SEMI), 20)
    res["shapes"].append(s)
    s, li = run("li_inner", orders, 0, oq, True, lineitem, plan(0, 2, aggs, 2526, g.GX_JOIN_INNER), 20)
    res["shapes"].append(s)
    s, la = run("li_anti", orders, 0, oq, True, lineitem, plan(0, 2, aggs, 2526, g.GX_JOIN_ANTI), 20)
    res["shapes"].append(s)
    s, ln = run("li_nojoin", None, 0, (), False, lineitem, g.make_plan(group_cols=[(0, 2)], aggs=aggs, est_groups=2526), 12)
    res["shapes"].append(s)
    ks, ki = by_key(ls[0], ls[1]), by_key(li[0], li[1])
    assert set(ks) == set(ki) and all(int(ks[k][0:1].view(np.int64)[0]) == int(ki[k][0:1].view(np.int64)[0]) for k in ks), \
        "SEMI and INNER counts differ on the unique build"
    res["li_semi_equals_inner_groups"] = len(ks)
    res["li_groups_checked"] = counts_add_up(ls, la, ln, sum_col=1)
    print(json.dumps({k: v for k, v in res.items() if k != "shapes"}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "semi_anti_probe.json"), "w") as f:
            json.dump(res, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
