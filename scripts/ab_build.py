"""A/B of two built trees of this project on one GPU: the headline benchmark alternated old, new, old, new, ...,
the key-ordered build alone at SF100, the join table's statistics on a TPC-H-style key set, and the configs[2]
outputs of every run compared against the first old run.

    python scripts/ab_build.py --old <tree> --new <tree> --out <dir> [--rounds 3] [--steps 50]

Each tree must have been built (libgpuexec.so, oracle).  Writes <dir>/ab.json and prints a summary."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

# runs inside one tree (its package on sys.path): the fill alone at SF100 and the table's statistics on a bunched key set
PROBE = r"""
import json, sys
import numpy as np
import opentenbase_b200 as g
sf = 100
ctx = g.Context(0)
no = 1_500_000 * sf
ot = ctx.table([g.GX_INT8, g.GX_DATE], no); ot.generate(g.T_ORDERS, sf, 0, no, colmap=[g.O_ORDERKEY, g.O_ORDERDATE])
for _ in range(3):
    ctx.hash_build(ot, 0, [1], unique=True).free()
ctx.profile(True)
reps = 20
for _ in range(reps):
    ht = ctx.hash_build(ot, 0, [1], unique=True); info = ht.info(); nent = ht.nentries; ht.free()
names = ("build", "build_bounds", "build_sample", "build_fill_staged", "build_fill_rows", "build_sorted_search", "build_compact",
         "build_narrow", "build_narrow_refill")
ph = {k: ctx.profile_get(k) for k in names}
ctx.profile(False)
ot.free()
# 3 M rows, 8 keys used of every 32 (TPC-H order keys), int4 payload: the chain statistics the fill reports
n = 3_000_000
i = np.arange(n, dtype=np.int64)
keys = (i // 8) * 32 + (i % 8) + 1
pay = np.random.default_rng(20261015).integers(-2**31, 2**31, n).astype(np.int32)
t = ctx.table_from([g.GX_INT8, g.GX_INT4], [keys, pay])
ht = ctx.hash_build(t, 0, [1], unique=True)
bunched = {"avg_chain": ht.info()["avg_chain"], "slot_mode": ht.info()["slot_mode"], "nentries": ht.nentries}
ht.free(); t.free()
print(json.dumps({"sf100_info": info, "sf100_nentries": nent,
                  "sf100_ms": {k: (v[0] / reps, v[1] / reps) for k, v in ph.items()}, "bunched_3m": bunched}))
"""


def last_json(text):
    for line in reversed(text.splitlines()):
        line = line.strip()
        if line.startswith("{"):
            return json.loads(line)
    raise RuntimeError("no JSON line in output:\n" + text[-3000:])


def run(cmd, cwd):
    p = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"{cmd} in {cwd} exited {p.returncode}:\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
    return p.stdout, p.stderr


def copy_rate():
    """A device-to-device copy of the build's traffic (3.95 GB: 1.975 GB read, 1.975 GB written): the streaming rate
    this card reaches for a 1:1 read/write mix."""
    import torch
    n = 1_975_000_000 // 8
    a = torch.ones(n, dtype=torch.int64, device="cuda")
    b = torch.empty_like(a)
    for _ in range(3):
        b.copy_(a)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        b.copy_(a)
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / reps
    del a, b
    torch.cuda.empty_cache()
    return {"bytes": 2 * n * 8, "ms": ms, "tb_per_s": 2 * n * 8 / (ms / 1e3) / 1e12}


def card():
    q = "name,power.limit,clocks.max.sm,clocks.max.mem"
    p = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return p.stdout.strip().splitlines()[0] if p.returncode == 0 and p.stdout.strip() else "unknown"


def compare(dir_a, dir_b):
    ka, kb = np.load(os.path.join(dir_a, "keys.npy")), np.load(os.path.join(dir_b, "keys.npy"))
    aa, ab = np.load(os.path.join(dir_a, "aggs.npy")), np.load(os.path.join(dir_b, "aggs.npy"))
    same_keys = ka.shape == kb.shape and bool(np.array_equal(ka, kb))
    same_count = aa.shape == ab.shape and bool(np.array_equal(aa[:, 0], ab[:, 0]))
    rel = float(np.max(np.abs(aa[:, 1:] - ab[:, 1:]) / np.maximum(np.abs(aa[:, 1:]), 1e-300))) if same_keys and aa.shape[1] > 1 else None
    return {"keys_identical": same_keys, "count_identical": same_count, "max_rel_sum_diff": rel}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old", required=True)
    ap.add_argument("--new", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    out = os.path.abspath(args.out)
    os.makedirs(out, exist_ok=True)
    trees = {"old": os.path.abspath(args.old), "new": os.path.abspath(args.new)}
    res = {"card": card(), "copy": copy_rate(), "probe": {}, "bench": [], "outputs": {}}
    print("card:", res["card"], "| copy:", res["copy"], flush=True)
    for name, tree in trees.items():
        so, se = run([sys.executable, "-c", PROBE], tree)
        res["probe"][name] = last_json(so)
        res["probe"][name]["stderr"] = se[-2000:]
        print(name, "probe:", json.dumps(res["probe"][name]), flush=True)
    for rnd in range(args.rounds):
        for name, tree in trees.items():
            dump = os.path.join(out, f"dump_{name}{rnd}")
            so, se = run([sys.executable, "bench.py", "--gpus", "1", "--steps", str(args.steps), "--no-unclustered",
                          "--dump-outputs", dump], tree)
            r = last_json(so)
            row = {"tree": name, "round": rnd, "ms_per_step": r.get("ms_per_step"), "clocks": r.get("clocks"),
                   "build_ms": r.get("phases_ms", {}).get("build", {}).get("ms_per_step"),
                   "probe_agg_ms": r.get("phases_ms", {}).get("probe_agg", {}).get("ms_per_step"),
                   "checks_all_true": all(v is not False for v in r.get("checks", {}).values()),
                   "failed_checks": [k for k, v in r.get("checks", {}).items() if v is False]}
            res["bench"].append(row)
            print(json.dumps(row), flush=True)
    ref = os.path.join(out, "dump_old0")
    for rnd in range(args.rounds):
        for name in trees:
            if (name, rnd) != ("old", 0):
                res["outputs"][f"{name}{rnd}_vs_old0"] = compare(ref, os.path.join(out, f"dump_{name}{rnd}"))
    for name in trees:
        ms = [b["ms_per_step"] for b in res["bench"] if b["tree"] == name]
        bl = [b["build_ms"] for b in res["bench"] if b["tree"] == name]
        pa = [b["probe_agg_ms"] for b in res["bench"] if b["tree"] == name]
        res[f"summary_{name}"] = {"ms_per_step": ms, "build_ms": bl, "probe_agg_ms": pa}
    with open(os.path.join(out, "ab.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in res if k.startswith("summary") or k == "outputs"}, indent=1))


if __name__ == "__main__":
    main()
