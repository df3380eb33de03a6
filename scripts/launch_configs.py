"""Lists every kernel launch of the aggregate-family GPU tests -- kernel name, grid, block and shared memory -- as
torch.profiler (CUDA activities) records them, so that two builds can be compared launch for launch:

    python scripts/launch_configs.py --tree OLD --out old.json
    python scripts/launch_configs.py --tree .   --out new.json
    python scripts/launch_configs.py --compare old.json new.json

The tests are seeded, so two builds that launch alike give the same multiset of launches.  Each --tree runs in a
process of its own and imports the package of that tree."""
import argparse
import collections
import json
import os
import sys
import tempfile

MODULES = ["tests/test_gpu_fp_edges.py", "tests/test_gpu_quals_exprs.py", "tests/test_gpu_join_edges.py",
           "tests/test_gpu_runjoin_seg.py", "tests/test_gpu_narrow_slots.py"]


def record(tree, out, extra):
    tree = os.path.abspath(tree)
    os.chdir(tree)
    sys.path.insert(0, tree)
    import pytest
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rc = pytest.main(["-q", "-m", "gpu", "-p", "no:cacheprovider", *extra, *MODULES])
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    launches = collections.Counter()
    for e in events:
        if e.get("cat") != "kernel":
            continue
        a = e.get("args", {})
        launches[json.dumps([e["name"], a.get("grid"), a.get("block"), a.get("shared memory")])] += 1
    with open(out, "w") as f:
        json.dump({"pytest_exit": int(rc), "device": torch.cuda.get_device_name(0), "launches": dict(sorted(launches.items()))}, f, indent=0)
    print(f"{tree}: pytest exit {int(rc)}, {sum(launches.values())} launches, {len(launches)} distinct configurations")


def compare(a_path, b_path):
    a, b = (json.load(open(p))["launches"] for p in (a_path, b_path))
    diff = sorted(set(a) | set(b), key=lambda k: (k not in a, k))
    bad = [(k, a.get(k, 0), b.get(k, 0)) for k in diff if a.get(k, 0) != b.get(k, 0)]
    print(f"{len(a)} / {len(b)} distinct configurations, {sum(a.values())} / {sum(b.values())} launches")
    for k, x, y in bad:
        print(f"  {x:6d} {y:6d}  {k}")
    print("identical" if not bad else f"{len(bad)} configurations differ")
    return 0 if not bad else 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=".")
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    ap.add_argument("pytest_args", nargs="*", help="extra pytest arguments (after --), e.g. -k probe_agg")
    a = ap.parse_args()
    if a.compare:
        sys.exit(compare(*a.compare))
    record(a.tree, os.path.abspath(a.out), a.pytest_args)


if __name__ == "__main__":
    main()
