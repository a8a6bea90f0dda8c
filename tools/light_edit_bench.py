"""What a tick's scattered Mutation::set batch costs on the GPU, on C4's lit Space converged to epsilon 1.  Lists of
10 .. 10^6 edits from scenes.c4_edits, each list taken by every arm in alternating order:
  - light_edit_cubes: the list in one call (no propagation);
  - light_edit_region x n: the same cubes as 1x1x1 boxes, one call each (lists of at most --region-max edits);
  - light_edit_and_propagate(1): its edit part is the call's host time minus the propagation's device time
    (aicb_light_stats), as tools/region_fill_bench.py computes it.  This arm alone runs against an older build of the
    library too (--arms propagate), which is how the edit part of two builds is compared.
Every call returns synchronised, so the host clock around it is its time; no profiler runs meanwhile.  An arm that does
not propagate is followed by an untimed light_evaluate(1), so every list starts from a converged field.  A separate pass
under torch.profiler then gives the device time of the edit kernels.  Prints one JSON line per measurement, then
medians with ranges and the GPU's name and power limit, read in the same run.

    python tools/light_edit_bench.py --reps 5
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from aicb200 import GraphicsOptions, SpaceRaytracer, scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

KERNELS = ("k_edit_cells", "k_edit_light", "k_edits")
ARMS = ("cubes", "region", "propagate")


def ms_since(t0):
    return 1e3 * (time.perf_counter() - t0)


def arm_call(rt, arm, cubes, ids):
    """One list through `arm`: the measurement's fields."""
    if arm == "cubes":
        t0 = time.perf_counter()
        changed = rt.light_edit_cubes(cubes, ids)
        out = {"edit_ms": ms_since(t0), "changed": changed}
    elif arm == "region":
        t0 = time.perf_counter()
        changed = sum(rt.light_edit_region(c, (1, 1, 1), int(i)) for c, i in zip(cubes, ids))
        out = {"edit_ms": ms_since(t0), "changed": changed}
    else:
        t0 = time.perf_counter()
        updates = rt.light_edit_and_propagate(cubes, ids, 1)[0]
        total = ms_since(t0)
        device = 1e3 * rt.light_stats()["device_seconds"]
        return {"edit_ms": total - device, "total_ms": total, "propagate_device_ms": device, "cube_updates": updates}
    t1 = time.perf_counter()
    out["cube_updates"] = rt.light_evaluate(1)[0]
    out["propagate_ms"] = ms_since(t1)
    return out


def timed(rt, space, arms, sizes, reps, region_max):
    rows, batch = [], 0
    for n in sizes:
        mine = [a for a in arms if a != "region" or n <= region_max]
        for k in range(reps):
            order = mine if k % 2 == 0 else mine[::-1]
            for arm in order:
                batch += 1
                cubes, ids = scenes.c4_edits(space, n, batch)
                rows.append(dict(arm_call(rt, arm, cubes, ids), arm=arm, n=n, rep=k))
                print(json.dumps(rows[-1]), flush=True)
    return rows


def profiled(rt, space, arms, sizes):
    """One list of each size per arm under torch.profiler: the device time of the edit kernels."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    rows = []
    for n in sizes:
        for k, arm in enumerate(a for a in arms if a != "region"):
            cubes, ids = scenes.c4_edits(space, n, 10**7 + 10 * n + k)   # a list no arm has applied yet
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                arm_call(rt, arm, cubes, ids)
                torch.cuda.synchronize()
            us = {k: sum(e.time_range.elapsed_us() for e in prof.events() if k in e.name) for k in KERNELS}
            rows.append({"profiled": arm, "n": n, "kernel_us": {k: v for k, v in us.items() if v}})
            print(json.dumps(rows[-1]), flush=True)
    return rows


def spread(values):
    return {"median": float(np.median(values)), "min": float(np.min(values)), "max": float(np.max(values))}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=5, help="lists per size and arm")
    p.add_argument("--n", type=int, default=256, help="edge of the Space")
    p.add_argument("--sizes", type=int, nargs="+", default=[10, 100, 1000, 10000, 100000, 1000000])
    p.add_argument("--region-max", type=int, default=1000, help="longest list the 1x1x1 box arm takes")
    p.add_argument("--arms", nargs="+", default=list(ARMS), choices=ARMS)
    p.add_argument("--no-profile", action="store_true")
    args = p.parse_args()
    space = scenes.config_c4(n=args.n)
    rt = SpaceRaytracer(space, GraphicsOptions())
    rt.light_fast_evaluate()
    t0 = time.perf_counter()
    rt.light_evaluate(1)
    print(json.dumps({"converge_ms": ms_since(t0), "cube_updates": rt.light_stats()["cube_updates"]}), flush=True)
    for arm in args.arms:   # warm every arm's kernels up
        cubes, ids = scenes.c4_edits(space, 10, 0)
        arm_call(rt, arm, cubes, ids)
    rows = timed(rt, space, args.arms, args.sizes, args.reps, args.region_max)
    kernels = [] if args.no_profile else profiled(rt, space, args.arms, args.sizes)
    summary = {}
    for n in args.sizes:
        out = {}
        for arm in args.arms:
            mine = [r for r in rows if r["arm"] == arm and r["n"] == n]
            if mine:
                out[arm] = {key: spread([r[key] for r in mine]) for key in mine[0] if key.endswith("_ms")}
        out["kernel_us"] = {r["profiled"]: r["kernel_us"] for r in kernels if r["n"] == n}
        summary[str(n)] = out
    print(json.dumps({"n": args.n, "reps": args.reps, "summary": summary, "gpu": gpu_identity()}), flush=True)
    rt.close()


if __name__ == "__main__":
    main()
