"""What a tick's light step costs on the GPU (aicb_light_update_from_queue), on the C4 shape (bench.py --workload c4): the
N^3 Space of scenes.config_c4 converged to epsilon 1 (fast_evaluate_light + evaluate_light(1)), then a 32^3 box in the
middle of the ground filled with random blocks by aicb_light_edit_region, which queues it.  Every case starts from a new
scene holding the converged Space with the same fill.
  (a) per budget (10^3 .. 10^6, and none): --calls steps in a row, as a game loop would make them, each timed on the
      host (the call returns with its work done) with its device time (aicb_light_stats out[3]) and cube updates;
      medians over the calls.
  (b) an unbounded step against aicb_light_evaluate(0) on identical scenes, alternating, --runs runs each: the
      difference is the cost of the budgeted gather.
Prints one JSON line per measurement, then the GPU's name and power limit, read in the same run.

    python tools/light_step_bench.py --n 256
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from aicb200 import GraphicsOptions, Space, SpaceRaytracer, scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

EPSILON = 1
BOX = 32


def converged(n):
    space = scenes.config_c4(n)
    rt = SpaceRaytracer(space, GraphicsOptions())
    rt.light_fast_evaluate()
    rt.light_evaluate(EPSILON)
    field = rt.light_download()
    rt.close()
    return Space(space.lower, space.block_ids, space.blocks, light=field, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


def edited(space):
    """A new scene with the converged light and the box filled (queued, not propagated)."""
    rt = SpaceRaytracer(space, GraphicsOptions())
    n = space.size[0]
    lower = [space.lower[0] + (n - BOX) // 2, space.lower[1] + n // 4 - BOX // 2, space.lower[2] + (n - BOX) // 2]
    ids = np.random.default_rng(5).integers(0, len(space.blocks), (BOX,) * 3).astype(np.uint16)
    changed = rt.light_edit_region(lower, (BOX,) * 3, ids)
    return rt, changed


def timed(call):
    t0 = time.perf_counter()
    out = call()
    return out, 1e3 * (time.perf_counter() - t0)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=256, help="edge of the Space")
    p.add_argument("--calls", type=int, default=10, help="steps in a row per budget")
    p.add_argument("--runs", type=int, default=3, help="runs of each arm of (b)")
    args = p.parse_args()
    if args.n < 64:
        p.error("--n must be >= 64")
    space = converged(args.n)
    rt, changed = edited(space)   # warm-up: module load and first launches
    rt.light_update_from_queue(1000)
    rt.close()
    print(json.dumps({"box": BOX, "cubes_changed": changed}), flush=True)
    for budget in (10**3, 10**4, 10**5, 10**6, None):
        rt, _ = edited(space)
        host, device, updates = [], [], []
        for _ in range(args.calls if budget is not None else 1):
            info, ms = timed(lambda: rt.light_update_from_queue(budget))
            host.append(ms)
            device.append(rt.light_stats()["device_seconds"] * 1e6)
            updates.append(info["update_count"])
            if info["queue_count"] == 0:
                break
        rt.close()
        print(json.dumps({"budget": budget, "calls": len(host), "host_ms_median": statistics.median(host),
                          "device_us_median": statistics.median(device), "updates_per_call": statistics.median(updates),
                          "host_ms": [round(v, 3) for v in host],
                          "mupdates_per_s": sum(updates) / (sum(host) * 1e3)}), flush=True)
    for run in range(args.runs):
        for arm in ("step", "evaluate") if run % 2 == 0 else ("evaluate", "step"):
            rt, _ = edited(space)
            if arm == "step":
                info, ms = timed(lambda: rt.light_update_from_queue())
                n = info["update_count"]
            else:
                (n, _, _), ms = timed(lambda: rt.light_evaluate(0))
            stats = rt.light_stats()
            rt.close()
            print(json.dumps({"run": run, "arm": arm, "updates": n, "host_ms": ms, "rounds": stats["rounds"],
                              "device_us": stats["device_seconds"] * 1e6}), flush=True)
    print(json.dumps({"workload": f"C4: {args.n}^3 res-1 Space, LightPhysics::Rays{{30}}, octant sky, converged to "
                                  f"epsilon {EPSILON}, a {BOX}^3 box filled with random blocks", "gpu": gpu_identity()}),
          flush=True)


if __name__ == "__main__":
    main()
