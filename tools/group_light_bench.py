"""Times light propagation on device groups against one context, on the C4 shape (bench.py --workload c4): the N^3
Space of scenes.config_c4, converged (fast_evaluate_light + evaluate_light(1)), then K steps of scenes.c4_edits (10 000
random edits each) propagated to epsilon 1.  Every arm holds its own copy of the Space and takes the same edits; the
arms alternate step by step.  Prints one JSON line per arm: cube updates per device second, rounds and device time per
step, the initial convergence, how far its final field is from the single context's, and the GPU's name and power
limit read in the same run.

    python tools/group_light_bench.py --devices 0 0,0 --steps 5 --warmup 2
    python tools/group_light_bench.py --devices 0,1,2,3,4,5,6,7 --n 256
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
import aicb200  # noqa: E402
import bench  # noqa: E402  (the clock sampler)
from aicb200 import scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

EDITS = 10000


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--devices", nargs="+", default=["0"],
                   help="one group per argument: its device ids, comma separated (may repeat)")
    p.add_argument("--n", type=int, default=256, help="edge of the Space")
    p.add_argument("--steps", type=int, default=5)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--no-single", action="store_true", help="leave out the single-context arm")
    args = p.parse_args()
    if args.steps < 1 or args.n < 8:
        p.error("--steps must be >= 1 and --n >= 8")
    space = scenes.config_c4(args.n)

    arms = {}   # name -> (the scene's light calls, what to close)
    if not args.no_single:
        rt = aicb200.SpaceRaytracer(space, aicb200.GraphicsOptions())
        arms["single"] = (rt, [rt])
    for d in args.devices:
        g = aicb200.DeviceGroup([int(v) for v in d.split(",")])
        arms[f"group[{d}]"] = (g.add_scene(space), [g])

    conv = {}
    for name, (s, _) in arms.items():
        t0 = time.perf_counter()
        s.light_fast_evaluate()
        upd, md, nv = s.light_evaluate(1)
        st = s.light_stats()
        conv[name] = {"cube_updates": upd, "wall_seconds": time.perf_counter() - t0, "rounds": st["rounds"],
                      "device_seconds": st["device_seconds"],
                      "cube_updates_per_s": upd / max(st["device_seconds"], 1e-9)}
    runs = {name: [] for name in arms}
    sampler = bench.ClockSampler(0)
    for k in range(args.warmup + args.steps):
        if k == args.warmup:
            sampler.start()
            sampler.mark()
        cubes, ids = scenes.c4_edits(space, EDITS, k)
        for name, (s, _) in arms.items():
            t0 = time.perf_counter()
            upd, md = s.light_edit_and_propagate(cubes, ids, 1)
            wall = time.perf_counter() - t0
            st = s.light_stats()
            if k >= args.warmup:
                runs[name].append((upd, st["rounds"], st["device_seconds"], wall))
    clocks = sampler.stop()
    single = arms["single"][0].light_download() if "single" in arms else None
    gpu = gpu_identity()
    for name, (s, owners) in arms.items():
        r = np.array(runs[name], dtype=np.float64)
        line = {
            "arm": name, "workload": f"C4: {args.n}^3 res-1 Space, LightPhysics::Rays{{30}}, octant sky; converge, then "
                                     f"{EDITS} random edits per step, propagated to epsilon 1",
            "steps": args.steps, "warmup": args.warmup,
            "cube_updates_per_s": float(r[:, 0].sum() / r[:, 2].sum()),
            "cube_updates_per_step": float(r[:, 0].mean()), "rounds_per_step": float(r[:, 1].mean()),
            "device_ms_per_step": float(1e3 * r[:, 2].mean()), "device_ms_min_max": [float(1e3 * r[:, 2].min()), float(1e3 * r[:, 2].max())],
            "wall_ms_per_step": float(1e3 * r[:, 3].mean()),
            "initial_convergence": conv[name], "gpu": gpu, "clocks": clocks,
        }
        if single is not None and name != "single":
            f = s.light_download()
            d = np.abs(f[..., :3].astype(int) - single[..., :3].astype(int)).max(axis=-1)
            line["vs_single"] = {"statuses_equal": bool(np.array_equal(f[..., 3], single[..., 3])),
                                 "max_units": int(d.max()), "frac_cubes_differ": float((d > 0).mean())}
        print(json.dumps(line), flush=True)
    for name, (s, owners) in arms.items():
        for o in owners:
            o.close()


if __name__ == "__main__":
    main()
