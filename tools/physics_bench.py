"""What SpaceChange::Physics costs (SpaceRaytracer.set_physics), next to what following it cost before: a new scene
and its light from nothing.  On the C4 shape as tools/light_relight_bench.py builds it (the N^3 Space of
scenes.config_c4, LightPhysics::Rays{30}, octant sky), with its light state in place (fast_evaluate_light).  Each of
--reps repetitions times, on the host (every call returns once its device work is done):
  - "sky": a new sky alone (octants <-> uniform, same distance);
  - "distance": a new maximum_distance (30 <-> 20): the light is reinitialised (fast_evaluate_light, every cube
    changed);
  - "rebuild": aicb_scene_create + aicb_light_fast_evaluate of the same Space with the new physics.
One JSON line per measurement, then the GPU's name and power limit, read in the same run.

    python tools/physics_bench.py --n 256 --reps 5
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
import aicb200  # noqa: E402
from aicb200 import Space, scenes  # noqa: E402
from light_relight_bench import bench_space  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

UNIFORM_SKY = [(0.4, 0.5, 0.9)]


def timed(call):
    t0 = time.perf_counter()
    call()
    return 1e3 * (time.perf_counter() - t0)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=256, help="edge of the Space")
    p.add_argument("--reps", type=int, default=5, help="repetitions of each change")
    args = p.parse_args()
    if args.n < 32:
        p.error("--n must be >= 32")
    space, _ = bench_space(args.n)
    skies = (space.sky_colors, UNIFORM_SKY)
    distances = (space.light_max_distance, 20)
    opts = aicb200.GraphicsOptions()
    rt = aicb200.SpaceRaytracer(space, opts)
    rt.light_fast_evaluate()
    rt.light_take_changes(discard=True)
    print(json.dumps({"case": "scene with light state", "device_bytes": rt.device_bytes}), flush=True)
    for k in range(args.reps):
        sky = skies[(k + 1) % 2]
        ms = timed(lambda: rt.set_physics(sky, distances[0]))
        print(json.dumps({"case": "sky", "rep": k, "sky": "uniform" if len(sky) == 1 else "octants", "host_ms": ms}),
              flush=True)
    rt.set_physics(skies[0], distances[0])
    for k in range(args.reps):
        d = distances[(k + 1) % 2]
        ms = timed(lambda: rt.set_physics(skies[0], d))
        changed = rt.light_changes_count()
        rt.light_take_changes(discard=True)
        print(json.dumps({"case": "distance", "rep": k, "light_max_distance": d, "host_ms": ms,
                          "cubes_changed": changed}), flush=True)
    rt.close()
    for k in range(args.reps):
        d = distances[(k + 1) % 2]
        other = Space(space.lower, space.block_ids, space.blocks, light=space.light, sky_colors=skies[0],
                      light_max_distance=d)
        holder = {}

        def rebuild():
            holder["rt"] = aicb200.SpaceRaytracer(other, opts)
            holder["rt"].light_fast_evaluate()

        ms = timed(rebuild)
        holder["rt"].close()
        print(json.dumps({"case": "rebuild", "rep": k, "light_max_distance": d, "host_ms": ms}), flush=True)
    print(json.dumps({"workload": f"C4: {args.n}^3 res-1 Space, octant sky, LightPhysics::Rays{{30}}",
                      "gpu": gpu_identity()}), flush=True)


if __name__ == "__main__":
    main()
