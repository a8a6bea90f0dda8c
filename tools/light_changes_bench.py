"""What following GPU light costs a host: the set of changed cubes against a whole-volume download, on the C4 shape
(bench.py --workload c4): the N^3 Space of scenes.config_c4, converged (fast_evaluate_light + evaluate_light(1)), then
  (a) one emissive block placed in the air above the ground, propagated to epsilon 1, at --lamps places in turn;
  (b) steps of scenes.c4_edits (10 000 random edits each), propagated to epsilon 1.
For each propagation it prints one JSON line: the propagation's device time and cube updates, the size of the set of
changed cubes, the host time of light_changes_count + light_take_changes, and the host time of a whole-volume
light_download right after it; then the GPU's name and power limit, read in the same run.

    python tools/light_changes_bench.py --n 256 --lamps 3 --steps 3
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
from aicb200 import scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

EDITS = 10000
EPSILON = 1


def measure(rt, case, updates, volume):
    st = rt.light_stats()
    t0 = time.perf_counter()
    n = rt.light_changes_count()
    t1 = time.perf_counter()
    idx, tx = rt.light_take_changes()
    t2 = time.perf_counter()
    rt.light_download()
    t3 = time.perf_counter()
    assert len(idx) == n
    return {"case": case, "cube_updates": updates, "propagation_device_ms": 1e3 * st["device_seconds"],
            "changed_cubes": n, "changed_fraction": n / volume, "take_bytes": 8 * n,
            "count_ms": 1e3 * (t1 - t0), "take_ms": 1e3 * (t2 - t1), "count_plus_take_ms": 1e3 * (t2 - t0),
            "download_ms": 1e3 * (t3 - t2), "download_bytes": 4 * volume}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=256, help="edge of the Space")
    p.add_argument("--lamps", type=int, default=3, help="single emissive blocks placed, one propagation each")
    p.add_argument("--steps", type=int, default=3, help="steps of 10 000 random edits")
    args = p.parse_args()
    if args.n < 32:
        p.error("--n must be >= 32")
    space = scenes.config_c4(args.n)
    volume = args.n ** 3
    rt = aicb200.SpaceRaytracer(space, aicb200.GraphicsOptions())
    rt.light_fast_evaluate()
    rt.light_evaluate(EPSILON)
    # warm the take and download paths, and start from an empty set
    rt.light_take_changes()
    rt.light_download()
    rt.light_take_changes(discard=True)
    emitter = len(space.blocks) - 1
    assert any(v != 0.0 for v in space.blocks[emitter].light_emission)
    ids = space.block_ids.copy()
    n, placed = args.n, 0
    for k in range(args.n * args.n):
        if placed == args.lamps:
            break
        cube = (n // 2 + 37 * k % (n // 2) - n // 4, n // 4 + 6 + (11 * k) % (n // 2), n // 2 + (53 * k) % (n // 2) - n // 4)
        if ids[cube] != 0:
            continue
        ids[cube] = emitter
        upd, _ = rt.light_edit_and_propagate([cube], [emitter], EPSILON)
        print(json.dumps(measure(rt, f"one emissive block at {list(cube)}", upd, volume)), flush=True)
        placed += 1
    for k in range(args.steps):
        cubes, new_ids = scenes.c4_edits(space, EDITS, k)
        upd, _ = rt.light_edit_and_propagate(cubes, new_ids, EPSILON)
        print(json.dumps(measure(rt, f"scenes.c4_edits step {k} ({EDITS} edits)", upd, volume)), flush=True)
    print(json.dumps({"workload": f"C4: {args.n}^3 res-1 Space, LightPhysics::Rays{{30}}, octant sky, converged to "
                                  f"epsilon {EPSILON}", "gpu": gpu_identity()}), flush=True)
    rt.close()


if __name__ == "__main__":
    main()
