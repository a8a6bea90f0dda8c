"""What a block redefinition costs the light (SpaceRaytracer.light_relight_blocks), next to the full re-convergence it
replaces, on the C4 shape (bench.py --workload c4): the N^3 Space of scenes.config_c4 with two changes, so that one
block is rare and one is common:
  - "rare": a new grey block placed in about 100 air cubes above the ground;
  - "common": the ground cubes of blocks 1..7 all hold block 1 (about 12 % of the volume).
The Space is converged (fast_evaluate_light + evaluate_light(1)), timed as the full re-convergence.  Then each block is
redefined --reps times in turn (the rare one lit as a lamp and dark again, the common one in one face colour and the
other), each time update_blocks + light_relight_blocks(epsilon 1).  For each relight it prints one JSON line: the
host time of the call, its cube updates and the propagation's device time (light_stats), and, once per block, the
device time of the scan kernel (k_relight_blocks) from torch.profiler in a call of its own; then the GPU's name and
power limit, read in the same run.

    python tools/light_relight_bench.py --n 256 --reps 3
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
from aicb200 import Block, Space, scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

EPSILON = 1
RARE_CUBES = 100


def bench_space(n):
    base = scenes.config_c4(n)
    ids = base.block_ids.copy()
    ground = ids[:, : n // 4, :]
    ground[(ground >= 1) & (ground <= 7)] = 1
    rare = len(base.blocks)
    rng = np.random.default_rng(12)
    placed = 0
    while placed < RARE_CUBES:
        c = (int(rng.integers(0, n)), int(rng.integers(n // 4 + 2, n)), int(rng.integers(0, n)))
        if ids[c] == 0:
            ids[c] = rare
            placed += 1
    blocks = base.blocks + [Block(color=(0.6, 0.6, 0.6, 1.0))]
    space = Space(base.lower, ids, blocks, light=base.light, sky_colors=base.sky_colors,
                  light_max_distance=base.light_max_distance)
    return space, rare


def scan_ms(call):
    """Device time of k_relight_blocks during call(), from torch.profiler (CUDA activities), in milliseconds."""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        total = 0.0
        for e in prof.events():
            if "k_relight_blocks" in e.name:
                total += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        return total * 1e-3
    except Exception as e:   # the profiler is an aid to this tool, not a requirement of the library
        return f"not measured: {type(e).__name__}: {e}"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=256, help="edge of the Space")
    p.add_argument("--reps", type=int, default=3, help="redefinitions of each block, alternating its two definitions")
    args = p.parse_args()
    if args.n < 32:
        p.error("--n must be >= 32")
    space, rare = bench_space(args.n)
    volume = args.n ** 3
    rt = aicb200.SpaceRaytracer(space, aicb200.GraphicsOptions())
    t0 = time.perf_counter()
    rt.light_fast_evaluate()
    updates, _, _ = rt.light_evaluate(EPSILON)
    t1 = time.perf_counter()
    st = rt.light_stats()
    print(json.dumps({"case": "full re-convergence (fast_evaluate_light + evaluate_light(1))", "host_ms": 1e3 * (t1 - t0),
                      "cube_updates": updates, "propagation_device_ms": 1e3 * st["device_seconds"]}), flush=True)
    cases = {
        "rare": (rare, [Block(color=(0.6, 0.6, 0.6, 1.0), emission=(4.0, 3.5, 2.0)), Block(color=(0.6, 0.6, 0.6, 1.0))]),
        "common": (1, [Block(color=(0.8, 0.3, 0.2, 1.0)), Block(color=tuple(space.blocks[1].palette[0, :4]))]),
    }
    for name, (index, definitions) in cases.items():
        held = int((space.block_ids == index).sum())
        for k in range(2 * args.reps):
            rt.update_blocks([index], [definitions[k % 2]])
            t0 = time.perf_counter()
            upd, md = rt.light_relight_blocks([index], EPSILON)
            t1 = time.perf_counter()
            st = rt.light_stats()
            print(json.dumps({"case": name, "block": index, "cubes_holding": held, "fraction": held / volume,
                              "definition": k % 2, "host_ms": 1e3 * (t1 - t0), "cube_updates": upd, "max_diff": md,
                              "propagation_device_ms": 1e3 * st["device_seconds"]}), flush=True)
        rt.update_blocks([index], [definitions[0]])
        ms = scan_ms(lambda: rt.light_relight_blocks([index], EPSILON))
        print(json.dumps({"case": name, "block": index, "scan_kernel_ms": ms}), flush=True)
        rt.update_blocks([index], [definitions[1]])
        rt.light_relight_blocks([index], EPSILON)
    print(json.dumps({"workload": f"C4: {args.n}^3 res-1 Space, LightPhysics::Rays{{30}}, octant sky, converged to "
                                  f"epsilon {EPSILON}", "gpu": gpu_identity()}), flush=True)


if __name__ == "__main__":
    main()
