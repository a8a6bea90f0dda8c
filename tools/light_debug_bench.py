"""What a host pays for compute_light's rays: light_compute_debug (Space::compute_light::<LightUpdateCubeInfo>) against
light_compute on the same cubes, for one cube (GraphicsOptions::debug_light_rays_at_cursor asks for one per frame) and
for 4096 cubes, on the C4 shape (bench.py --workload c4): the N^3 Space of scenes.config_c4, converged
(fast_evaluate_light + evaluate_light(1)).  The cubes are the air cubes just above the ground, where rays end on many
faces.  Each call is timed on the host (every light call returns after its device work); the median of --reps calls
after --warmup calls is printed as one JSON line per case, then the GPU's name and power limit, read in the same run.

    python tools/light_debug_bench.py --n 256 --reps 20
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
import aicb200  # noqa: E402
from aicb200 import scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

EPSILON = 1


def median_ms(call, warmup, reps):
    for _ in range(warmup):
        call()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()
        times.append(1e3 * (time.perf_counter() - t0))
    return statistics.median(times)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=256, help="edge of the Space")
    p.add_argument("--reps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    args = p.parse_args()
    if args.n < 32:
        p.error("--n must be >= 32")
    space = scenes.config_c4(args.n)
    rt = aicb200.SpaceRaytracer(space, aicb200.GraphicsOptions())
    rt.light_fast_evaluate()
    rt.light_evaluate(EPSILON)
    n = args.n
    y = n // 4   # the first layer above the ground slab
    xz = [(x, z) for x in range(n) for z in range(n) if space.block_ids[x, y, z] == 0]
    pick = np.random.default_rng(0).permutation(len(xz))[:4096]
    cubes = np.array([(space.lower[0] + xz[k][0], space.lower[1] + y, space.lower[2] + xz[k][1]) for k in pick],
                     dtype=np.int32)
    for count in (1, len(cubes)):
        c = cubes[:count]
        texels, rays = rt.light_compute_debug(c)
        assert np.array_equal(texels, rt.light_compute(c))
        plain = median_ms(lambda: rt.light_compute(c), args.warmup, args.reps)
        debug = median_ms(lambda: rt.light_compute_debug(c), args.warmup, args.reps)
        print(json.dumps({"cubes": count, "rays": int(sum(r.size for r in rays)), "light_compute_ms": plain,
                          "light_compute_debug_ms": debug}), flush=True)
    print(json.dumps({"workload": f"C4: {n}^3 res-1 Space, LightPhysics::Rays{{30}}, octant sky, converged to "
                                  f"epsilon {EPSILON}", "gpu": gpu_identity()}), flush=True)
    rt.close()


if __name__ == "__main__":
    main()
