"""Times aicb_render_layers_texture — RaytraceToTexture's colour and depth texels (raytrace_to_texture.rs:591-683) — on
one of bench.py's raytracing workloads: world layer only, no backdrop, NO_WORLD_TO_SHOW paint, one batch of N pixels
in PixelPicker order per step (N = 0: the whole texture).  Prints one JSON line with Mrays/s over the device time, the
median device and wall time per batch, and the GPU's name and power limit read in the same run.

    python tools/texture_bench.py --workload c2 --pixels 60000 --steps 30 --warmup 3
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
import aicb200  # noqa: E402
import bench  # noqa: E402  (the workload definitions and the clock sampler)
from aicb200 import scenes  # noqa: E402


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=10)
        name, power = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit_w": float(power)}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return {"name": None, "power_limit_w": None}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--workload", default="c2", choices=["c0", "c1", "c2", "c3"])
    p.add_argument("--pixels", type=int, default=0, help="pixels per batch in PixelPicker order (0 = the whole texture)")
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=3)
    args = p.parse_args()
    if args.pixels < 0 or args.steps < 1:
        p.error("--pixels must be >= 0 and --steps >= 1")
    space, opts, w, h, desc = bench.make_workload(args.workload)
    cam = scenes.standard_camera(space, opts, w, h)
    rt = aicb200.SpaceRaytracer(space, opts)
    m = cam.depth_transform()
    n = args.pixels
    pixels = aicb200.pixel_picker_order(w, h, n) if n else None
    no_world = aicb200.srgb8_to_linear((0xBC, 0xBC, 0xBC)) + (1.0,)
    layer = (rt, cam, opts)
    for _ in range(max(1, args.warmup)):
        aicb200.render_layers_texture(layer, None, None, no_world, m, pixels)
    sampler = bench.ClockSampler(0)
    sampler.start()
    sampler.mark()
    dev_ms, wall_ms, rays = [], [], 0
    for _ in range(args.steps):
        t0 = time.perf_counter()
        _, _, info = aicb200.render_layers_texture(layer, None, None, no_world, m, pixels)
        wall_ms.append(1e3 * (time.perf_counter() - t0))
        dev_ms.append(info.kernel_ms)
        rays += info.rays
    clocks = sampler.stop()
    print(json.dumps({
        "metric": "Mrays/s", "value": rays / (sum(dev_ms) / 1e3) / 1e6, "unit": "Mrays/s", "steps": args.steps,
        "pixels_per_batch": n if n else w * h,
        "pixels": f"{n} in PixelPicker order" if n else "the whole texture, row-major",
        "batch_device_ms": float(np.median(dev_ms)), "batch_wall_ms": float(np.median(wall_ms)),
        "workload": desc, "layers": "world only, no backdrop, NO_WORLD_TO_SHOW",
        "gpu": gpu_identity(), "clocks": clocks,
    }))


if __name__ == "__main__":
    main()
