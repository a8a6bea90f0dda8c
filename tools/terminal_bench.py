"""Times aicb_render_layers_terminal — the desktop terminal's frame (all-is-cubes-desktop/src/terminal.rs:114-142) —
against aicb_render_layers_srgb8 on the same layers: one of bench.py's raytracing workloads as the world layer, a small
UI Space in front of it and NO_WORLD_TO_SHOW paint, at each framebuffer size given.  The default sizes are a terminal's
framebuffer (240x134: a 240x67-character terminal in Split mode, two pixels per character cell, nominal 120x67, whose
aspect ratio it shares) and 1920x1080.  The two calls alternate step by step.  Prints one JSON line per size and call
with Mrays/s over the device time, the median device time (its passes summed) and wall time per frame, and the GPU's
name and power limit read in the same run.

    python tools/terminal_bench.py --workload c2 --sizes 240x134,1920x1080 --steps 30 --warmup 3
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
import bench  # noqa: E402  (the workload definitions and the clock sampler)
from aicb200 import FOG_NONE, LIGHT_FLAT, GraphicsOptions, scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--workload", default="c2", choices=["c0", "c1", "c2", "c3"])
    p.add_argument("--sizes", default="240x134,1920x1080", help="framebuffer sizes WxH, comma separated")
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=3)
    args = p.parse_args()
    if args.steps < 1:
        p.error("--steps must be >= 1")
    sizes = [tuple(int(v) for v in s.split("x")) for s in args.sizes.split(",")]
    space, wopts, _, _, desc = bench.make_workload(args.workload)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT)
    no_world = aicb200.srgb8_to_linear((0xBC, 0xBC, 0xBC)) + (1.0,)
    wrt = aicb200.SpaceRaytracer(space, wopts)
    urt = aicb200.SpaceRaytracer(ui_space, uopts, wrt.ctx)
    gpu = gpu_identity()
    for w, h in sizes:
        wcam = scenes.standard_camera(space, wopts, w, h)
        ucam = scenes.standard_camera(ui_space, uopts, w, h, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
        lw, lu = (wrt, wcam, wopts), (urt, ucam, uopts)
        calls = {"terminal": lambda: aicb200.render_layers_terminal(lw, lu, None, no_world)["info"],
                 "srgb8": lambda: aicb200.render_layers(lw, lu, None, no_world).info}
        for _ in range(max(1, args.warmup)):
            for fn in calls.values():
                fn()
        times = {k: ([], [], []) for k in calls}
        sampler = bench.ClockSampler(0)
        sampler.start()
        sampler.mark()
        for _ in range(args.steps):
            for name, fn in calls.items():
                t0 = time.perf_counter()
                info = fn()
                times[name][1].append(1e3 * (time.perf_counter() - t0))
                times[name][0].append(info.kernel_ms)
                times[name][2].append(info.rays)
        clocks = sampler.stop()
        for name, (dev_ms, wall_ms, rays) in times.items():
            print(json.dumps({
                "call": name, "frame": f"{w}x{h}", "workload": desc,
                "layers": "world + 6^3 UI Space, NO_WORLD_TO_SHOW", "steps": args.steps,
                "metric": "Mrays/s", "value": sum(rays) / (sum(dev_ms) / 1e3) / 1e6, "unit": "Mrays/s",
                "frame_device_ms": float(np.median(dev_ms)), "frame_wall_ms": float(np.median(wall_ms)),
                "gpu": gpu, "clocks": clocks,
            }))


if __name__ == "__main__":
    main()
