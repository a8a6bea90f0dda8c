"""Times a layered frame and a texture batch through a device group against the same calls on one context, on one of
bench.py's raytracing workloads: the workload's Space as the world layer, a small UI Space in front of it, a backdrop
and NO_WORLD_TO_SHOW paint.  Per step every arm draws the sRGB8 frame (aicb_render_layers_srgb8 /
aicb_group_render_layers_srgb8) and one batch of N pixels in PixelPicker order (aicb_render_layers_texture /
aicb_group_render_layers_texture); the arms alternate step by step.  Prints one JSON line per arm with the median device
time (the slowest device's, its passes summed) and the median wall time of each call, and the GPU's name and power
limit read in the same run.

    python tools/group_bench.py --workload c2 --pixels 60000 --devices 0 --steps 30 --warmup 3
    python tools/group_bench.py --arms single   # only the single-context calls
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
    p.add_argument("--pixels", type=int, default=60000, help="pixels of the texture batch, in PixelPicker order")
    p.add_argument("--devices", default="0", help="the group's device ids, comma separated (may repeat)")
    p.add_argument("--arms", default="single,group")
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=3)
    args = p.parse_args()
    if args.pixels < 1 or args.steps < 1:
        p.error("--pixels and --steps must be >= 1")
    arms = args.arms.split(",")
    space, wopts, w, h, desc = bench.make_workload(args.workload)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT)
    wcam = scenes.standard_camera(space, wopts, w, h)
    ucam = scenes.standard_camera(ui_space, uopts, w, h, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    m = wcam.depth_transform()
    pixels = aicb200.pixel_picker_order(w, h, args.pixels)
    backdrop = (0.1, 0.3, 0.6, 0.5)
    no_world = aicb200.srgb8_to_linear((0xBC, 0xBC, 0xBC)) + (1.0,)

    calls = {}
    if "single" in arms:
        wrt = aicb200.SpaceRaytracer(space, wopts)
        urt = aicb200.SpaceRaytracer(ui_space, uopts, wrt.ctx)
        lw, lu = (wrt, wcam, wopts), (urt, ucam, uopts)
        calls["single"] = (lambda: aicb200.render_layers(lw, lu, backdrop, no_world).info,
                           lambda: aicb200.render_layers_texture(lw, lu, backdrop, no_world, m, pixels)[2])
    if "group" in arms:
        g = aicb200.DeviceGroup([int(d) for d in args.devices.split(",")])
        gw, gu = g.add_scene(space), g.add_scene(ui_space)
        gl, gul = (gw, wcam, wopts), (gu, ucam, uopts)
        calls["group"] = (lambda: g.render_layers(gl, gul, backdrop, no_world).info,
                          lambda: g.render_layers_texture(gl, gul, backdrop, no_world, m, pixels)[2])
    for _ in range(max(1, args.warmup)):
        for frame, batch in calls.values():
            frame()
            batch()
    times = {a: {"frame": ([], []), "batch": ([], [])} for a in calls}
    sampler = bench.ClockSampler(0)
    sampler.start()
    sampler.mark()
    for _ in range(args.steps):
        for arm, (frame, batch) in calls.items():
            for kind, fn in (("frame", frame), ("batch", batch)):
                t0 = time.perf_counter()
                info = fn()
                times[arm][kind][1].append(1e3 * (time.perf_counter() - t0))
                times[arm][kind][0].append(info.kernel_ms)
    clocks = sampler.stop()
    for arm, t in times.items():
        print(json.dumps({
            "arm": arm, "devices": args.devices if arm == "group" else None, "workload": desc, "frame": f"{w}x{h}",
            "layers": "world + 6^3 UI Space + backdrop, NO_WORLD_TO_SHOW", "steps": args.steps,
            "frame_device_ms": float(np.median(t["frame"][0])), "frame_wall_ms": float(np.median(t["frame"][1])),
            "batch_pixels": args.pixels, "batch_device_ms": float(np.median(t["batch"][0])),
            "batch_wall_ms": float(np.median(t["batch"][1])), "gpu": gpu_identity(), "clocks": clocks,
        }))


if __name__ == "__main__":
    main()
