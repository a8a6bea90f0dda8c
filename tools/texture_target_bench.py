"""Times a RaytraceToTexture target kept on the device (aicb_texture_target_*) against the host-side path it replaces, on
one of bench.py's raytracing workloads (world layer only, no backdrop, NO_WORLD_TO_SHOW paint):

  target:  aicb_texture_target_trace — the picks, the tracing and the full-frame store all on the device;
  host:    a slice of pixel_picker_order (the restated PixelPicker, its order computed once) -> aicb_render_layers_texture
           (pixel list up, texels down) -> a scatter into full-frame host arrays, as RaytraceToTexture's set_pixel does.

Per batch size (--picks, and a whole cycle_length) it reports the median device ms and wall ms per batch of each path,
and the order build at each --order-size: the target's create (order on the device) against pixel_picker_order on the
host.  Prints one JSON line with the GPU's name and power limit read in the same run.

    python tools/texture_target_bench.py --workload c2 --picks 50000 --steps 20 --warmup 3
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
import aicb200  # noqa: E402
import bench  # noqa: E402  (the workload definitions)
from aicb200 import scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402


def time_batches(batch, steps, warmup):
    for _ in range(warmup):
        batch()
    dev, wall = [], []
    for _ in range(steps):
        t0 = time.perf_counter()
        info = batch()
        wall.append(1e3 * (time.perf_counter() - t0))
        dev.append(info.kernel_ms)
    return float(np.median(dev)), float(np.median(wall))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--workload", default="c2", choices=["c0", "c1", "c2", "c3"])
    p.add_argument("--picks", type=int, default=50000, help="picks per batch (a whole cycle_length is timed as well)")
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--order-size", action="append", default=None, help="WxH viewports to time the order build at")
    args = p.parse_args()
    if args.picks < 1 or args.steps < 1:
        p.error("--picks and --steps must be >= 1")
    order_sizes = [tuple(int(v) for v in s.split("x")) for s in (args.order_size or ["1920x1080", "3840x2160"])]
    space, opts, w, h, desc = bench.make_workload(args.workload)
    cam = scenes.standard_camera(space, opts, w, h)
    ctx = aicb200.Context()
    rt = aicb200.SpaceRaytracer(space, opts, ctx)
    m = cam.depth_transform()
    no_world = aicb200.srgb8_to_linear((0xBC, 0xBC, 0xBC)) + (1.0,)
    layer = (rt, cam, opts)

    target = aicb200.TextureTarget(w, h, aicb200.TEXTURE_INCREMENTAL, ctx)
    cycle = target.state["cycle_length"]
    order = aicb200.pixel_picker_order(w, h, 2 * cycle)   # the host path's picker, built once
    frame_rgba = np.zeros((w * h, 4), np.uint16)
    frame_depth = np.zeros(w * h, np.float32)
    results = {}
    for n in (args.picks, cycle):
        def on_device():
            target.mark_dirty()
            _, info = target.trace(layer, None, None, no_world, m, n)
            return info

        pos = [0]

        def on_host():
            start = pos[0] % cycle
            px = order[start:start + n]
            pos[0] += n
            rgba, depth, info = aicb200.render_layers_texture(layer, None, None, no_world, m, px)
            frame_rgba[px] = rgba     # set_pixel into the full-frame DrawableTextures
            frame_depth[px] = depth
            return info

        t_dev, t_wall = time_batches(on_device, args.steps, args.warmup)
        h_dev, h_wall = time_batches(on_host, args.steps, args.warmup)
        results[str(n)] = {"target": {"device_ms": t_dev, "wall_ms": t_wall},
                           "host_list": {"device_ms": h_dev, "wall_ms": h_wall}}
    target.close()

    builds = {}
    for ow, oh in order_sizes:
        dev_t, host_t = [], []
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            t = aicb200.TextureTarget(ow, oh, aicb200.TEXTURE_INCREMENTAL, ctx)   # create returns once the order is built
            t1 = time.perf_counter()
            t.close()
            t2 = time.perf_counter()
            aicb200.pixel_picker_order(ow, oh, 1)   # the sort of every pixel; one pick taken
            t3 = time.perf_counter()
            if i >= args.warmup:
                dev_t.append(1e3 * (t1 - t0))
                host_t.append(1e3 * (t3 - t2))
        builds[f"{ow}x{oh}"] = {"target_create_ms": float(np.median(dev_t)),
                                "host_pixel_picker_order_ms": float(np.median(host_t))}
    rt.close()
    ctx.close()
    print(json.dumps({
        "metric": "texture target batch wall ms", "workload": desc, "viewport": [w, h], "cycle_length": cycle,
        "steps": args.steps, "batches": results, "order_build": builds,
        "layers": "world only, no backdrop, NO_WORLD_TO_SHOW", "gpu": gpu_identity(),
    }))


if __name__ == "__main__":
    main()
