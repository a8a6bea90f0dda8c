"""Device time per frame of the C2 frame under motion: the camera orbits the Space's centre, its view direction turning
0.5 degrees of yaw per frame, for 200 frames, as an interactive caller draws it.  Each frame's ray order (by the
previous frame's steps) is then one frame stale, where bench.py repeats one identical frame.  Frames are issued as
bench.py issues them (asynchronous sRGB8 frames into device memory, no per-kernel events, the L2 flushed between
frames) and each is timed with CUDA events on the launch stream.

  python tools/orbit_bench.py [--workload c2] [--frames 200] [--deg 0.5] [--json OUT]

AICB200_LIB selects another build of the library, so that two builds can be compared in alternating runs.  The card's
name, power limit and maximum SM clock are printed with the times.
"""
import argparse
import ctypes as C
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from stage_times import card  # noqa: E402


def orbit(name, frames, deg, warmup):
    import torch
    import aicb200
    from aicb200 import abi, scenes
    lib = aicb200.load_library()

    space, opts, w, h, desc = bench.make_workload(name)
    x0, y0, z0 = 1.0, 0.6, 1.0   # scenes.standard_camera's default direction
    r0, a0 = math.hypot(x0, z0), math.atan2(z0, x0)

    def camera(k):
        a = a0 + math.radians(deg) * k
        return scenes.standard_camera(space, opts, w, h, direction=(r0 * math.cos(a), y0, r0 * math.sin(a)))

    cams = [camera(k) for k in range(warmup + frames)]
    ctx = aicb200.Context(0)
    rt = aicb200.SpaceRaytracer(space, opts, ctx)
    o_abi = opts.to_abi(True)
    shard = abi.Shard(bench.STRIP_ROWS, 0, 1)
    n = lib.aicb_shard_pixel_count(C.byref(cams[0].data), C.byref(shard))
    d_out = torch.empty((n, 4), dtype=torch.uint8, device="cuda")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    info = abi.RenderInfo()

    def check(st):
        if st != 0:
            raise RuntimeError(lib.aicb_last_error().decode())

    # blocking renders size the hit stream for every view of the orbit (as bench.py sizes it for its one view)
    sizing = torch.empty((n, 4), dtype=torch.uint8).pin_memory()
    for cam in cams[::10]:
        check(lib.aicb_render_srgb8(rt.handle, C.byref(cam.data), C.byref(o_abi), C.byref(shard), sizing.data_ptr(), n,
                                    None))
    del sizing
    check(lib.aicb_ctx_stage_timing(ctx.handle, 0))
    sampler = bench.ClockSampler(0)
    sampler.start()
    evs = []
    for k, cam in enumerate(cams):
        if k == warmup:
            torch.cuda.synchronize()
            sampler.mark()
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        check(lib.aicb_render_srgb8_device(rt.handle, C.byref(cam.data), C.byref(o_abi), C.byref(shard),
                                           d_out.data_ptr(), n, C.c_void_p(stream.cuda_stream)))
        e1.record(stream)
        if k >= warmup:
            evs.append((e0, e1))
    torch.cuda.synchronize()
    check(lib.aicb_render_finish(rt.handle, C.byref(info)))
    clocks = sampler.stop()
    ms = np.array([a.elapsed_time(b) for a, b in evs])
    return {"workload": name, "desc": desc, "frames": frames, "deg_per_frame": deg,
            "frame_ms_median": round(float(np.median(ms)), 4), "frame_ms_mean": round(float(ms.mean()), 4),
            "ray_order_last": int(info.ray_order), "sm_mhz": clocks.get("sm_mhz"), "clock_reasons": clocks.get("reasons")}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--workload", default="c2")
    p.add_argument("--frames", type=int, default=200)
    p.add_argument("--deg", type=float, default=0.5, help="yaw per frame, degrees")
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--json", default=None, help="also write the result to this file")
    args = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("orbit_bench.py: no CUDA device")
    dev = card()
    r = orbit(args.workload, args.frames, args.deg, args.warmup)
    print(f"card: {dev['name']}, power limit {dev['power_limit']}, max SM clock {dev['sm_max']}")
    print(f"{r['workload']}: {r['frames']} frames, {r['deg_per_frame']} deg of yaw per frame: device ms per frame "
          f"median {r['frame_ms_median']:.4f} mean {r['frame_ms_mean']:.4f} (ray_order {r['ray_order_last']}); "
          f"SM clock {r['sm_mhz']} MHz {r['clock_reasons']}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": dev, "result": r}, f, indent=1)


if __name__ == "__main__":
    main()
