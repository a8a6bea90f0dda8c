"""What a wide brick pool (u32 words, for blocks with more than 32768 palette entries) costs, on bench.py's C1 and C2:
  (a) frame time with the pool narrow against the same Space's pool widened by one appended block of resolution 64
      with 40000 palette entries that no cube holds (every brick word is then read as u32).  Two scenes on one
      context, one frame of each per round, the narrow one first in even rounds; the frame's kernel time
      (aicb_render_info::kernel_ms) and host time;
  (b) that widening append: the call's host time, and widen_bricks_kernel's device time (as torch.profiler records
      it), one fresh narrow scene per repetition.
Prints one JSON line per measurement, then the medians with the GPU's name and power limit, read in the same run.

    python tools/wide_palette_bench.py --steps 20 --reps 3
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import aicb200  # noqa: E402
import bench  # noqa: E402
import widepal  # noqa: E402
from aicb200 import RtRenderer, SpaceRaytracer, scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402


def frames(name, space, opts, w, h, wide, steps, warmup):
    cam = scenes.standard_camera(space, opts, w, h)
    narrow = SpaceRaytracer(space, opts)
    widened = SpaceRaytracer(space, opts, narrow.ctx)
    widened.append_blocks([wide])
    arms = {}
    for label, rt in (("narrow", narrow), ("widened", widened)):
        r = RtRenderer(cam, narrow.ctx)
        r.rt = rt
        arms[label] = r
    assert np.array_equal(arms["narrow"].draw().data, arms["widened"].draw().data)
    for _ in range(warmup):
        for r in arms.values():
            r.draw()
    rows = []
    for k in range(steps):
        for label in (("narrow", "widened") if k % 2 == 0 else ("widened", "narrow")):
            t0 = time.perf_counter()
            img = arms[label].draw()
            rows.append({"workload": name, "pool": label, "step": k, "kernel_ms": img.info.kernel_ms,
                         "host_ms": 1e3 * (time.perf_counter() - t0)})
            print(json.dumps(rows[-1]), flush=True)
    widened.close()
    narrow.close()
    return rows


def widening(name, space, opts, wide, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    rows = []
    for k in range(reps):
        rt = SpaceRaytracer(space, opts)
        before = rt.device_bytes
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            rt.append_blocks([wide])
            call_ms = 1e3 * (time.perf_counter() - t0)
            torch.cuda.synchronize()
        kernel_us = [e.time_range.elapsed_us() for e in prof.events() if "widen_bricks_kernel" in e.name]
        rows.append({"workload": name, "rep": k, "call_ms": call_ms, "widen_kernel_us": kernel_us[0] if kernel_us else None,
                     "device_bytes_added": rt.device_bytes - before})
        print(json.dumps(rows[-1]), flush=True)
        rt.close()
    return rows


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20, help="rounds of (a), one frame of each pool per round")
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--reps", type=int, default=3, help="widening appends of (b), one fresh scene each")
    args = p.parse_args()
    if args.steps < 1 or args.reps < 1 or args.warmup < 0:
        p.error("--steps and --reps must be >= 1, --warmup >= 0")
    wide, _ = widepal.wide_block(11, 64, 40000)
    med = lambda rows, key: float(np.median([r[key] for r in rows if r.get(key) is not None])) if rows else None
    summary = {}
    for name in ("c1", "c2"):
        space, opts, w, h, desc = bench.make_workload(name)
        a = frames(name, space, opts, w, h, wide, args.steps, args.warmup)
        b = widening(name, space, opts, wide, args.reps)
        summary[name] = {"workload": desc,
                         "median_kernel_ms": {p: med([r for r in a if r["pool"] == p], "kernel_ms")
                                              for p in ("narrow", "widened")},
                         "median_host_ms": {p: med([r for r in a if r["pool"] == p], "host_ms")
                                            for p in ("narrow", "widened")},
                         "median_widening_call_ms": med(b, "call_ms"),
                         "median_widen_kernel_us": med(b, "widen_kernel_us")}
    print(json.dumps({"steps": args.steps, "reps": args.reps, "summary": summary, "gpu": gpu_identity()}), flush=True)


if __name__ == "__main__":
    main()
