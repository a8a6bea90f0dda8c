"""What a new kind of block costs a live scene, on C2's 256^3 Space (bench.py's default workload):
  (a) the first placement of a block the Space never held: append it (aicb_scene_append_blocks) + place it at one cube
      (aicb_scene_update_cubes) + one 1920x1080 frame, against rebuilding the scene with the longer table
      (aicb_scene_create) + one frame.  The arms alternate, --steps times each.
  (b) the append that takes a table of 16384 blocks past 16384: C2's cells on a table padded to 16384 entries, one block
      appended, which re-encodes the 256^3 cells from u16 to u32 on the device.  The call's host time, and the
      widening kernel's device time (its start and end on the device, as torch.profiler records them), --reps times.
Prints one JSON line per measurement, then the medians with the GPU's name and power limit, read in the same run.

    python tools/append_blocks_bench.py --steps 10 --reps 3
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
import bench  # noqa: E402
from aicb200 import Block, RtRenderer, Space, SpaceRaytracer, scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402


def ms_since(t0):
    return 1e3 * (time.perf_counter() - t0)


def first_placements(space, opts, w, h, steps):
    """(a): one step of each arm per round, the append arm first in even rounds."""
    cam = scenes.standard_camera(space, opts, w, h)
    blocks, ids = list(space.blocks), space.block_ids.copy()
    live = SpaceRaytracer(space, opts)
    r = RtRenderer(cam, live.ctx)
    r.rt = live
    r.draw()   # sizes the frame's buffers
    rng = np.random.default_rng(1)
    rows = []
    for k in range(steps):
        block = Block(color=tuple(float(v) for v in rng.uniform(0.1, 1.0, 3)) + (1.0,))
        cube = tuple(int(v) for v in rng.integers(0, space.size[0], 3))
        blocks.append(block)
        ids[cube] = len(blocks) - 1
        world = tuple(cube[a] + space.lower[a] for a in range(3))

        def append_arm():
            t0 = time.perf_counter()
            live.append_blocks([block])
            t1 = time.perf_counter()
            live.update_cubes([world], [len(blocks) - 1])
            t2 = time.perf_counter()
            r.draw()
            return {"arm": "append + update_cubes + frame", "step": k, "total_ms": ms_since(t0),
                    "append_ms": 1e3 * (t1 - t0), "update_cubes_ms": 1e3 * (t2 - t1), "frame_ms": ms_since(t2)}

        def rebuild_arm():
            fresh_space = Space(space.lower, ids, blocks, light=space.light, sky_colors=space.sky_colors,
                                light_max_distance=space.light_max_distance)
            t0 = time.perf_counter()
            fresh = SpaceRaytracer(fresh_space, opts, live.ctx)
            t1 = time.perf_counter()
            f = RtRenderer(cam, live.ctx)
            f.rt = fresh
            f.draw()
            row = {"arm": "scene_create + frame", "step": k, "total_ms": ms_since(t0), "create_ms": 1e3 * (t1 - t0),
                   "frame_ms": ms_since(t1)}
            fresh.close()
            return row

        for arm in ((append_arm, rebuild_arm) if k % 2 == 0 else (rebuild_arm, append_arm)):
            rows.append(arm())
            print(json.dumps(rows[-1]), flush=True)
    live.close()
    return rows


def widening_appends(space, opts, reps):
    """(b): a 256^3 scene created with 16384 blocks (C2's table, padded), one block appended."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    pad = [Block(color=(0.5, 0.5, 0.5, 1.0))] * (16384 - len(space.blocks))
    narrow = Space(space.lower, space.block_ids, list(space.blocks) + pad, light=space.light, sky_colors=space.sky_colors)
    rows = []
    for k in range(reps):
        rt = SpaceRaytracer(narrow, opts)
        before = rt.device_bytes
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            rt.append_blocks([Block(color=(0.9, 0.2, 0.1, 1.0))])
            call_ms = ms_since(t0)
            torch.cuda.synchronize()
        kernel_us = [e.time_range.elapsed_us() for e in prof.events() if "widen_cells_kernel" in e.name]
        rows.append({"case": "append past 16384 blocks (256^3 cells u16 -> u32)", "rep": k, "call_ms": call_ms,
                     "widen_kernel_us": kernel_us[0] if kernel_us else None,
                     "cells_bytes_read": int(space.block_ids.size * 2), "cells_bytes_written": int(space.block_ids.size * 4),
                     "device_bytes_added": rt.device_bytes - before})
        print(json.dumps(rows[-1]), flush=True)
        rt.close()
    return rows


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10, help="rounds of (a), one step of each arm per round")
    p.add_argument("--reps", type=int, default=3, help="widening appends of (b), one fresh scene each")
    args = p.parse_args()
    if args.steps < 1 or args.reps < 1:
        p.error("--steps and --reps must be >= 1")
    space, opts, w, h, desc = bench.make_workload("c2")
    a = first_placements(space, opts, w, h, args.steps)
    b = widening_appends(space, opts, args.reps)
    med = lambda rows, key: float(np.median([r[key] for r in rows if r.get(key) is not None])) if rows else None
    appended = [r for r in a if r["arm"].startswith("append")]
    rebuilt = [r for r in a if r["arm"].startswith("scene_create")]
    print(json.dumps({"workload": desc, "steps": args.steps, "reps": args.reps,
                      "median_ms": {"append + update_cubes + frame": med(appended, "total_ms"),
                                    "append": med(appended, "append_ms"), "frame after append": med(appended, "frame_ms"),
                                    "scene_create + frame": med(rebuilt, "total_ms"),
                                    "scene_create": med(rebuilt, "create_ms"),
                                    "widening append call": med(b, "call_ms")},
                      "median_widen_kernel_us": med(b, "widen_kernel_us"), "gpu": gpu_identity()}), flush=True)


if __name__ == "__main__":
    main()
