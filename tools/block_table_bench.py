"""What following a live Space's block table costs on the GPU:
  (a) SpaceChange::EveryBlock on C4's lit 256^3 Space: aicb_scene_fill_uniform + aicb_light_queue_region(bounds, 210),
      against rebuilding the scene from host arrays (aicb_scene_create + aicb_light_queue_uninitialized +
      aicb_light_queue_region).  The arms alternate, --steps times each, both timed by a host clock around calls that
      return synchronised and with no profiler running; fill_cells_kernel's device time comes from a separate pass under
      torch.profiler.
  (b) --updates redefinitions of one full resolution-16 block, then of one full resolution-128 block, each in a Space
      holding only that block: the time per aicb_scene_update_blocks call (no profiler running), then in a separate pass
      under torch.profiler compact_pool_kernel's device time, and its effective bandwidth (bytes read + written by the compaction over kernel time) against the H100 SXM data sheet's
      3.35 TB/s.
Prints one JSON line per measurement, then the medians with the GPU's name and power limit, read in the same run.

    python tools/block_table_bench.py --steps 6 --updates 40
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
from aicb200 import Block, GraphicsOptions, Space, SpaceRaytracer, scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet (not measured)


def ms_since(t0):
    return 1e3 * (time.perf_counter() - t0)


def kernel_us(prof, name):
    return [e.time_range.elapsed_us() for e in prof.events() if name in e.name]


def fills(steps):
    """(a): one step of each arm per round, the fill arm first in even rounds."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    space = scenes.config_c4(n=256)
    opts = GraphicsOptions()
    live = SpaceRaytracer(space, opts)
    live.light_fast_evaluate()
    filled = Space(space.lower, np.zeros_like(space.block_ids), [Block.air()], light=live.light_download(),
                   sky_colors=space.sky_colors, light_max_distance=space.light_max_distance)
    rows = []
    for k in range(steps):
        def fill_arm():
            t0 = time.perf_counter()
            live.fill_uniform(Block.air())
            live.light_queue_region(space.lower, space.size, 210)
            return {"arm": "fill_uniform + queue_region", "step": k, "total_ms": ms_since(t0)}

        def rebuild_arm():
            t0 = time.perf_counter()
            fresh = SpaceRaytracer(filled, opts, live.ctx)
            t1 = time.perf_counter()
            fresh.light_queue_uninitialized()
            fresh.light_queue_region(space.lower, space.size, 210)
            row = {"arm": "scene_create + queue_uninitialized + queue_region", "step": k, "total_ms": ms_since(t0),
                   "create_ms": 1e3 * (t1 - t0)}
            fresh.close()
            return row

        for arm in ((fill_arm, rebuild_arm) if k % 2 == 0 else (rebuild_arm, fill_arm)):
            rows.append(arm())
            print(json.dumps(rows[-1]), flush=True)
    for k in range(steps):   # the kernel's device time, in a pass of its own
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            live.fill_uniform(Block.air())
            torch.cuda.synchronize()
        us = kernel_us(prof, "fill_cells_kernel")
        rows.append({"arm": "profiled fill_uniform", "step": k, "fill_kernel_us": us[0] if us else None})
        print(json.dumps(rows[-1]), flush=True)
    live.close()
    return rows


def redefinitions(resolution, updates):
    """(b) for one resolution: two full definitions alternate at index 1 of a 4^3 Space."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    defs = [scenes.make_voxel_block(s, resolution=resolution, partial_bounds=False) for s in (3, 4)]
    ids = np.zeros((4, 4, 4), np.uint16)
    ids[1, 2, 1] = 1
    rt = SpaceRaytracer(Space((0, 0, 0), ids, [Block.air(), defs[0]]), GraphicsOptions())
    # what one compaction moves: the live bricks (u16) and palette entries (two float4 and one float2), read and written
    live_bytes = defs[0].indices.size * 2 + len(defs[0].palette) * (32 + 8)
    rows = []
    for k in range(updates):
        before = rt.device_bytes
        t0 = time.perf_counter()
        rt.update_blocks([1], [defs[(k + 1) % 2]])
        rows.append({"case": f"update_blocks, full resolution-{resolution} block", "call": k, "call_ms": ms_since(t0),
                     "compacted": rt.device_bytes < before})
        print(json.dumps(rows[-1]), flush=True)
    for k in range(updates):   # the compaction kernel's device time, in a pass of its own
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            rt.update_blocks([1], [defs[(k + 1) % 2]])
            torch.cuda.synchronize()
        us = kernel_us(prof, "compact_pool_kernel")
        row = {"case": f"profiled update_blocks, full resolution-{resolution} block", "call": k,
               "compact_launches": len(us)}
        if us:
            t = sum(us) * 1e-6
            row.update({"compact_kernel_us": sum(us), "compact_bytes": 2 * live_bytes,
                        "compact_gb_per_s": 2 * live_bytes / t / 1e9, "share_of_datasheet_hbm": 2 * live_bytes / t / HBM_BYTES_PER_S})
        rows.append(row)
        print(json.dumps(row), flush=True)
    rt.close()
    return rows


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=6, help="rounds of (a), one step of each arm per round")
    p.add_argument("--updates", type=int, default=40, help="update_blocks calls of (b) per resolution")
    args = p.parse_args()
    if args.steps < 1 or args.updates < 4:
        p.error("--steps must be >= 1 and --updates >= 4")
    a = fills(args.steps)
    b = {res: redefinitions(res, args.updates) for res in (16, 128)}
    med = lambda rows, key: float(np.median([r[key] for r in rows if r.get(key) is not None])) \
        if any(r.get(key) is not None for r in rows) else None
    filled = [r for r in a if r["arm"].startswith("fill")]
    rebuilt = [r for r in a if r["arm"].startswith("scene_create")]
    profiled = [r for r in a if r["arm"].startswith("profiled")]
    summary = {"fill_256": {"fill_uniform + queue_region ms": med(filled, "total_ms"),
                            "fill_kernel_us": med(profiled, "fill_kernel_us"),
                            "rebuild ms": med(rebuilt, "total_ms"), "scene_create ms": med(rebuilt, "create_ms")}}
    for res, rows in b.items():
        timed = [r for r in rows if "call_ms" in r][2:]   # the first calls warm the pools' allocations up
        prof = [r for r in rows if "compact_launches" in r]
        summary[f"update_res{res}"] = {"call_ms": med(timed, "call_ms"),
                                       "calls_that_compacted": sum(1 for r in timed if r["compacted"]),
                                       "timed_calls": len(timed),
                                       "compact_kernel_us": med(prof, "compact_kernel_us"),
                                       "compact_gb_per_s": med(prof, "compact_gb_per_s"),
                                       "share_of_datasheet_hbm": med(prof, "share_of_datasheet_hbm")}
    print(json.dumps({"steps": args.steps, "updates": args.updates, "median": summary, "gpu": gpu_identity()}), flush=True)


if __name__ == "__main__":
    main()
