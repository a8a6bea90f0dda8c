"""What following a filled box costs on the GPU, on C4's lit Space converged to epsilon 1:
  (a) Mutation::fill / fill_uniform(region) on a scene whose light the library computes: aicb_light_edit_region +
      aicb_light_evaluate(1), against aicb_light_edit_and_propagate(1) with the same cubes listed.  Two scenes on one
      context hold the same Space and light; every step both take the same fill, in alternating order.  The uniform
      fills alternate between an opaque block and AIR, the array fills between random ids and the Space's own.  The
      list call propagates inside the call, so its edit part is the call's host time minus the propagation's device time
      (aicb_light_stats); the box call's edit part is timed on its own.  Both propagations' cube updates are reported.
  (b) SpaceChange::CubeBlock for the same boxes on a scene that only draws: aicb_scene_update_region against
      aicb_scene_update_cubes, each followed by one 1920x1080 frame.
Host clock around calls that return synchronised (the frame synchronises (b)), no profiler running; the kernels' device
times come from a separate pass under torch.profiler.  Prints one JSON line per measurement, then medians with ranges
and the GPU's name and power limit, read in the same run.

    python tools/region_fill_bench.py --steps 4
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
from aicb200 import GraphicsOptions, RtRenderer, Space, SpaceRaytracer, scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

KERNELS = ("k_region_cells", "k_region_light", "k_region_texels", "k_edits", "scatter_cubes_kernel")


def ms_since(t0):
    return 1e3 * (time.perf_counter() - t0)


def box_cubes(lower, edge):
    x, y, z = np.meshgrid(*[np.arange(lower[a], lower[a] + edge) for a in range(3)], indexing="ij")
    return np.stack([x.ravel(), y.ravel(), z.ravel()], axis=1).astype(np.int32)


def fill_of(space, lower, edge, form, step, rng):
    """The step's fill of the box: block_ids as the box calls take them, and one id per cube."""
    size = (edge,) * 3
    if form == "uniform":
        ids = 1 if step % 2 == 0 else 0
    elif step % 2 == 0:
        ids = rng.integers(0, len(space.blocks), size).astype(np.uint16)
    else:
        ids = space.block_ids[tuple(slice(lower[a], lower[a] + edge) for a in range(3))].copy()
    return ids, np.broadcast_to(np.asarray(ids, dtype=np.uint16), size).reshape(-1)


def light_fills(boxed, listed, space, cases, steps):
    rows = []
    rng = np.random.default_rng(1)
    for lower, edge, form in cases:
        cubes = box_cubes(lower, edge)
        for k in range(steps):
            ids, flat = fill_of(space, lower, edge, form, k, rng)

            def box_arm():
                t0 = time.perf_counter()
                changed = boxed.light_edit_region(lower, (edge,) * 3, ids)
                edit = ms_since(t0)
                t1 = time.perf_counter()
                updates = boxed.light_evaluate(1)[0]
                return {"arm": "light_edit_region + light_evaluate", "edit_ms": edit, "propagate_ms": ms_since(t1),
                        "propagate_device_ms": 1e3 * boxed.light_stats()["device_seconds"], "cube_updates": updates,
                        "changed": changed}

            def list_arm():
                t0 = time.perf_counter()
                updates = listed.light_edit_and_propagate(cubes, flat, 1)[0]
                total = ms_since(t0)
                device = 1e3 * listed.light_stats()["device_seconds"]
                return {"arm": "light_edit_and_propagate", "edit_ms": total - device, "propagate_device_ms": device,
                        "total_ms": total, "cube_updates": updates}

            for arm in ((box_arm, list_arm) if k % 2 == 0 else (list_arm, box_arm)):
                rows.append(dict(arm(), edge=edge, form=form, step=k))
                print(json.dumps(rows[-1]), flush=True)
    return rows


def cell_fills(boxed, listed, space, cases, steps):
    opts = GraphicsOptions()
    cam = scenes.standard_camera(space, opts, 1920, 1080)
    renderers = []
    for rt in (boxed, listed):
        r = RtRenderer(cam, rt.ctx)
        r.rt = rt
        r.draw()
        renderers.append(r)
    rows = []
    rng = np.random.default_rng(2)
    for lower, edge, form in cases:
        cubes = box_cubes(lower, edge)
        for k in range(steps):
            ids, flat = fill_of(space, lower, edge, form, k, rng)

            def box_arm():
                t0 = time.perf_counter()
                boxed.update_region(lower, (edge,) * 3, ids)
                call = ms_since(t0)
                renderers[0].draw()
                return {"arm": "update_region + frame", "call_ms": call, "total_ms": ms_since(t0)}

            def list_arm():
                t0 = time.perf_counter()
                listed.update_cubes(cubes, flat)
                call = ms_since(t0)
                renderers[1].draw()
                return {"arm": "update_cubes + frame", "call_ms": call, "total_ms": ms_since(t0)}

            for arm in ((box_arm, list_arm) if k % 2 == 0 else (list_arm, box_arm)):
                rows.append(dict(arm(), edge=edge, form=form, step=k))
                print(json.dumps(rows[-1]), flush=True)
    return rows


def profiled(boxed, listed, space, cases):
    """One fill of each case per call under torch.profiler: the device time of every kernel of the edit."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    rows = []
    rng = np.random.default_rng(3)
    for lower, edge, form in cases:
        cubes = box_cubes(lower, edge)
        ids, flat = fill_of(space, lower, edge, form, 0, rng)
        texels = np.zeros((edge,) * 3 + (4,), dtype=np.uint8)
        calls = {"light_edit_region": lambda: boxed.light_edit_region(lower, (edge,) * 3, ids),
                 "light_edit_and_propagate": lambda: listed.light_edit_and_propagate(cubes, flat, 255),
                 "update_region with light": lambda: boxed.update_region(lower, (edge,) * 3, ids, texels),
                 "update_cubes with light": lambda: listed.update_cubes(cubes, flat, texels.reshape(-1, 4))}
        for name, call in calls.items():
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call()
                torch.cuda.synchronize()
            us = {k: sum(e.time_range.elapsed_us() for e in prof.events() if k in e.name) for k in KERNELS}
            rows.append({"profiled": name, "edge": edge, "form": form, "kernel_us": {k: v for k, v in us.items() if v}})
            print(json.dumps(rows[-1]), flush=True)
    return rows


def spread(values):
    return {"median": float(np.median(values)), "min": float(np.min(values)), "max": float(np.max(values))}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=4, help="fills per box and form, each taken by both arms")
    p.add_argument("--n", type=int, default=256, help="edge of the Space")
    p.add_argument("--edges", type=int, nargs="+", default=[16, 64, 128], help="edges of the boxes")
    args = p.parse_args()
    if args.steps < 2 or max(args.edges) + 8 > args.n:
        p.error("--steps must be >= 2 and the boxes must fit the Space")
    space = scenes.config_c4(n=args.n)
    opts = GraphicsOptions()
    boxed = SpaceRaytracer(space, opts)
    boxed.light_fast_evaluate()
    t0 = time.perf_counter()
    boxed.light_evaluate(1)
    print(json.dumps({"converge_ms": ms_since(t0), "cube_updates": boxed.light_stats()["cube_updates"]}), flush=True)
    boxed.light_take_changes(discard=True)
    # the second scene starts from the same light and an empty queue
    lit = Space(space.lower, space.block_ids, space.blocks, light=boxed.light_download(), sky_colors=space.sky_colors,
                light_max_distance=space.light_max_distance)
    listed = SpaceRaytracer(lit, opts, boxed.ctx)
    # boxes off the 16-byte grid of the cells: rows start at z = 5
    cases = [((8, args.n // 8, 5), edge, form) for edge in args.edges for form in ("uniform", "array")]
    a = light_fills(boxed, listed, space, cases, args.steps)
    b = cell_fills(boxed, listed, space, cases, args.steps)
    c = profiled(boxed, listed, space, cases)
    summary = {}
    for _, edge, form in cases:
        rows = [r for r in a + b if r["edge"] == edge and r["form"] == form]
        out = {}
        for arm in sorted({r["arm"] for r in rows}):
            mine = [r for r in rows if r["arm"] == arm]
            out[arm] = {key: spread([r[key] for r in mine]) for key in mine[0] if key.endswith("_ms") or key == "cube_updates"}
        out["kernel_us"] = {r["profiled"]: r["kernel_us"] for r in c if r["edge"] == edge and r["form"] == form}
        summary[f"{edge}^3 {form}"] = out
    print(json.dumps({"n": args.n, "steps": args.steps, "summary": summary, "gpu": gpu_identity()}), flush=True)
    listed.close()
    boxed.close()


if __name__ == "__main__":
    main()
