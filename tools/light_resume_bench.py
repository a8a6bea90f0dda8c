"""What saving and resuming a Space's light costs (SpaceRaytracer.light_download_queue, light_queue_uninitialized),
next to today's load, which throws the saved field away.  On the C4 shape (bench.py --workload c4): the N^3 Space of
scenes.config_c4, converged (fast_evaluate_light + evaluate_light(1)), then one scenes.c4_edits step propagated to
epsilon 32, so that work is left in the queue.  It prints one JSON line per measurement:
  - "scan": the device time of the load rule's scan (k_queue_cubes) from torch.profiler in a call of its own, and the
    host time of light_queue_uninitialized over --reps calls;
  - "save": the host time of light_download + light_download_queue (what a save reads), --reps times;
  - "resume": aicb_scene_create from the saved form + light_queue_uninitialized + light_evaluate(1), and "reload":
    aicb_scene_create + light_fast_evaluate + light_evaluate(1), each --reps times, alternating, with their cube updates;
then the GPU's name and power limit, read in the same run.

    python tools/light_resume_bench.py --n 256 --reps 3
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
from aicb200 import Space, scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

EPSILON = 1


def kernel_ms(call, name):
    """Device time of the kernels whose name holds `name` during call(), from torch.profiler, in milliseconds."""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        total = 0.0
        for e in prof.events():
            if name in e.name:
                total += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        return total * 1e-3
    except Exception as e:   # the profiler is an aid to this tool, not a requirement of the library
        return f"not measured: {type(e).__name__}: {e}"


def timed(call):
    t0 = time.perf_counter()
    out = call()
    return 1e3 * (time.perf_counter() - t0), out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=256, help="edge of the Space")
    p.add_argument("--edits", type=int, default=1000, help="cube edits of the step propagated to epsilon 32")
    p.add_argument("--reps", type=int, default=3, help="repetitions of each measurement")
    args = p.parse_args()
    if args.n < 32:
        p.error("--n must be >= 32")
    space = scenes.config_c4(args.n)
    opts = aicb200.GraphicsOptions()
    a = aicb200.SpaceRaytracer(space, opts)
    a.light_fast_evaluate()
    a.light_evaluate(EPSILON)
    cubes, ids = scenes.c4_edits(space, args.edits, 0)
    a.light_edit_and_propagate(cubes, ids, 32)
    for k in range(args.reps):
        ms_light, field = timed(a.light_download)
        ms_queue, queue = timed(a.light_download_queue)
        print(json.dumps({"case": "save", "rep": k, "download_ms": ms_light, "download_queue_ms": ms_queue,
                          "queued": int((queue > 0).sum())}), flush=True)
    a.close()
    saved = field.copy()
    saved[queue > 0, 3] = 0   # Serialize for space::Read: a queued cube is saved Uninitialized
    block_ids = space.block_ids.copy()
    for c, i in zip(cubes, ids):
        block_ids[tuple(c)] = i
    loaded = Space(space.lower, block_ids, space.blocks, light=saved, sky_colors=space.sky_colors,
                   light_max_distance=space.light_max_distance)
    n_uninit = int((saved[..., 3] == 0).sum())

    b = aicb200.SpaceRaytracer(loaded, opts)
    b.light_queue_uninitialized()   # (the light state and the module's kernels are in place from here on)
    scan = kernel_ms(b.light_queue_uninitialized, "k_queue_cubes")
    host = [timed(b.light_queue_uninitialized)[0] for _ in range(max(args.reps, 10))]
    print(json.dumps({"case": "scan", "uninitialized": n_uninit, "scan_kernel_ms": scan, "host_ms_min": min(host),
                      "host_ms_median": float(np.median(host)),
                      "bytes_read": int(loaded.light.nbytes + np.prod(space.size))}), flush=True)
    b.close()

    def resume():
        rt = aicb200.SpaceRaytracer(loaded, opts)
        rt.light_queue_uninitialized()
        n, _, _ = rt.light_evaluate(EPSILON)
        rt.close()
        return n

    def reload():
        rt = aicb200.SpaceRaytracer(loaded, opts)
        rt.light_fast_evaluate()
        n, _, _ = rt.light_evaluate(EPSILON)
        rt.close()
        return n

    for k in range(args.reps):
        for name, call in (("resume", resume), ("reload", reload)):
            ms, updates = timed(call)
            print(json.dumps({"case": name, "rep": k, "host_ms": ms, "cube_updates": updates}), flush=True)
    print(json.dumps({"workload": f"C4: {args.n}^3 res-1 Space, octant sky, LightPhysics::Rays{{30}}, "
                                  f"{args.edits} edits propagated to epsilon 32",
                      "gpu": gpu_identity()}), flush=True)


if __name__ == "__main__":
    main()
