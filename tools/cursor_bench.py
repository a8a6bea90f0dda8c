"""Times the cursor (aicb_cursor_raycast and its device form) on C2's 256^3 Space (one context, device 0), and the
cost the cursor avoids: rebuilding the host mirror of the block ids after a device update, which is what a host that
picks with block_ids() would pay.  Workloads:

  pick host        one ray through the host call (upload, kernel, download, synchronise);
  pick device      one ray through the device form on the torch stream (wall: issue + synchronise);
  batch            2^20 rays (--rays) from random eyes outside the Space towards random points of it, host call;
                   rays/s over the median GPU-event time;
  oracle           the same batch through the cursor oracle, split over the host's threads;
  mirror refresh   a one-cube device update then aicb_light_edit_cubes of the same cube, which rebuilds the mirror
                   (a 2-byte-per-cube download) before it edits, against the same device update alone.

Per call: wall_ms, a host clock around the call and a device synchronise, and gpu_ms, CUDA events on the torch
stream around it; medians over --steps calls after --warmup.  The batch's results are checked bit for bit against
the oracle's before timing.  Prints one JSON line per workload and a last line with the GPU's name and power limit
read in the same run.

    python tools/cursor_bench.py --steps 9 --warmup 2
"""
import argparse
import concurrent.futures
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
from aicb200 import GraphicsOptions, SpaceRaytracer, scenes  # noqa: E402
import cursororc  # noqa: E402
from device_inputs_bench import timed  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402


def batch_rays(space, n, seed):
    rng = np.random.default_rng(seed)
    lo = np.array(space.lower, np.float64)
    size = np.array(space.size, np.float64)
    eye = lo + size * rng.uniform(-0.2, 1.2, (n, 3))
    aim = lo + size * rng.uniform(0.0, 1.0, (n, 3))
    return np.ascontiguousarray(np.concatenate([eye, aim - eye], axis=1))


def median(xs):
    return round(float(np.median(xs)), 4)


def run(torch, dev, name, call, steps, warmup, extra=None):
    wall, gpu = [], []
    for i in range(warmup + steps):
        w, g = timed(torch, dev, call)
        if i >= warmup:
            wall.append(w)
            gpu.append(g)
    row = {"workload": name, "wall_ms": median(wall), "gpu_ms": median(gpu)}
    row.update(extra(np.median(wall), np.median(gpu)) if extra else {})
    print(json.dumps(row), flush=True)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=9)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--rays", type=int, default=1 << 20)
    p.add_argument("--oracle-rays", type=int, default=1 << 16,
                   help="rays of the batch the oracle is timed on (its rate is per ray)")
    args = p.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    space = scenes.config_c2(n=256, seed=3, with_light=True)
    space.light_max_distance = 20
    rt = SpaceRaytracer(space, GraphicsOptions())
    rays = batch_rays(space, args.rays, seed=1)
    one = rays[:1].copy()
    d_one = torch.from_numpy(one).to(dev)
    d_rays = torch.from_numpy(rays).to(dev)

    oracle = cursororc.CursorScene(space)
    n_check = min(len(rays), 1 << 16)
    assert cursororc.same_bits(rt.cursor_raycast(rays[:n_check]), oracle.cursor_raycast(rays[:n_check])), \
        "the GPU differs from the oracle"
    got = rt.cursor_raycast(rays)
    hits = int((got["block_id"] != aicb200.abi.CURSOR_NONE).sum())

    run(torch, dev, "pick host", lambda: rt.cursor_raycast(one), args.steps, args.warmup)
    run(torch, dev, "pick device", lambda: rt.cursor_raycast(d_one, device=True), args.steps, args.warmup)
    run(torch, dev, "batch host", lambda: rt.cursor_raycast(rays), args.steps, args.warmup,
        lambda w, g: {"rays": len(rays), "selected": hits, "rays_per_s_wall": round(len(rays) / (w * 1e-3)),
                      "rays_per_s_gpu": round(len(rays) / (g * 1e-3))})
    run(torch, dev, "batch device", lambda: rt.cursor_raycast(d_rays, device=True), args.steps, args.warmup,
        lambda w, g: {"rays": len(rays), "rays_per_s_gpu": round(len(rays) / (g * 1e-3))})

    threads = os.cpu_count() or 1
    orays = rays[:args.oracle_rays]
    chunks = np.array_split(orays, threads)
    times = []
    with concurrent.futures.ThreadPoolExecutor(threads) as ex:
        for i in range(1 + max(1, args.steps // 3)):
            t0 = time.perf_counter()
            list(ex.map(oracle.cursor_raycast, chunks))
            if i:
                times.append(time.perf_counter() - t0)
    t = float(np.median(times))
    print(json.dumps({"workload": "oracle", "rays": len(orays), "threads": threads, "wall_ms": round(t * 1e3, 3),
                      "rays_per_s": round(len(orays) / t)}), flush=True)

    # the mirror refresh a device update forces on the next host reader of the ids
    cube = torch.tensor([[5, 6, 7]], dtype=torch.int32, device=dev)
    ids = [torch.tensor([k], dtype=torch.int16, device=dev).view(torch.uint16) for k in (1, 2)]
    k = [0]

    def update():
        k[0] ^= 1
        rt.update_cubes(cube, ids[k[0]])

    def update_then_read():
        update()
        rt.light_edit_cubes(np.array([[5, 6, 7]], np.int32), np.array([k[0] + 1], np.uint16))

    run(torch, dev, "device update", update, args.steps, args.warmup)
    run(torch, dev, "device update + mirror refresh", update_then_read, args.steps, args.warmup)
    print(json.dumps({"gpu": gpu_identity()}), flush=True)
    rt.close()


if __name__ == "__main__":
    main()
