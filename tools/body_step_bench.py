"""Times the body step (aicb_step_bodies and its device form) on C2's 256^3 Space (one context, device 0), and the cost
it replaces: downloading the block ids after a device update so that the host can step its bodies.  Workloads:

  batch N          N character-sized bodies (2^10, 2^16, 2^20) at random points of the Space falling with random
                   velocities, one device-form call on the torch stream; gpu_ms is the CUDA-event time of the call;
  one body         one body through the host call and through the device form (wall: issue + synchronise);
  oracle           the 2^16 batch through the body oracle (a CPU step_one_body), over the host's threads;
  host step        what a host that stepped the 2^16 batch itself would pay after a device update: the block ids
                   downloaded to host memory (block_ids(), 2 bytes per cube, after a one-cube device update so that
                   nothing is cached), then the oracle's step of the batch; both parts and their sum.

Medians over --steps calls after --warmup.  The 2^16 batch's results are checked bit for bit against the oracle's
before timing.  Prints one JSON line per workload and a last line with the GPU's name and power limit read in the same
run.

    python tools/body_step_bench.py --steps 9 --warmup 2
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
from aicb200 import GraphicsOptions, SpaceRaytracer, scenes  # noqa: E402
import bodyorc  # noqa: E402
from device_inputs_bench import timed  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

GRAVITY = (0.0, -20.0, 0.0)
DT = 1.0 / 60.0


def batch(space, n, seed):
    rng = np.random.default_rng(seed)
    pos = np.array(space.lower) + rng.random((n, 3)) * np.array(space.size)
    return aicb200.bodies(n, position=pos, collision_box=(-0.35, -1.6, -0.35, 0.35, 0.2, 0.35),
                          velocity=rng.normal(0.0, 4.0, (n, 3)))


def median(xs):
    return round(float(np.median(xs)), 4)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=9)
    p.add_argument("--warmup", type=int, default=2)
    a = p.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    space = scenes.config_c2()
    rt = SpaceRaytracer(space, GraphicsOptions())
    for log2n in (10, 16, 20):
        b = batch(space, 1 << log2n, seed=log2n)
        if log2n == 16:
            want = bodyorc.BodyScene(space).step_bodies(b, DT, GRAVITY, max_contacts=8)
            got = rt.step_bodies(b, DT, GRAVITY, max_contacts=8)
            assert bodyorc.same_bits(got[0], want[0]) and bodyorc.same_bits(got[1], want[1]), "differs from the oracle"
            t0 = time.perf_counter()
            bodyorc.BodyScene(space).step_bodies(b, DT, GRAVITY, max_contacts=8)
            print(json.dumps({"workload": "oracle 2^16", "threads": os.cpu_count(),
                              "wall_ms": round(1e3 * (time.perf_counter() - t0), 3)}), flush=True)
        base = torch.from_numpy(b.view(np.uint8).reshape(len(b), -1).copy()).to(dev)
        wall, gpu = [], []
        for i in range(a.warmup + a.steps):
            d = base.clone()
            w, g = timed(torch, dev, lambda: rt.step_bodies(d, DT, GRAVITY, max_contacts=8, device=True))
            if i >= a.warmup:
                wall.append(w)
                gpu.append(g)
        print(json.dumps({"workload": f"batch 2^{log2n}", "wall_ms": median(wall), "gpu_ms": median(gpu),
                          "bodies_per_s": round((1 << log2n) / (np.median(gpu) * 1e-3))}), flush=True)
    one = batch(space, 1, seed=1)
    host = [timed(torch, dev, lambda: rt.step_bodies(one, DT, GRAVITY))[0] for _ in range(a.warmup + a.steps)]
    d1 = torch.from_numpy(one.view(np.uint8).reshape(1, -1).copy()).to(dev)
    devw = [timed(torch, dev, lambda: rt.step_bodies(d1.clone(), DT, GRAVITY, device=True))[0]
            for _ in range(a.warmup + a.steps)]
    print(json.dumps({"workload": "one body", "host_wall_ms": median(host[a.warmup:]),
                      "device_wall_ms": median(devw[a.warmup:])}), flush=True)
    cube = torch.tensor([[0, 0, 0]], dtype=torch.int32, device=dev)
    ids = torch.tensor([1], dtype=torch.int16, device=dev).view(torch.uint16)
    dl = []
    for _ in range(a.warmup + a.steps):
        rt.update_cubes(cube, ids)   # a device update: the host's copy of the ids is stale
        torch.cuda.synchronize(dev)
        dl.append(timed(torch, dev, lambda: rt.block_ids())[0])
    b = batch(space, 1 << 16, seed=16)
    t0 = time.perf_counter()
    bodyorc.BodyScene(space).step_bodies(b, DT, GRAVITY, max_contacts=8)
    step_ms = 1e3 * (time.perf_counter() - t0)
    print(json.dumps({"workload": "host step of 2^16 after a device update", "ids_download_ms": median(dl[a.warmup:]),
                      "oracle_step_ms": round(step_ms, 3), "total_ms": round(median(dl[a.warmup:]) + step_ms, 3)}),
          flush=True)
    print(json.dumps({"gpu": gpu_identity()}), flush=True)


if __name__ == "__main__":
    main()
