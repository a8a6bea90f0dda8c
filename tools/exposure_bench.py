"""Times one exposure step (aicb_step_exposure and its device form) on C2's 256^3 Space with light (one context,
device 0).  Workloads:

  one eye host       one eye through the host call (upload, kernel, download, synchronise);
  one eye device     one eye through the device form on the torch stream (wall: issue + synchronise);
  batch host/device  65 536 eyes (--eyes) at random positions and rotations inside the Space, eyes per second over
                     the median GPU-event time.

Per call: wall_ms, a host clock around the call and a device synchronise, and gpu_ms, CUDA events on the torch
stream around it; medians over --steps calls after --warmup.  The batch's results are checked bit for bit against
the exposure oracle's before timing.  Prints one JSON line per workload and a last line with the GPU's name and power
limit read in the same run.

    python tools/exposure_bench.py --steps 9 --warmup 2
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import aicb200  # noqa: E402
from aicb200 import GraphicsOptions, SpaceRaytracer, scenes  # noqa: E402
import exposureorc  # noqa: E402
from cursor_bench import run  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402


def eyes(space, n, seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    t = np.array(space.lower, np.float64) + np.array(space.size, np.float64) * rng.uniform(0.0, 1.0, (n, 3))
    return np.ascontiguousarray(np.stack([aicb200.view_transform_matrix(q[i], t[i]) for i in range(n)]))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=9)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--eyes", type=int, default=1 << 16)
    args = p.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    space = scenes.config_c2(n=256, seed=3, with_light=True)
    space.light_max_distance = 20
    rt = SpaceRaytracer(space, GraphicsOptions())
    m = eyes(space, args.eyes, seed=1)
    st = aicb200.exposure_states(args.eyes)

    exposureorc.set_libm(1)
    n_check = min(args.eyes, 1 << 12)
    want = exposureorc.ExposureScene(space).step(st[:n_check], m[:n_check], 0.05)
    got = rt.step_exposure(st[:n_check], m[:n_check], 0.05)
    assert exposureorc.same_bytes(got[0], want[0]) and exposureorc.same_bytes(got[1], want[1]), \
        "the GPU differs from the oracle"

    d_st = torch.from_numpy(st.view(np.uint8).reshape(-1, 408).copy()).to(dev)
    d_m = torch.from_numpy(m).to(dev)
    run(torch, dev, "one eye host", lambda: rt.step_exposure(st[:1], m[:1], 0.05), args.steps, args.warmup)
    run(torch, dev, "one eye device", lambda: rt.step_exposure(d_st[:1], d_m[:1], 0.05, device=True), args.steps,
        args.warmup)
    run(torch, dev, "batch host", lambda: rt.step_exposure(st, m, 0.05), args.steps, args.warmup,
        lambda w, g: {"eyes": args.eyes, "eyes_per_s_gpu": round(args.eyes / (g * 1e-3))})
    run(torch, dev, "batch device", lambda: rt.step_exposure(d_st, d_m, 0.05, device=True), args.steps, args.warmup,
        lambda w, g: {"eyes": args.eyes, "eyes_per_s_gpu": round(args.eyes / (g * 1e-3))})
    print(json.dumps({"gpu": gpu_identity()}), flush=True)
    rt.close()


if __name__ == "__main__":
    main()
