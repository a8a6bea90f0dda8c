"""Times scene creation from device memory (SpaceRaytracer from a DeviceSpace, that is aicb_scene_create_device)
against the host creation from numpy arrays (aicb_scene_create), on C2's and C4's 256^3 Spaces with their light
volumes (one context, device 0).  The device arm's ids, light and voxels are CUDA tensors made before timing.
Workloads:

  create          the Space with its blocks' light fields given;
  create derive   the device arm sets AICB_BLOCKS_DERIVE_LIGHT; the host arm creates from blocks whose light fields
                  derive_block_light computed before timing;
  fill res-128    fill_uniform with one resolution-128 block (2^21 voxels) against fill_uniform_device with the same
                  block as tensors, on the created C2 or C4 scene.

The arms alternate call by call.  Per call: wall_ms, a host clock around the call and a device synchronise, and
gpu_ms, CUDA events on the torch stream around it; medians over --steps calls after --warmup.  A created scene is
closed outside the timed window.  Before timing, each workload's arms are checked to leave the same block ids, light
and device_bytes.  Prints one JSON line per workload and a last line with the GPU's name and power limit read in the
same run.

    python tools/device_create_bench.py --steps 7 --warmup 2
"""
import argparse
import copy
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import aicb200  # noqa: E402
from aicb200 import DeviceSpace, GraphicsOptions, Space, SpaceRaytracer, scenes  # noqa: E402
import device_blocks_bench  # noqa: E402
from device_blocks_bench import voxel_block  # noqa: E402
from device_inputs_bench import compare, timed  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402


def tensor(torch, dev, a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint16:
        return torch.from_numpy(a.view(np.int16)).to(dev).view(torch.uint16)
    return torch.from_numpy(a).to(dev)


def device_block(torch, dev, b, derive=False):
    d = device_blocks_bench.device_block(torch, dev, b, derive)
    d.is_air = b.is_air
    return d


def device_space(torch, dev, space, derive):
    return DeviceSpace(space.lower, tensor(torch, dev, space.block_ids),
                       [device_block(torch, dev, b, derive) for b in space.blocks],
                       light=None if space.light is None else tensor(torch, dev, space.light),
                       sky_colors=space.sky_colors, light_max_distance=space.light_max_distance)


def same(a, b, label):
    assert a.block_ids().tobytes() == b.block_ids().tobytes(), f"{label}: block ids differ"
    assert a.light_download().tobytes() == b.light_download().tobytes(), f"{label}: light differs"
    assert a.device_bytes == b.device_bytes, f"{label}: device_bytes differ"


def creations(torch, dev, label, arms, steps, warmup):
    """arms: {"host": make, "device": make}, each returning a new scene; alternated, each scene closed untimed."""
    made = {k: arms[k]() for k in arms}
    same(made["host"], made["device"], label)
    for s in made.values():
        s.close()
    out = {k: [] for k in arms}
    for i in range(warmup + steps):
        for k in (list(arms) if i % 2 == 0 else list(reversed(list(arms)))):
            scene = []
            wall, gpu = timed(torch, dev, lambda: scene.append(arms[k]()))
            scene[0].close()
            if i >= warmup:
                out[k].append((wall, gpu))
    row = {"workload": label}
    for k, v in out.items():
        row[f"{k}_wall_ms"] = round(float(np.median([w for w, _ in v])), 3)
        row[f"{k}_gpu_ms"] = round(float(np.median([g for _, g in v])), 3)
    print(json.dumps(row), flush=True)


def run(torch, dev, name, space, steps, warmup):
    ctx = aicb200.Context(0)
    opts = GraphicsOptions()
    ds = device_space(torch, dev, space, False)
    creations(torch, dev, f"{name} create", {"host": lambda: SpaceRaytracer(space, opts, ctx),
                                             "device": lambda: SpaceRaytracer(ds, opts, ctx)}, steps, warmup)
    derived = [copy.copy(b) for b in space.blocks]   # (the Space's own blocks keep their light fields)
    for b, bl in zip(derived, ctx.derive_block_light(derived)):
        b.set_light_data(bl)
    host_space = Space(space.lower, space.block_ids, derived, light=space.light, sky_colors=space.sky_colors,
                       light_max_distance=space.light_max_distance)
    dd = device_space(torch, dev, space, True)
    creations(torch, dev, f"{name} create derive", {"host": lambda: SpaceRaytracer(host_space, opts, ctx),
                                                    "device": lambda: SpaceRaytracer(dd, opts, ctx)}, steps, warmup)
    block = voxel_block(128, resolution=128, partial_bounds=False)
    db = device_block(torch, dev, block)
    host, devs = SpaceRaytracer(space, opts, ctx), SpaceRaytracer(space, opts, ctx)
    host.fill_uniform(block)
    devs.fill_uniform(db)
    same(host, devs, f"{name} fill res-128")
    compare(torch, dev, f"{name} fill res-128", {"host": lambda: host.fill_uniform(block),
                                                 "device": lambda: devs.fill_uniform(db)}, steps, warmup)
    host.close()
    devs.close()
    ctx.close()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=7)
    p.add_argument("--warmup", type=int, default=2)
    a = p.parse_args()
    torch = aicb200._torch()
    dev = torch.device("cuda", 0)
    run(torch, dev, "C2", scenes.config_c2(with_light=True), a.steps, a.warmup)
    run(torch, dev, "C4", scenes.config_c4(), a.steps, a.warmup)
    print(json.dumps({"gpu": gpu_identity()}))


if __name__ == "__main__":
    main()
