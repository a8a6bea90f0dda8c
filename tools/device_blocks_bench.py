"""Times block definitions fed from device memory (update_blocks / append_blocks with DeviceBlocks, that is
aicb_scene_update_blocks_device and aicb_scene_append_blocks_device) against their host twins fed the same tensors
after .cpu(), on C2's and C4's 256^3 Spaces (one context, device 0).  Workloads:

  redefine res-128   one full resolution-128 block (2^21 voxels) redefined in place, two definitions alternating;
  redefine res-16    the same with a resolution-16 block;
  append 256 res-16  256 new resolution-16 blocks per call;
  ... derive         the same three with the light fields derived: the device arm sets AICB_BLOCKS_DERIVE_LIGHT, the
                     host arm calls derive_block_light on the .cpu() voxels and then the host call;
  kind change        a block held by ~1/30 of the cubes alternates between a single voxel and a resolution-16 brick,
                     right after a device cube update (so the host arm first rebuilds the host mirror of the ids).

The arms alternate call by call.  Per call: wall_ms, a host clock around the call and a device synchronise, and
gpu_ms, CUDA events on the torch stream around it (kernels and copies); medians over --steps calls after --warmup.
Before timing, each workload's arms are checked to leave the same block ids and device_bytes.  Prints one JSON line
per workload and a last line with the GPU's name and power limit read in the same run.

    python tools/device_blocks_bench.py --steps 10 --warmup 2
"""
import argparse
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import aicb200  # noqa: E402
from aicb200 import BlockLight, DeviceBlock, GraphicsOptions, SpaceRaytracer, scenes  # noqa: E402
from device_inputs_bench import compare, cube_list, timed, u16_host  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402


_voxels = {}


def voxel_block(seed, **kw):
    """scenes.make_voxel_block, made once per run (its numpy light restatement takes seconds at resolution 128)."""
    if seed not in _voxels:
        _voxels[seed] = scenes.make_voxel_block(seed, **kw)
    return _voxels[seed]


def device_block(torch, dev, b, derive=False):
    idx = None if b.indices is None else torch.from_numpy(b.indices.view(np.int16)).to(dev).view(torch.uint16)
    light = None if derive else BlockLight(tuple(tuple(c) for c in b.light_face_colors), tuple(b.light_color),
                                           tuple(b.light_emission), int(b.light_opaque_faces), bool(b.light_visible))
    return DeviceBlock(b.resolution, b.voxel_lower, idx, torch.from_numpy(b.palette).to(dev), light=light)


def host_twin(db, bl=None):
    """A DeviceBlock as the host call takes it: its tensors copied to the host (.cpu()), its light fields as given or
    `bl` (derive_block_light's)."""
    idx = None if db.indices is None else u16_host(db.indices)
    pal = db.palette.cpu().numpy()
    light = bl or db.light
    return types.SimpleNamespace(
        resolution=db.resolution if idx is not None else 1, is_air=db.is_air, indices=idx, palette=pal,
        voxel_lower=db.voxel_lower if idx is not None else (0, 0, 0),
        voxel_size=tuple(idx.shape) if idx is not None else (1, 1, 1),
        light_opaque_faces=light.opaque_faces if light else 0, light_visible=light.visible if light else False,
        light_face_colors=light.face_colors if light else [(0.0,) * 4] * 6,
        light_color=light.color if light else (0.0,) * 4, light_emission=light.emission if light else (0.0,) * 3)


def host_call(ctx, scene, indices, dbs, derive):
    blocks = [host_twin(db) for db in dbs]
    if derive:
        blocks = [host_twin(db, bl) for db, bl in zip(dbs, ctx.derive_block_light(blocks))]
    if indices is None:
        scene.append_blocks(blocks)
    else:
        scene.update_blocks(indices, blocks)


def same(a, b, label):
    assert a.block_ids().tobytes() == b.block_ids().tobytes(), f"{label}: block ids differ"
    assert a.device_bytes == b.device_bytes, f"{label}: device_bytes differ"


def run(torch, dev, name, space, steps, warmup):
    ctx = aicb200.Context(0)
    host, devs = SpaceRaytracer(space, GraphicsOptions(), ctx), SpaceRaytracer(space, GraphicsOptions(), ctx)
    k = 1   # an opaque single voxel in both Spaces, held by many cubes
    for derive in (False, True):
        tag = " derive" if derive else ""
        for res in (128, 16):
            defs = [device_block(torch, dev, voxel_block(900 + res + j, resolution=res, partial_bounds=False),
                                 derive) for j in range(2)]
            slot = 2 if res == 128 else 3   # a brick from here on
            turn = {"host": 0, "device": 0}

            def redefine(arm, scene):
                d = defs[turn[arm] % 2]
                turn[arm] += 1
                if arm == "host":
                    host_call(ctx, scene, [slot], [d], derive)
                else:
                    scene.update_blocks([slot], [d])

            redefine("host", host)
            redefine("device", devs)
            same(host, devs, f"{name} redefine res-{res}{tag}")
            compare(torch, dev, f"{name} redefine res-{res}{tag}",
                    {"host": lambda: redefine("host", host), "device": lambda: redefine("device", devs)}, steps, warmup)
        batch = [device_block(torch, dev, voxel_block(3000 + j, resolution=16), derive) for j in range(256)]
        host_call(ctx, host, None, batch, derive)
        devs.append_blocks(batch)
        same(host, devs, f"{name} append 256 res-16{tag}")
        compare(torch, dev, f"{name} append 256 res-16{tag}",
                {"host": lambda: host_call(ctx, host, None, batch, derive), "device": lambda: devs.append_blocks(batch)},
                steps, warmup)
    # a block of many cubes changes kind right after a device cube update
    kinds = [device_block(torch, dev, aicb200.Block(color=(0.3, 0.5, 0.7, 1.0))),
             device_block(torch, dev, voxel_block(77, resolution=16))]
    small = cube_list(torch, dev, 10**4, 9, 8)
    turn = {"host": 0, "device": 0}

    def change(arm, scene):
        d = kinds[turn[arm] % 2]
        turn[arm] += 1
        if arm == "host":
            host_call(ctx, scene, [k], [d], False)
        else:
            scene.update_blocks([k], [d])

    results = {"host": [], "device": []}
    for i in range(warmup + steps):
        for arm, scene in (("host", host), ("device", devs)):
            scene.update_cubes(*small)
            wall, gpu = timed(torch, dev, lambda: change(arm, scene))
            if i >= warmup:
                results[arm].append((wall, gpu))
    same(host, devs, f"{name} kind change")
    row = {"workload": f"{name} kind change after a device cube update"}
    for arm, v in results.items():
        row[f"{arm}_wall_ms"] = round(float(np.median([w for w, _ in v])), 3)
        row[f"{arm}_gpu_ms"] = round(float(np.median([g for _, g in v])), 3)
    print(json.dumps(row), flush=True)
    host.close()
    devs.close()
    ctx.close()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    a = p.parse_args()
    torch = aicb200._torch()
    dev = torch.device("cuda", 0)
    run(torch, dev, "C2", scenes.config_c2(), a.steps, a.warmup)
    run(torch, dev, "C4", scenes.config_c4(), a.steps, a.warmup)
    print(json.dumps({"gpu": gpu_identity()}))


if __name__ == "__main__":
    main()
