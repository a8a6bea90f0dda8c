"""Times the scene calls fed from device memory against their host twins fed from the same CUDA tensor after .cpu(),
on a lit 256^3 Space (one context, device 0).  Workloads:

  upload_light     a whole light volume (67 MB) from a tensor;
  download_light   the whole volume into a tensor (host twin: light_download, then .to(device));
  update_region    a 256^3 box of ids;
  update_cubes     10^4 and 10^6 scattered cubes, about 10 % of them named twice;
  light_edit_cubes the same lists as Mutation::set edits, the ids alternating between i and i + 1, so every
                   call changes about as many cubes as the list names;
  mirror_rebuild   the first host call (light_edit_cubes of 16 cubes) after a device update, which rebuilds the host
                   mirror of the block ids, against the same host call with a current mirror.

The arms alternate call by call.  Per call: wall_ms, a host clock around the call and a device synchronise, and
gpu_ms, CUDA events on the torch stream around it; medians over --steps calls after --warmup.  Before timing, each
workload's device arm is checked to leave the same block ids and light as its host arm.  Prints one JSON line per
workload and a last line with the GPU's name and power limit read in the same run.

    python tools/device_inputs_bench.py --steps 10 --warmup 2
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
from aicb200 import Block, GraphicsOptions, Space, SpaceRaytracer, scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

N = 256


def world(n=N):
    """A lit n^3 Space: a floor and hash-scattered opaque, glass and lamp blocks (~12 % fill)."""
    blocks = [Block.air(), Block(color=(0.8, 0.7, 0.6, 1.0)), Block(color=(0.2, 0.9, 0.3, 1.0)),
              Block(color=(0.9, 0.2, 0.1, 0.5)), Block(color=(0.1, 0.1, 0.1, 1.0), emission=(4.0, 3.0, 1.0))]
    h = scenes.grid_hash(17, (n, n, n))
    sel = (h % np.uint64(32)).astype(np.int64)
    ids = np.where(sel < 4, sel + 1, 0).astype(np.uint16)
    ids[:, 0, :] = 1
    light = np.zeros((n, n, n, 4), dtype=np.uint8)
    light[..., 3] = 1   # NO_RAYS
    return Space((0, 0, 0), ids, blocks, light=light, sky_colors=scenes.OCTANT_SKY, light_max_distance=12)


def cube_list(torch, dev, n, seed, n_blocks):
    """n entries: 90 % distinct random cubes, then 10 % of them again with other ids, shuffled."""
    rng = np.random.default_rng(seed)
    m = n - n // 10
    cubes = rng.integers(0, N, (m, 3)).astype(np.int32)
    cubes = np.concatenate([cubes, cubes[rng.integers(0, m, n - m)]])
    order = rng.permutation(n)
    ids = rng.integers(0, n_blocks, n).astype(np.uint16)
    return (torch.from_numpy(cubes[order]).to(dev),
            torch.from_numpy(ids.view(np.int16)).to(dev).view(torch.uint16))


def u16_host(t):
    return t.view(aicb200._torch().int16).cpu().numpy().view(np.uint16)


def timed(torch, dev, call):
    stream = torch.cuda.current_stream(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    e0.record(stream)
    call()
    e1.record(stream)
    torch.cuda.synchronize(dev)
    return 1e3 * (time.perf_counter() - t0), e0.elapsed_time(e1)


def compare(torch, dev, name, arms, steps, warmup):
    """arms: {"host": f, "device": f}, alternated; medians of wall and GPU-event ms."""
    out = {k: ([], []) for k in arms}
    for i in range(warmup + steps):
        for k in (arms if i % 2 == 0 else list(reversed(list(arms)))):
            wall, gpu = timed(torch, dev, arms[k])
            if i >= warmup:
                out[k][0].append(wall)
                out[k][1].append(gpu)
    row = {"workload": name}
    for k, (wall, gpu) in out.items():
        row[f"{k}_wall_ms"] = round(float(np.median(wall)), 3)
        row[f"{k}_gpu_ms"] = round(float(np.median(gpu)), 3)
    print(json.dumps(row), flush=True)


def same_state(a, b, label):
    assert a.block_ids().tobytes() == b.block_ids().tobytes(), f"{label}: block ids differ"
    assert a.light_download().tobytes() == b.light_download().tobytes(), f"{label}: light differs"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    a = p.parse_args()
    torch = aicb200._torch()
    dev = torch.device("cuda", 0)
    space = world()
    ctx = aicb200.Context(0)
    host = SpaceRaytracer(space, GraphicsOptions(), ctx)
    devs = SpaceRaytracer(space, GraphicsOptions(), ctx)
    nb = len(space.blocks)
    rng = np.random.default_rng(1)
    shape = (N, N, N)

    light_t = torch.from_numpy(rng.integers(0, 256, shape + (4,)).astype(np.uint8)).to(dev)
    host.upload_light(light_t.cpu().numpy())
    devs.upload_light(light_t)
    same_state(host, devs, "upload_light")
    compare(torch, dev, "upload_light 256^3", {"host": lambda: host.upload_light(light_t.cpu().numpy()),
                                               "device": lambda: devs.upload_light(light_t)}, a.steps, a.warmup)
    compare(torch, dev, "download_light 256^3", {"host": lambda: torch.from_numpy(host.light_download()).to(dev),
                                                 "device": lambda: devs.light_download(device=True)},
            a.steps, a.warmup)

    ids_t = torch.from_numpy(rng.integers(0, nb, shape).astype(np.uint16).view(np.int16)).to(dev).view(torch.uint16)
    host.update_region((0, 0, 0), shape, u16_host(ids_t))
    devs.update_region((0, 0, 0), shape, ids_t)
    same_state(host, devs, "update_region")
    compare(torch, dev, "update_region 256^3 ids",
            {"host": lambda: host.update_region((0, 0, 0), shape, u16_host(ids_t)),
             "device": lambda: devs.update_region((0, 0, 0), shape, ids_t)}, a.steps, a.warmup)

    for n in (10**4, 10**6):
        c, i = cube_list(torch, dev, n, 3, nb)
        host.update_cubes(c.cpu().numpy(), u16_host(i))
        devs.update_cubes(c, i)
        same_state(host, devs, f"update_cubes {n}")
        compare(torch, dev, f"update_cubes {n}",
                {"host": lambda: host.update_cubes(c.cpu().numpy(), u16_host(i)),
                 "device": lambda: devs.update_cubes(c, i)}, a.steps, a.warmup)

    for n in (10**4, 10**6):
        c, i = cube_list(torch, dev, n, 5, nb)
        lists = [(c, i), (c, ((i.view(torch.int16).to(torch.int32) + 1) % nb).to(torch.int16).view(torch.uint16))]
        turn = {"host": 0, "device": 0}

        def edit(arm, scene):
            c, i = lists[turn[arm] % 2]
            turn[arm] += 1
            if arm == "host":
                return scene.light_edit_cubes(c.cpu().numpy(), u16_host(i))
            return scene.light_edit_cubes(c, i)

        assert edit("host", host) == edit("device", devs), "n_changed differs"
        same_state(host, devs, f"light_edit_cubes {n}")
        assert (host.light_download_queue().tobytes() == devs.light_download_queue().tobytes()), "queue differs"
        compare(torch, dev, f"light_edit_cubes {n}", {"host": lambda: edit("host", host),
                                                      "device": lambda: edit("device", devs)}, a.steps, a.warmup)

    small = [cube_list(torch, dev, 10**4, 9 + k, nb) for k in range(2)]
    probe = np.array([[1 + k, 2, 3] for k in range(16)], dtype=np.int32)
    probe_ids = [np.full(16, v, dtype=np.uint16) for v in (1, 0)]
    rebuild, fresh = [], []
    for k in range(a.warmup + a.steps):
        devs.update_cubes(*small[k % 2])
        w_stale, _ = timed(torch, dev, lambda: devs.light_edit_cubes(probe, probe_ids[k % 2]))
        w_fresh, _ = timed(torch, dev, lambda: devs.light_edit_cubes(probe, probe_ids[(k + 1) % 2]))
        if k >= a.warmup:
            rebuild.append(w_stale)
            fresh.append(w_fresh)
    print(json.dumps({"workload": "mirror_rebuild 256^3 (host light_edit_cubes of 16 cubes)",
                      "stale_mirror_wall_ms": round(float(np.median(rebuild)), 3),
                      "current_mirror_wall_ms": round(float(np.median(fresh)), 3)}), flush=True)
    print(json.dumps({"gpu": gpu_identity()}))
    host.close()
    devs.close()
    ctx.close()


if __name__ == "__main__":
    main()
