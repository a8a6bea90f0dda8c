"""Times compute_derived's light fields of voxel block tables on the GPU (Context.derive_block_light) against the two
host restatements: Block's numpy derivation and the C++ oracle (oracle_derive/, one thread).

Tables: 256 blocks of resolution 16, 64 of 64 and 16 of 128 (scenes.make_voxel_block, whole data bounds, 3/4 of the
voxels solid), each with every palette alpha 1, every alpha 0.5, and mostly alpha 0.05 (long rays).  Per table:

  wall_ms     median host time of one blocking call (validation, staging, upload, kernels, download);
  device_ms   mean over calls of the summed GPU time of the call's four kernels and its copies, from torch.profiler's
              CUDA activity records (CUPTI timestamps) in a separate profiled run;
  kernels_ms  the kernels alone, and the longest of them (the sequential face sums, k_derive_reduce, at high res);
  numpy_ms / oracle_ms  the host restatements, timed on the first --host-blocks blocks and scaled to the table.

The device's results for the timed blocks are checked bit for bit against the oracle first.  Prints one JSON line per
table and a last line with the GPU's name and power limit read in the same run.

    python tools/derive_bench.py --steps 10 --warmup 2
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import aicb200  # noqa: E402
import deriveorc  # noqa: E402  (the oracle: test infrastructure, read here to check and to compare)
from aicb200 import scenes  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

TABLES = [(256, 16), (64, 64), (16, 128)]
ALPHAS = {"alpha1": dict(alpha=1.0), "alpha0.5": dict(alpha=0.5),
          "alpha0.05": dict(alpha=0.05, transparent_palette_entry=True)}


def table(n, res, kind):
    return [scenes.make_voxel_block(1000 * res + i, resolution=res, partial_bounds=False, **ALPHAS[kind])
            for i in range(n)]


def bits(lights):
    return [np.array([v for c in b.face_colors for v in c] + list(b.color) + list(b.emission), dtype=np.float32)
            .view(np.uint32).tolist() + [b.opaque_faces, int(b.visible)] for b in lights]


def device_times(ctx, blocks, calls):
    """Per call: (kernel ms, copy ms, longest kernel name and ms), from CUDA activity records."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ctx.derive_block_light(blocks)
    kern, copies, longest = [], [], {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        ms = e.device_time / 1e3 if hasattr(e, "device_time") else e.cuda_time / 1e3
        if "k_derive" in e.name:
            kern.append(ms)
            short = e.name.split("k_derive_")[1].split("(")[0]
            longest[short] = max(longest.get(short, 0.0), ms)
        elif "Memcpy" in e.name or "Memset" in e.name:
            copies.append(ms)
    return sum(kern) / calls, sum(copies) / calls, max(longest.items(), key=lambda kv: kv[1])


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--host-blocks", type=int, default=2, help="blocks the host restatements are timed on")
    a = p.parse_args()
    deriveorc.set_libm(deriveorc.LIBM_CR)
    ctx = aicb200.Context(0)
    for n, res in TABLES:
        for kind in ALPHAS:
            blocks = table(n, res, kind)
            hb = blocks[:a.host_blocks]
            t0 = time.perf_counter()
            ref = deriveorc.derive(hb)
            oracle_ms = 1e3 * (time.perf_counter() - t0) * n / len(hb)
            assert bits(ctx.derive_block_light(blocks)[:len(hb)]) == bits(ref), "device differs from the oracle"
            for _ in range(a.warmup):
                ctx.derive_block_light(blocks)
            wall = []
            for _ in range(a.steps):
                t0 = time.perf_counter()
                ctx.derive_block_light(blocks)
                wall.append(1e3 * (time.perf_counter() - t0))
            kern, copies, (longest, longest_ms) = device_times(ctx, blocks, a.steps)
            t0 = time.perf_counter()
            for b in hb:
                b._derive_for_light()
            numpy_ms = 1e3 * (time.perf_counter() - t0) * n / len(hb)
            print(json.dumps({"blocks": n, "resolution": res, "palette": kind, "wall_ms": round(float(np.median(wall)), 3),
                              "device_ms": round(kern + copies, 3), "kernels_ms": round(kern, 3),
                              "longest_kernel": longest, "longest_kernel_ms": round(longest_ms, 3),
                              "numpy_ms": round(numpy_ms, 1), "oracle_ms": round(oracle_ms, 1),
                              "host_blocks_timed": len(hb)}), flush=True)
    print(json.dumps({"gpu": gpu_identity()}))
    ctx.close()


if __name__ == "__main__":
    main()
