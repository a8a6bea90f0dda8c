"""Times batches of views (aicb_render_views_*) against a loop of single frames, on C2 (256^3 mixed transparent) and C1
(128^3 res-16 voxel blocks), one context on device 0.  For V views of S x S, (V, S) in (1024, 64), (256, 128),
(64, 256), (16, 512), antialiasing off and on:

  loop device    V x (aicb_render_device + aicb_render_finish), one camera each, sRGB8 into one CUDA buffer;
  batch device   one aicb_render_views_device + aicb_render_finish into the same buffer;
  batch host     one aicb_render_views_srgb8 into a numpy array.

Per call: wall_ms, a host clock around the call and a device synchronise, and gpu_ms, CUDA events on the torch stream
around it; medians over --steps calls after --warmup.  Each batch is checked byte for byte against the loop's frames of
the same run before it is timed.  Prints one JSON line per workload and a last line with the GPU's name and power
limit read in the same run.

    python tools/views_bench.py --steps 5 --warmup 1
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import aicb200  # noqa: E402
from aicb200 import GraphicsOptions, SpaceRaytracer, abi, scenes  # noqa: E402
from cursor_bench import run  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

SHAPES = ((1024, 64), (256, 128), (64, 256), (16, 512))
DIRS = [(1.0, 0.6, 1.0), (-1.0, 0.3, 0.5), (0.2, 0.9, 0.4), (0.7, 0.1, -1.0), (-0.4, 0.8, -0.6), (1.0, 0.2, -0.3)]


def cameras(space, opts, n, size):
    cams = []
    for v in range(n):
        cam = scenes.standard_camera(space, opts, size, size, direction=DIRS[v % len(DIRS)],
                                     distance_scale=0.8 + 0.4 * (v % 7) / 6.0)
        cam.data.exposure = 0.75 + 0.05 * (v % 11)
        cams.append(cam)
    return cams


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=5)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--workloads", default="c2,c1")
    args = p.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    lib = aicb200.load_library()
    for wl in args.workloads.split(","):
        space = scenes.config_c2(n=256) if wl == "c2" else scenes.config_c1(n=128)
        for aa in (False, True):
            opts = GraphicsOptions(antialiasing_always=aa)
            rt = SpaceRaytracer(space, opts)
            o = opts.to_abi(True)
            for n_views, size in SHAPES:
                cams = cameras(space, opts, n_views, size)
                px = size * size
                table = aicb200.camera_table(cams)
                d_table = torch.from_numpy(table.view(np.uint8).reshape(n_views, -1)).to(dev)
                loop_buf = torch.empty((n_views * px, 4), dtype=torch.uint8, device=dev)
                batch_buf = torch.empty_like(loop_buf)
                stream = torch.cuda.current_stream(dev).cuda_stream or 1
                loop_outs = [abi.DeviceOutputs(srgb8=loop_buf.data_ptr() + 4 * px * v, len=px) for v in range(n_views)]
                batch_outs = abi.DeviceOutputs(srgb8=batch_buf.data_ptr(), len=n_views * px)

                def finish(issue):
                    while True:
                        assert issue() == abi.OK, lib.aicb_last_error()
                        st = lib.aicb_render_finish(rt.handle, None)
                        if st != abi.ERR_RETRY:
                            assert st == abi.OK, lib.aicb_last_error()
                            return

                def loop():
                    for v in range(n_views):
                        finish(lambda v=v: lib.aicb_render_device(rt.handle, C.byref(cams[v].data), C.byref(o), None,
                                                                  C.byref(loop_outs[v]), stream))

                def batch():
                    finish(lambda: lib.aicb_render_views_device(rt.handle, d_table.data_ptr(), n_views, size, size,
                                                                C.byref(o), C.byref(batch_outs), stream))

                host = np.empty((n_views, size, size, 4), np.uint8)

                def batch_host():
                    assert lib.aicb_render_views_srgb8(rt.handle, table.ctypes.data, n_views, C.byref(o),
                                                       host.ctypes.data, n_views * px, None) == abi.OK

                loop()
                batch()
                batch_host()
                torch.cuda.synchronize(dev)
                ref = loop_buf.cpu().numpy()
                assert np.array_equal(batch_buf.cpu().numpy(), ref), "the batch differs from the single frames"
                assert np.array_equal(host.reshape(-1, 4), ref), "the host batch differs from the single frames"
                tag = f"{wl} {n_views}x{size}^2 aa={int(aa)}"
                rays = n_views * px * (4 if aa else 1)
                extra = lambda w, g: {"views": n_views, "size": size, "rays": rays,
                                      "us_per_view_gpu": round(g * 1e3 / n_views, 2)}
                run(torch, dev, tag + " loop device", loop, args.steps, args.warmup, extra)
                run(torch, dev, tag + " batch device", batch, args.steps, args.warmup, extra)
                run(torch, dev, tag + " batch host", batch_host, args.steps, args.warmup, extra)
            rt.close()
    print(json.dumps({"gpu": gpu_identity()}), flush=True)


if __name__ == "__main__":
    main()
