"""Per-kernel times of the bench frames: the median `stage_ms` of each stage (gen, march, shade / resolve, encode) over
many frames of C0-C3, built as bench.py builds them, with the same 256 MiB L2 flush before every frame.

  python tools/stage_times.py [--workloads c2,c0,c1,c3] [--frames 60] [--json OUT]

The stage times come from the library's own CUDA events around each kernel of the frame (aicb_ctx_stage_timing), so
the kernels of a frame do not overlap as they do in the timed bench frames (no programmatic dependent launch): the
sum of the stages is a little more than bench.py's frame time.  The card's name and power limit, and the SM clock
sampled while the frames run, are printed with the times.  AICB200_LIB selects another build of the library.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
import bench  # noqa: E402

STAGES = ("gen", "march", "shade", "encode")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return {"name": None, "power_limit": None, "sm_max": None}
    parts = [p.strip() for p in out.split(",")]
    return dict(zip(("name", "power_limit", "sm_max"), parts + [None] * (3 - len(parts))))


def stage_times(name, frames, warmup):
    import torch
    import aicb200
    from aicb200 import abi, scenes
    lib = aicb200.load_library()

    space, opts, w, h, desc = bench.make_workload(name)
    cam = scenes.standard_camera(space, opts, w, h)
    ctx = aicb200.Context(0)
    rt = aicb200.SpaceRaytracer(space, opts, ctx)
    o_abi = opts.to_abi(True)
    shard = abi.Shard(bench.STRIP_ROWS, 0, 1)
    n = lib.aicb_shard_pixel_count(C.byref(cam.data), C.byref(shard))
    d_out = torch.empty((n, 4), dtype=torch.uint8, device="cuda")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    info = abi.RenderInfo()

    def check(st):
        if st != 0:
            raise RuntimeError(lib.aicb_last_error().decode())

    # a blocking render sizes the hit stream for the workload (as in bench.py)
    sizing = torch.empty((n, 4), dtype=torch.uint8).pin_memory()
    check(lib.aicb_render_srgb8(rt.handle, C.byref(cam.data), C.byref(o_abi), C.byref(shard), sizing.data_ptr(), n, None))
    del sizing
    check(lib.aicb_ctx_stage_timing(ctx.handle, 1))
    sampler = bench.ClockSampler(0)
    sampler.start()
    stage_ms, frame_ms = [], []
    for k in range(warmup + frames):
        if k == warmup:
            sampler.mark()
        flush.zero_()
        check(lib.aicb_render_srgb8_device(rt.handle, C.byref(cam.data), C.byref(o_abi), C.byref(shard),
                                           d_out.data_ptr(), n, C.c_void_p(stream.cuda_stream)))
        torch.cuda.synchronize()
        check(lib.aicb_render_finish(rt.handle, C.byref(info)))
        if k >= warmup:
            stage_ms.append([float(v) for v in info.stage_ms][:len(STAGES)])
            frame_ms.append(float(info.kernel_ms))
    clocks = sampler.stop()
    check(lib.aicb_ctx_stage_timing(ctx.handle, 0))
    med = np.median(np.array(stage_ms), axis=0)
    return {"workload": name, "desc": desc, "frames": frames,
            "stage_ms": {s: round(float(v), 4) for s, v in zip(STAGES, med)},
            "frame_ms": round(float(np.median(frame_ms)), 4),
            "sm_mhz": clocks.get("sm_mhz"), "clock_reasons": clocks.get("reasons")}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--workloads", default="c2,c0,c1,c3")
    p.add_argument("--frames", type=int, default=60)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--json", default=None, help="also write the results to this file")
    args = p.parse_args()
    if args.frames < 50:
        p.error("--frames must be at least 50 (the medians are compared between builds)")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("stage_times.py: no CUDA device")
    dev = card()
    print(f"card: {dev['name']}, power limit {dev['power_limit']}, max SM clock {dev['sm_max']}")
    results = []
    for name in args.workloads.split(","):
        r = stage_times(name, args.frames, args.warmup)
        results.append(r)
        stages = "  ".join(f"{s} {v:.4f}" for s, v in r["stage_ms"].items())
        print(f"{name}: median over {r['frames']} frames, ms: {stages}  (frame {r['frame_ms']:.4f}); "
              f"SM clock {r['sm_mhz']} MHz {r['clock_reasons']}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": dev, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
