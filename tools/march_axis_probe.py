"""How much the cell layout costs the marching kernel: C2's Space drawn from a view mostly along x and from the same
view mostly along z.  The Space is statistically isotropic, so both views do the same work (the AUX counters say how
much); the difference in march time is the price of the direction the cells are laid out in.

  python tools/march_axis_probe.py [--frames 60] [--json OUT]

Each view reports the median march `stage_ms` over the frames, with the same 256 MiB L2 flush before every frame as
bench.py and tools/stage_times.py, and the outer / inner steps and surface hits of one AUX pass.  The card's name and
power limit, and the SM clock sampled while the frames run, are printed with the times.  AICB200_LIB selects another
build of the library.
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
import bench  # noqa: E402
from stage_times import STAGES, card  # noqa: E402

VIEWS = {"x": (1.0, 0.15, 0.2), "z": (0.2, 0.15, 1.0)}


def probe(space, opts, w, h, direction, frames, warmup):
    import torch
    import aicb200
    from aicb200 import abi, scenes
    lib = aicb200.load_library()

    cam = scenes.standard_camera(space, opts, w, h, direction=direction)
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

    sizing = torch.empty((n, 4), dtype=torch.uint8).pin_memory()
    check(lib.aicb_render_srgb8(rt.handle, C.byref(cam.data), C.byref(o_abi), C.byref(shard), sizing.data_ptr(), n, None))
    del sizing
    check(lib.aicb_ctx_stage_timing(ctx.handle, 1))
    sampler = bench.ClockSampler(0)
    sampler.start()
    stage_ms = []
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
    clocks = sampler.stop()
    check(lib.aicb_ctx_stage_timing(ctx.handle, 0))

    r = aicb200.RtRenderer(cam, ctx)
    r.rt = rt
    ai = r.draw_colorbuf(shard=(bench.STRIP_ROWS, 0, 1), want_depth=False, want_hit=False, want_steps=False)["info"]
    med = np.median(np.array(stage_ms), axis=0)
    return {"direction": direction, "frames": frames,
            "stage_ms": {s: round(float(v), 4) for s, v in zip(STAGES, med)},
            "outer_steps": ai.counters[0], "inner_steps": ai.counters[1], "surface_hits": ai.counters[2],
            "sm_mhz": clocks.get("sm_mhz"), "clock_reasons": clocks.get("reasons")}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--frames", type=int, default=60)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--json", default=None, help="also write the results to this file")
    args = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("march_axis_probe.py: no CUDA device")
    dev = card()
    print(f"card: {dev['name']}, power limit {dev['power_limit']}, max SM clock {dev['sm_max']}")
    space, opts, w, h, _ = bench.make_workload("c2")
    results = {}
    for view, d in VIEWS.items():
        r = probe(space, opts, w, h, d, args.frames, args.warmup)
        results[view] = r
        print(f"{view} view {d}: march {r['stage_ms']['march']:.4f} ms (gen {r['stage_ms']['gen']:.4f}, shade "
              f"{r['stage_ms']['shade']:.4f}, encode {r['stage_ms']['encode']:.4f}); outer {r['outer_steps']}, inner "
              f"{r['inner_steps']}, hits {r['surface_hits']}; SM clock {r['sm_mhz']} MHz {r['clock_reasons']}",
              flush=True)
    x, z = results["x"], results["z"]
    gap = x["stage_ms"]["march"] / z["stage_ms"]["march"] - 1.0
    steps = x["outer_steps"] / z["outer_steps"] - 1.0
    print(f"march x / z - 1: {100 * gap:+.1f} %  (outer steps x / z - 1: {100 * steps:+.1f} %)")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": dev, "views": results, "march_gap": gap, "outer_step_gap": steps}, f, indent=1)


if __name__ == "__main__":
    main()
