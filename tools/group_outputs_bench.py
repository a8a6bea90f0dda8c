"""Times the world-only outputs of one context on a device group against the same calls on one context: a ColorBuf
frame (+ depth, hit, steps) of a bench.py workload (aicb_render_colorbuf / aicb_group_render_colorbuf), a batch of
explicit rays (aicb_trace_rays / aicb_group_trace_rays) and an orthographic image of the C1 Space
(aicb_render_orthographic / aicb_group_render_orthographic).  The arms alternate call by call.  Prints one JSON line per
arm and call with the median device time (the slowest device's) and the median wall time, and the GPU's name, power
limit and clocks read in the same run.

    python tools/group_outputs_bench.py --workload c2 --rays 1000000 --resolution 32 --devices 0 --steps 20
    python tools/group_outputs_bench.py --calls ortho --arms single --package DIR   # another build of the package
"""
import argparse
import importlib.util
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def load_package(path):
    """The aicb200 package from `path` (a directory holding aicb200/ and its built library), or this tree's."""
    if not path:
        import aicb200
        return aicb200
    spec = importlib.util.spec_from_file_location("aicb200", os.path.join(path, "aicb200", "__init__.py"),
                                                  submodule_search_locations=[os.path.join(path, "aicb200")])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["aicb200"] = mod
    spec.loader.exec_module(mod)
    return mod


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--workload", default="c2", choices=["c0", "c1", "c2", "c3"], help="the ColorBuf frame's workload")
    p.add_argument("--rays", type=int, default=1_000_000)
    p.add_argument("--resolution", type=int, default=32, help="pixels per cube of the C1 orthographic image")
    p.add_argument("--devices", default="0", help="the group's device ids, comma separated (may repeat)")
    p.add_argument("--arms", default="single,group")
    p.add_argument("--calls", default="colorbuf,rays,ortho")
    p.add_argument("--package", default=None, help="directory of another build of the aicb200 package (single arm)")
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    args = p.parse_args()
    aicb200 = load_package(args.package)   # before bench imports this tree's package under the same name
    import bench  # (the workload definitions and the clock sampler)
    from aicb200 import GraphicsOptions, scenes
    from texture_bench import gpu_identity
    arms, kinds = args.arms.split(","), args.calls.split(",")
    space, opts, w, h, desc = bench.make_workload(args.workload)
    cam = scenes.standard_camera(space, opts, w, h)
    ortho_space = scenes.config_c1()
    rng = np.random.default_rng(1)
    lo, size = np.array(space.lower, np.float64), np.array(space.size, np.float64)
    rays = np.concatenate([lo + rng.uniform(-0.25, 1.25, size=(args.rays, 3)) * size,
                           rng.normal(size=(args.rays, 3))], axis=1)

    calls = {}
    if "single" in arms:
        r = aicb200.RtRenderer(cam)
        r.update(space)
        ort = aicb200.SpaceRaytracer(ortho_space, GraphicsOptions.unaltered_colors(), r.ctx)
        calls["single"] = {"colorbuf": lambda: r.draw_colorbuf()["info"],
                           "rays": lambda: r.rt.trace_rays(rays, True, True, True, True)["info"],
                           "ortho": lambda: aicb200.render_orthographic(ort, args.resolution).info}
    if "group" in arms:
        g = aicb200.DeviceGroup([int(d) for d in args.devices.split(",")])
        g.update(space)
        go = aicb200.DeviceGroup([int(d) for d in args.devices.split(",")])
        go.update(ortho_space)
        calls["group"] = {"colorbuf": lambda: g.draw_colorbuf(cam, cam.options)["info"],
                          "rays": lambda: g.trace_rays(rays, cam.options, True, True, True, True)["info"],
                          "ortho": lambda: go.render_orthographic(args.resolution).info}
    for _ in range(max(1, args.warmup)):
        for arm in calls.values():
            for k in kinds:
                arm[k]()
    times = {a: {k: ([], []) for k in kinds} for a in calls}
    sampler = bench.ClockSampler(0)
    sampler.start()
    sampler.mark()
    for _ in range(args.steps):
        for k in kinds:
            for arm, fns in calls.items():
                t0 = time.perf_counter()
                info = fns[k]()
                times[arm][k][1].append(1e3 * (time.perf_counter() - t0))
                times[arm][k][0].append(info.kernel_ms)
    clocks = sampler.stop()
    what = {"colorbuf": f"{desc} {w}x{h} ColorBuf + depth + hit + steps", "rays": f"{args.rays} rays into {desc}",
            "ortho": f"C1 orthographic image, resolution {args.resolution}"}
    for arm, t in times.items():
        for k, (dev, wall) in t.items():
            print(json.dumps({"arm": arm, "package": args.package, "devices": args.devices if arm == "group" else None,
                              "call": k, "what": what[k], "steps": args.steps,
                              "device_ms": float(np.median(dev)), "wall_ms": float(np.median(wall)),
                              "gpu": gpu_identity(), "clocks": clocks}))


if __name__ == "__main__":
    main()
