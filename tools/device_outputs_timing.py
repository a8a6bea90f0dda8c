"""Times a ColorBuf frame (+ depth, hit) of a bench.py workload delivered to the host against the same frame left in
device memory: RtRenderer.draw_colorbuf (aicb_render_colorbuf: a device->host copy of 16 + 8 + 32 bytes per pixel and
a host synchronisation inside the call) against draw_colorbuf(device=True) + result() (aicb_render_device +
aicb_render_finish), and the same pair on a device group (aicb_group_render_colorbuf against
aicb_group_render_device).  The host arms' outputs are preallocated numpy arrays, as a caller reusing its buffers has:
pageable ones (the driver stages that copy) and pinned ones (the copy goes straight to them); the device arms' are
preallocated CUDA tensors (out=).  The arms alternate frame by frame, each frame behind a 256 MiB
L2 flush outside the timed region.  Prints one JSON line per arm with the median and spread of the end-to-end wall
time (issue to outputs final, host clock around work that ends in a synchronisation), the outputs' equality, and the
GPU's name and power limit read in the same run.

    python tools/device_outputs_timing.py --workload c2 --steps 30 --warmup 3 --devices 0,1,2,3
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
import bench  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return None
    return out.splitlines()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--workload", default="c2", choices=["c0", "c1", "c2", "c3"])
    p.add_argument("--devices", default="", help="the group's device ids, comma separated (default: every GPU)")
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=3)
    args = p.parse_args()

    import torch
    import aicb200
    from aicb200 import abi, scenes

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement runs on the GPU only")
    space, opts, w, h, desc = bench.make_workload(args.workload)
    cam = scenes.standard_camera(space, opts, w, h)
    n = w * h
    devices = [int(d) for d in args.devices.split(",")] if args.devices else list(range(torch.cuda.device_count()))
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda:0")

    r = aicb200.RtRenderer(cam, aicb200.Context(0))
    r.update(space)
    g = aicb200.DeviceGroup(devices)
    g.update(space)
    lib = aicb200.load_library()

    host_out = {"colorbuf": np.empty((n, 4), np.float32), "depth": np.empty(n, np.float64),
                "hit": np.empty((n, 8), np.int32)}
    pinned_out = {"colorbuf": torch.empty((n, 4), dtype=torch.float32, pin_memory=True).numpy(),
                  "depth": torch.empty(n, dtype=torch.float64, pin_memory=True).numpy(),
                  "hit": torch.empty((n, 8), dtype=torch.int32, pin_memory=True).numpy()}
    dev_out = {"colorbuf": torch.empty((n, 4), dtype=torch.float32, device="cuda:0"),
               "depth": torch.empty(n, dtype=torch.float64, device="cuda:0"),
               "hit": torch.empty((n, 8), dtype=torch.int32, device="cuda:0")}
    o = opts.to_abi(True)

    def host_single(out=host_out):
        info = abi.RenderInfo()
        st = lib.aicb_render_colorbuf(r.rt.handle, C.byref(cam.data), C.byref(o), None,
                                      out["colorbuf"].ctypes.data, out["depth"].ctypes.data,
                                      out["hit"].ctypes.data, None, n, C.byref(info))
        assert st == abi.OK, lib.aicb_last_error()

    def device_single():
        r.draw_colorbuf(want_steps=False, device=True, out=dev_out).result()

    def host_group(out=host_out):
        info = abi.RenderInfo()
        st = lib.aicb_group_render_colorbuf(g.scene.handle, C.byref(cam.data), C.byref(o),
                                            out["colorbuf"].ctypes.data, out["depth"].ctypes.data,
                                            out["hit"].ctypes.data, None, n, C.byref(info))
        assert st == abi.OK, lib.aicb_last_error()

    def device_group():
        g.draw_colorbuf(cam, opts, want_steps=False, device=True, out=dev_out)
        torch.cuda.current_stream(0).synchronize()   # the outputs are final on the caller's stream

    arms = {"single_host": host_single, "single_host_pinned": lambda: host_single(pinned_out),
            "single_device": device_single,
            "group_host": host_group, "group_host_pinned": lambda: host_group(pinned_out), "group_device": device_group}
    times = {k: [] for k in arms}
    same = {}
    for step in range(args.warmup + args.steps):
        for name, fn in arms.items():
            flush.zero_()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            t1 = time.perf_counter()
            if step >= args.warmup:
                times[name].append((t1 - t0) * 1e3)
            if step == 0 and name.endswith("device"):
                host_name = name.replace("device", "host")
                arms[host_name]()
                same[name] = all(np.ascontiguousarray(dev_out[k].cpu().numpy()).tobytes() == host_out[k].tobytes()
                                 for k in dev_out)
    gpus = card()
    for name, t in times.items():
        t = np.array(t)
        print(json.dumps({"arm": name, "workload": desc, "pixels": n, "devices": devices if "group" in name else [0],
                          "median_ms": round(float(np.median(t)), 3), "p10_ms": round(float(np.percentile(t, 10)), 3),
                          "p90_ms": round(float(np.percentile(t, 90)), 3), "steps": len(t),
                          "outputs_equal_host": same.get(name), "gpus": gpus}))
    g.close()
    r.rt.close()


if __name__ == "__main__":
    main()
