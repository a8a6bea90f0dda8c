"""Where a shading round's cycles go: clock64 around each phase of shade_hit<LC_INTERP> on a bench frame.

  python tools/shade_phases.py [--workload c2] [--frames 20]

Builds the library a second time, with AICB_SHADE_PHASES defined, into a temporary directory (the timed library is not
touched), renders the workload's frames as tools/stage_times.py does, and prints the mean cycles per shaded hit of each
phase.  A warp shades its 32 queued hits in lockstep, so a phase's mean per hit is also its share of a 32-slot round.
A load's latency shows up in the phase that first uses its value.  The timers and the per-hit atomics that collect them
slow the kernel down, so the phases are a split of the round, not the timed kernel's round.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

# g_shade_phase[0..6]: the phases of shade_hit, in order; 7..9 are taken around it in shade_kernel
SHADE_PHASE_NAMES = ("record loads", "decode", "transmittance pow", "fog exp", "f64 geometry + ray loads",
                     "texel gather", "colour")


def build_phase_library(out_dir):
    import __graft_entry__ as g
    pkg = g.PKG
    srcs = [os.path.join(pkg, "csrc", f) for f in ("aicb200.cu", "light.cu", "group.cu")]
    srcs.append(os.path.join(pkg, "host", "camera.cpp"))
    lib = os.path.join(out_dir, "libaicb200_phases.so")
    r = subprocess.run([g.NVCC] + g.NVCC_FLAGS + ["-DAICB_SHADE_PHASES", "-o", lib] + srcs, capture_output=True,
                       text=True)
    if r.returncode != 0:
        raise SystemExit("nvcc failed:\n" + r.stdout + r.stderr)
    return lib


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--workload", default="c2")
    p.add_argument("--frames", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    args = p.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        os.environ["AICB200_LIB"] = build_phase_library(tmp)
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("shade_phases.py: no CUDA device")
        import bench
        import stage_times
        import aicb200
        from aicb200 import abi, scenes
        lib = aicb200.load_library()
        lib.aicb_debug_shade_phases.argtypes = [C.POINTER(C.c_ulonglong)]
        lib.aicb_debug_shade_phases.restype = C.c_int
        dev = stage_times.card()
        print(f"card: {dev['name']}, power limit {dev['power_limit']}, max SM clock {dev['sm_max']}")

        space, opts, w, h, desc = bench.make_workload(args.workload)
        cam = scenes.standard_camera(space, opts, w, h)
        ctx = aicb200.Context(0)
        rt = aicb200.SpaceRaytracer(space, opts, ctx)
        o_abi = opts.to_abi(True)
        shard = abi.Shard(bench.STRIP_ROWS, 0, 1)
        n = lib.aicb_shard_pixel_count(C.byref(cam.data), C.byref(shard))
        out = torch.empty((n, 4), dtype=torch.uint8).pin_memory()
        sums = (C.c_ulonglong * 10)()
        for k in range(args.warmup + args.frames):
            if k == args.warmup and lib.aicb_debug_shade_phases(sums) != 0:
                raise SystemExit("aicb_debug_shade_phases failed")
            if lib.aicb_render_srgb8(rt.handle, C.byref(cam.data), C.byref(o_abi), C.byref(shard), out.data_ptr(),
                                     n, None) != 0:
                raise SystemExit(lib.aicb_last_error().decode())
        if lib.aicb_debug_shade_phases(sums) != 0:
            raise SystemExit("aicb_debug_shade_phases failed")
        hits = sums[9]
        if hits == 0:
            raise SystemExit(f"{args.workload}: no hit was shaded by shade_kernel<LC_INTERP>")
        print(f"{args.workload} ({desc}): {hits / args.frames:.0f} shaded hits per frame; mean cycles per hit:")
        for name, v in zip(SHADE_PHASE_NAMES, sums[:7]):
            print(f"  {name:28s} {v / hits:8.0f}")
        print(f"  {'store':28s} {sums[7] / hits:8.0f}")
        print(f"  {'whole hit (shade_hit + store)':28s} {sums[8] / hits:8.0f}")


if __name__ == "__main__":
    main()
