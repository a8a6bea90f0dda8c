"""Times one tick of N characters' eyes on C2's 256^3 Space with light (one context, device 0), for N in --chars
(64, 1024 and 16384 by default).  Two ways to run the same tick:

  device chain   aicb_step_bodies_device, aicb_step_exposure_device, aicb_step_eyes_device, aicb_eye_views_device and
                 aicb_cursor_raycast_device at the look rays, all on the torch stream with no host wait;
  host trips     the same body, exposure and cursor device calls, with the eye work on the host as it was done
                 before the eye calls existed: download the bodies, step the eyes (numpy), build each eye-to-world
                 matrix (aicb_view_transform_matrix) and upload them, download the exposures, build each camera
                 (aicb_camera_from_view, Camera.set_measured_exposure's rule) and its look ray
                 (aicb_camera_project_ndc) and upload the camera table and the rays.  The per-eye host calls go
                 through ctypes, one call per eye, as a Python host makes them.

Before timing, both run three ticks from the same state and every output (bodies, exposure states, eyes, matrices,
camera table, cursors) is checked equal byte for byte.  Per tick: wall_ms, a host clock around the tick and a device
synchronise, and gpu_ms, CUDA events on the torch stream around it; medians over --steps ticks after --warmup.  Prints
one JSON line per workload and a last line with the GPU's name and power limit read in the same run.

    python tools/eyes_bench.py --steps 9 --warmup 2
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import aicb200  # noqa: E402
from aicb200 import GraphicsOptions, SpaceRaytracer, Viewport, abi, scenes  # noqa: E402
import eyeorc  # noqa: E402
from cursor_bench import run  # noqa: E402
from texture_bench import gpu_identity  # noqa: E402

DT = 1.0 / 20.0
GRAVITY = (0.0, -20.0, 0.0)
OPTS = GraphicsOptions(exposure=aicb200.EXPOSURE_AUTOMATIC)
VIEWPORT = Viewport.with_scale(1.0, (128, 96))


class Tick:
    """N characters' state on the device, and the two ways to step it by one tick."""

    def __init__(self, torch, dev, rt, space, n, seed):
        self.torch, self.dev, self.rt, self.n = torch, dev, rt, n
        rng = np.random.default_rng(seed)
        lo, size = np.array(space.lower, np.float64), np.array(space.size, np.float64)
        b = aicb200.bodies(n, position=lo + size * rng.uniform(0.1, 0.9, (n, 3)),
                           collision_box=(-0.3, -0.8, -0.3, 0.3, 0.9, 0.3), velocity=rng.normal(size=(n, 3)) * 4.0,
                           flying=rng.random(n) < 0.5)
        rot = np.array([aicb200.look_rotation(y, p) for y, p in zip(rng.uniform(0, 360, n), rng.uniform(-60, 60, n))])
        u8 = lambda a: torch.from_numpy(a.view(np.uint8).reshape(n, a.dtype.itemsize).copy()).to(dev)  # noqa: E731
        self.bodies = u8(b)
        self.eyes = u8(aicb200.eyes(n))
        self.states = u8(aicb200.exposure_states(n))
        self.m = torch.zeros((n, 16), dtype=torch.float64, device=dev)
        self.table = u8(aicb200.eye_cameras(n, OPTS, VIEWPORT))
        self.rays = torch.zeros((n, 6), dtype=torch.float64, device=dev)
        self.rot_host = rot
        self.rot = torch.from_numpy(rot).to(dev)
        self.params = aicb200.eye_view_params(OPTS, VIEWPORT)
        self.cursor = None
        self.lib = aicb200.load_library()

    def clone(self):
        c = Tick.__new__(Tick)
        c.__dict__.update(self.__dict__)
        for k in ("bodies", "eyes", "states", "m", "table", "rays"):
            setattr(c, k, getattr(self, k).clone())
        return c

    def device(self):
        rt = self.rt
        rt.step_bodies(self.bodies, DT, GRAVITY, max_contacts=0, device=True)
        _, exposures = rt.step_exposure(self.states, self.m, DT, device=True)
        rt.step_eyes(self.eyes, self.bodies, DT)
        rt.eye_views(self.eyes, self.bodies, self.rot, exposures, self.params, self.m, self.table, self.rays)
        self.cursor = rt.cursor_raycast(self.rays, 6.0, device=True)

    def host(self):
        torch, rt, n, lib, p = self.torch, self.rt, self.n, self.lib, self.params
        rt.step_bodies(self.bodies, DT, GRAVITY, max_contacts=0, device=True)
        bodies = self.bodies.cpu().numpy().view(abi.BODY_DTYPE).reshape(n)          # device-to-host read 1
        _, exposures = rt.step_exposure(self.states, self.m, DT, device=True)
        exposures = exposures.cpu().numpy()                                            # device-to-host read 2
        eyes = eyeorc.step(self.eyes.cpu().numpy().view(abi.EYE_DTYPE).reshape(n), bodies, DT)
        t = eyeorc.eye_translation(eyes, bodies)
        m = np.empty((n, 16))
        table = self.table.cpu().numpy().view(abi.CAMERA_DTYPE).reshape(n).copy()
        rays = np.empty((n, 6))
        cam, out6, out16 = abi.CameraData(), (C.c_double * 6)(), (C.c_double * 16)()
        automatic_none = p.automatic_exposure and p.lighting_display == aicb200.LIGHT_NONE
        for i in range(n):
            q, tr = (C.c_double * 4)(*self.rot_host[i]), (C.c_double * 3)(*t[i])
            lib.aicb_view_transform_matrix(q, tr, out16)
            m[i] = out16[:]
            v = float(exposures[i])
            e = table["exposure"][i]
            if not p.automatic_exposure:
                e = p.fixed_exposure
            elif not (v != v or v < 0.0):
                e = 1.0 if automatic_none else abs(v)
            lib.aicb_camera_from_view(q, tr, p.fov_y_degrees, p.view_distance, p.nominal_width, p.nominal_height,
                                      p.fb_width, p.fb_height, e, C.byref(cam))
            table[i] = np.frombuffer(bytes(cam), abi.CAMERA_DTYPE)[0]
            lib.aicb_camera_project_ndc(C.byref(cam), 0.0, 0.0, out6)
            rays[i] = out6[:]
        self.eyes.copy_(torch.from_numpy(eyes.view(np.uint8).reshape(n, 72)))
        self.m.copy_(torch.from_numpy(m))
        self.table.copy_(torch.from_numpy(table.view(np.uint8).reshape(n, 144)))
        self.rays.copy_(torch.from_numpy(rays))
        self.cursor = rt.cursor_raycast(self.rays, 6.0, device=True)

    def outputs(self):
        return [t.cpu().numpy().tobytes() for t in (self.bodies, self.states, self.eyes, self.m, self.table,
                                                    self.rays, self.cursor)]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=9)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--chars", default="64,1024,16384")
    args = p.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    space = scenes.config_c2(n=256, seed=3, with_light=True)
    space.light_max_distance = 20
    rt = SpaceRaytracer(space, GraphicsOptions())
    for n in (int(v) for v in args.chars.split(",")):
        a = Tick(torch, dev, rt, space, n, seed=n)
        b = a.clone()
        for _ in range(3):
            a.device()
            b.host()
        names = ("bodies", "exposure states", "eyes", "eye_to_world", "cameras", "look rays", "cursors")
        for name, x, y in zip(names, a.outputs(), b.outputs()):
            assert x == y, f"{n} characters: the device chain's {name} differ from the host calls'"
        run(torch, dev, f"device chain {n}", a.device, args.steps, args.warmup, lambda w, g: {"characters": n})
        run(torch, dev, f"host trips {n}", b.host, args.steps, args.warmup, lambda w, g: {"characters": n})
    print(json.dumps({"gpu": gpu_identity()}), flush=True)
    rt.close()


if __name__ == "__main__":
    main()
