"""ctypes wrapper over oracle/liborc.so — TEST INFRASTRUCTURE (the checker, never the product)."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "oracle", "liborc.so")

from aicb200 import abi  # noqa: E402  (conftest puts the package on sys.path)

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    # built (and rebuilt when its sources change) by __graft_entry__.build_oracle(), which the test session runs first;
    # an existing library is loaded as it is, so bench.py also runs from a read-only tree
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-B"], check=True, capture_output=True)
    L = C.CDLL(LIB_PATH)
    L.orc_scale_to_integer_step.restype = C.c_double
    L.orc_scale_to_integer_step.argtypes = [C.c_double, C.c_double]
    L.orc_raycast.restype = C.c_int
    L.orc_raycast.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_recursive_raycast.restype = C.c_int
    L.orc_recursive_raycast.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_void_p]
    L.orc_apply_transmittance.argtypes = [C.c_void_p, C.c_float, C.c_void_p]
    L.orc_apply_transmittance.restype = None
    L.orc_packed_light_lut.restype = C.c_float
    L.orc_packed_light_lut.argtypes = [C.c_int]
    L.orc_packed_light_scalar_in.restype = C.c_int
    L.orc_packed_light_scalar_in.argtypes = [C.c_float]
    L.orc_to_srgb8.argtypes = [C.c_void_p, C.c_float, C.c_int, C.c_float, C.c_void_p]
    L.orc_to_srgb8.restype = None
    L.orc_scene_create.restype = C.c_void_p
    L.orc_scene_create.argtypes = [C.POINTER(abi.SceneDesc)]
    L.orc_scene_destroy.argtypes = [C.c_void_p]
    L.orc_scene_destroy.restype = None
    L.orc_surface_steps.restype = C.c_int
    L.orc_surface_steps.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.orc_trace_rays.restype = C.c_int
    L.orc_trace_rays.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(abi.Options), C.c_int, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_render.restype = C.c_uint64
    L.orc_render.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.POINTER(abi.Shard),
                             C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_render_rows.restype = C.c_uint64
    L.orc_render_rows.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_uint32,
                                  C.c_uint32, C.c_int, C.c_void_p, C.c_void_p]
    L.orc_render_rowlist.restype = C.c_uint64
    L.orc_render_rowlist.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_void_p,
                                     C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    L.orc_render_layers.restype = C.c_uint64
    L.orc_render_layers.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_void_p,
                                    C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p]
    L.orc_colorbuf_to_srgb8.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    L.orc_colorbuf_to_srgb8.restype = None
    L.orc_pixel_ray.argtypes = [C.POINTER(abi.CameraData), C.c_uint32, C.c_uint32, C.c_int, C.c_void_p]
    L.orc_pixel_ray.restype = None
    L.orc_hardware_threads.restype = C.c_int
    L.orc_set_libm.argtypes = [C.c_int]
    L.orc_set_libm.restype = None
    L.orc_get_libm.restype = C.c_int
    L.orc_powf.restype = C.c_float
    L.orc_powf.argtypes = [C.c_float, C.c_float, C.c_int]
    L.orc_expf.restype = C.c_float
    L.orc_expf.argtypes = [C.c_float, C.c_int]
    L.orc_light_chart.restype = C.c_size_t
    L.orc_light_chart.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_light_create.restype = C.c_void_p
    L.orc_light_create.argtypes = [C.POINTER(abi.SceneDesc)]
    L.orc_light_destroy.argtypes = [C.c_void_p]
    L.orc_light_fast_evaluate.argtypes = [C.c_void_p]
    L.orc_light_set_cubes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    L.orc_light_evaluate.restype = C.c_uint64
    L.orc_light_evaluate.argtypes = [C.c_void_p, C.c_uint8, C.c_uint64, C.c_void_p]
    L.orc_light_compute.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.orc_light_get.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_light_compute_by_chains.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_uint32, C.c_void_p, C.c_uint32]
    L.orc_light_evaluate_threaded.restype = C.c_uint64
    L.orc_light_evaluate_threaded.argtypes = [C.c_void_p, C.c_uint8, C.c_uint64, C.c_int, C.c_void_p]
    L.orc_light_compute_raw.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.orc_light_set_field.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_light_get_outside.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_light_set_pop_order.argtypes = [C.c_void_p, C.c_int]
    L.orc_light_queue_len.restype = C.c_size_t
    L.orc_light_queue_len.argtypes = [C.c_void_p]
    L.orc_light_queue_peek.restype = C.c_int
    L.orc_light_queue_peek.argtypes = [C.c_void_p]
    L.orc_light_node_visits.restype = C.c_uint64
    L.orc_light_node_visits.argtypes = [C.c_void_p]
    _lib = L
    return L


LIBM_PLATFORM, LIBM_CR = 0, 1


def set_libm(mode):
    """How the oracle evaluates f32::powf (raytracer_components.rs:233) and f32::exp (sr.rs:751): LIBM_PLATFORM = glibc
    powf / expf (what Rust's std calls on this host), LIBM_CR = correctly rounded (what the CUDA path does)."""
    lib().orc_set_libm(int(mode))


def get_libm():
    return int(lib().orc_get_libm())


FACES = ["Within", "NX", "NY", "NZ", "PX", "PY", "PZ"]


def scale_to_integer_step(s, ds):
    return lib().orc_scale_to_integer_step(s, ds)


def raycast(origin, direction, bounds=None, include_exit=True, max_steps=64):
    """Returns list of (cube(x,y,z), face_name, t, point(x,y,z)). bounds = (lo3, hi3) exclusive."""
    o = np.array(origin, dtype=np.float64)
    d = np.array(direction, dtype=np.float64)
    cf = np.zeros((max_steps, 4), dtype=np.int32)
    t = np.zeros(max_steps, dtype=np.float64)
    p = np.zeros((max_steps, 3), dtype=np.float64)
    b = None
    if bounds is not None:
        b = np.array(list(bounds[0]) + list(bounds[1]), dtype=np.int32)
    n = lib().orc_raycast(o.ctypes.data, d.ctypes.data, b.ctypes.data if b is not None else None,
                          1 if include_exit else 0, max_steps, cf.ctypes.data, t.ctypes.data, p.ctypes.data)
    return [(tuple(int(v) for v in cf[i, :3]), FACES[cf[i, 3]], float(t[i]), tuple(float(v) for v in p[i]))
            for i in range(n)]


def recursive_raycast(origin, direction, nth, resolution, bounds, max_steps=64):
    o = np.array(origin, dtype=np.float64)
    d = np.array(direction, dtype=np.float64)
    b = np.array(list(bounds[0]) + list(bounds[1]), dtype=np.int32)
    sub = np.zeros(6, dtype=np.float64)
    cf = np.zeros((max_steps, 4), dtype=np.int32)
    t = np.zeros(max_steps, dtype=np.float64)
    n = lib().orc_recursive_raycast(o.ctypes.data, d.ctypes.data, nth, resolution, b.ctypes.data, max_steps,
                                    sub.ctypes.data, cf.ctypes.data, t.ctypes.data)
    steps = [(tuple(int(v) for v in cf[i, :3]), FACES[cf[i, 3]], float(t[i])) for i in range(max(n, 0))]
    return sub, steps


def apply_transmittance(rgba, thickness):
    c = np.array(rgba, dtype=np.float32)
    out = np.zeros(5, dtype=np.float32)
    lib().orc_apply_transmittance(c.ctypes.data, thickness, out.ctypes.data)
    return tuple(float(v) for v in out[:4]), float(out[4])


def to_srgb8(colorbuf, exposure=1.0, tone_mapping=0, maximum_intensity=float("inf")):
    c = np.array(colorbuf, dtype=np.float32)
    out = np.zeros(4, dtype=np.uint8)
    lib().orc_to_srgb8(c.ctypes.data, exposure, tone_mapping, maximum_intensity, out.ctypes.data)
    return tuple(int(v) for v in out)


class OracleScene:
    def __init__(self, space):
        self.space = space
        desc, keep = space.to_desc()
        self.handle = lib().orc_scene_create(C.byref(desc))
        del keep

    def __del__(self):
        try:
            if self.handle:
                lib().orc_scene_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def surface_steps(self, origin_dir, depth_iter=False, max_steps=64):
        od = np.array(origin_dir, dtype=np.float64)
        rec = np.zeros((max_steps, 18), dtype=np.float64)
        n = lib().orc_surface_steps(self.handle, od.ctypes.data, 1 if depth_iter else 0, max_steps, rec.ctypes.data)
        return rec[:n]

    def trace_rays(self, origin_dir, options, include_sky=True, accum_mode=0):
        od = np.ascontiguousarray(origin_dir, dtype=np.float64).reshape(-1, 6)
        n = od.shape[0]
        cb = np.empty((n, 4), dtype=np.float32)
        depth = np.empty(n, dtype=np.float64)
        hit = np.empty((n, 8), dtype=np.int32)
        steps = np.empty(n, dtype=np.uint32)
        text = np.empty(n, dtype=np.int32)
        opt = options.to_abi(include_sky)
        lib().orc_trace_rays(self.handle, od.ctypes.data, n, C.byref(opt), accum_mode, cb.ctypes.data,
                             depth.ctypes.data, hit.ctypes.data, steps.ctypes.data, text.ctypes.data)
        return {"colorbuf": cb, "depth": depth, "hit": hit, "steps": steps, "text": text}

    def render(self, camera, options, shard=None, accum_mode=0, n_threads=0):
        cam = camera.data
        s = None
        rows = cam.fb_height
        if shard is not None:
            s = abi.Shard()
            s.strip_rows, s.index, s.count = shard
            sr = max(1, shard[0])
            rows = sum(1 for y in range(cam.fb_height) if (y // sr) % shard[2] == shard[1]) if shard[2] > 1 else rows
        n = cam.fb_width * rows
        srgb = np.empty((n, 4), dtype=np.uint8)
        cb = np.empty((n, 4), dtype=np.float32)
        depth = np.empty(n, dtype=np.float64)
        hit = np.empty((n, 8), dtype=np.int32)
        steps = np.empty(n, dtype=np.uint32)
        text = np.empty(n, dtype=np.int32)
        opt = options.to_abi(True)
        total = lib().orc_render(self.handle, C.byref(cam), C.byref(opt), C.byref(s) if s else None, accum_mode,
                                 n_threads, srgb.ctypes.data, cb.ctypes.data, depth.ctypes.data, hit.ctypes.data,
                                 steps.ctypes.data, text.ctypes.data)
        return {"srgb8": srgb, "colorbuf": cb, "depth": depth, "hit": hit, "steps": steps, "text": text,
                "cubes_traced": int(total)}

    def render_rows(self, camera, options, row_begin, row_end, n_threads=0, want_colorbuf=False):
        cam = camera.data
        n = cam.fb_width * (row_end - row_begin)
        srgb = np.empty((n, 4), dtype=np.uint8)
        cb = np.empty((n, 4), dtype=np.float32) if want_colorbuf else None
        opt = options.to_abi(True)
        total = lib().orc_render_rows(self.handle, C.byref(cam), C.byref(opt), row_begin, row_end, n_threads,
                                      srgb.ctypes.data, cb.ctypes.data if want_colorbuf else None)
        return {"srgb8": srgb, "colorbuf": cb, "cubes_traced": int(total)}


def render_rowlist(scene, camera, options, rows, n_threads=0, want_colorbuf=False):
    """Renders the given framebuffer rows (any order) with all host threads; outputs packed in list order."""
    cam = camera.data
    rows = np.ascontiguousarray(rows, dtype=np.uint32)
    n = cam.fb_width * len(rows)
    srgb = np.empty((n, 4), dtype=np.uint8)
    cb = np.empty((n, 4), dtype=np.float32) if want_colorbuf else None
    opt = options.to_abi(True)
    total = lib().orc_render_rowlist(scene.handle, C.byref(cam), C.byref(opt), rows.ctypes.data, len(rows), n_threads,
                                     srgb.ctypes.data, cb.ctypes.data if want_colorbuf else None)
    return {"srgb8": srgb, "colorbuf": cb, "cubes_traced": int(total)}


def pixel_ray(camera, x, y, sample=-1):
    out = np.zeros(6, dtype=np.float64)
    lib().orc_pixel_ray(C.byref(camera.data), x, y, sample, out.ctypes.data)
    return out


def hardware_threads():
    return lib().orc_hardware_threads()


def render_layers(world, ui, backdrop=None, no_world=None):
    """draw_rgba through the layers (renderer.rs:454-478).  world / ui = (OracleScene, Camera, GraphicsOptions) or None."""
    lead = world if world else ui
    cam = lead[1].data
    n = cam.fb_width * cam.fb_height
    srgb = np.empty((n, 4), dtype=np.uint8)
    cb = np.empty((n, 4), dtype=np.float32)

    def parts(layer):
        if not layer:
            return None, None, None
        return layer[0].handle, C.byref(layer[1].data), C.byref(layer[2].to_abi(True))

    wh, wc, wo = parts(world)
    uh, uc, uo = parts(ui)
    b = np.array(backdrop, dtype=np.float32) if backdrop is not None else None
    nw = np.array(no_world, dtype=np.float32) if no_world is not None else None
    total = lib().orc_render_layers(wh, wc, wo, uh, uc, uo, b.ctypes.data if b is not None else None,
                                    nw.ctypes.data if nw is not None else None, srgb.ctypes.data, cb.ctypes.data)
    return {"srgb8": srgb, "colorbuf": cb, "cubes_traced": int(total)}


def colorbuf_to_srgb8(cb):
    c = np.ascontiguousarray(cb, dtype=np.float32).reshape(-1, 4)
    out = np.empty((c.shape[0], 4), dtype=np.uint8)
    lib().orc_colorbuf_to_srgb8(c.ctypes.data, c.shape[0], out.ctypes.data)
    return out


def ulp_diff(a, b):
    """Elementwise distance in units-in-the-last-place between two float32 arrays."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    d = np.abs(ia - ib)
    both_nan = np.isnan(a) & np.isnan(b)
    return np.where(both_nan, 0, d)


def max_ulp_diff(a, b):
    return int(ulp_diff(a, b).max()) if np.size(a) else 0


def light_chart():
    n = lib().orc_light_chart(None, None)
    w = np.zeros((n, 6), dtype=np.float32)
    ch = np.zeros((n, 6), dtype=np.uint32)
    lib().orc_light_chart(w.ctypes.data, ch.ctypes.data)
    return w, ch


class OracleLight:
    """Light propagation oracle over a Space (space/light/updater.rs restatement)."""

    def __init__(self, space):
        self.space = space
        desc, keep = space.to_desc()
        self.handle = lib().orc_light_create(C.byref(desc))
        del keep
        self.shape = space.size

    def __del__(self):
        try:
            if self.handle:
                lib().orc_light_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def set_pop_order(self, order):
        lib().orc_light_set_pop_order(self.handle, order)

    def fast_evaluate(self):
        lib().orc_light_fast_evaluate(self.handle)

    def set_cubes(self, cubes, ids):
        c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
        i = np.ascontiguousarray(ids, dtype=np.uint16)
        lib().orc_light_set_cubes(self.handle, c.ctypes.data, i.ctypes.data, c.shape[0])

    def evaluate(self, epsilon=0, max_updates=2**62):
        md = C.c_uint8(0)
        n = lib().orc_light_evaluate(self.handle, epsilon, max_updates, C.byref(md))
        return int(n), int(md.value)

    def compute(self, cubes):
        c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
        out = np.zeros((c.shape[0], 4), dtype=np.uint8)
        lib().orc_light_compute(self.handle, c.ctypes.data, c.shape[0], out.ctypes.data)
        return out

    def compute_by_chains(self, cubes, preorder, chains, euler):
        """compute_light evaluated chain by chain with the terms added in the Euler tour of the chain tree — the CUDA
        chain walk's algorithm on the CPU, with the product library's chain tables."""
        c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
        out = np.zeros((c.shape[0], 4), dtype=np.uint8)
        raw = np.zeros((c.shape[0], 4), dtype=np.float32)
        pre = np.ascontiguousarray(preorder, dtype=np.uint32)
        chn = np.ascontiguousarray(chains, dtype=np.uint32)
        eul = np.ascontiguousarray(euler, dtype=np.uint16)
        lib().orc_light_compute_by_chains(self.handle, c.ctypes.data, c.shape[0], out.ctypes.data, raw.ctypes.data, pre.ctypes.data,
                                          chn.ctypes.data, chn.shape[0], eul.ctypes.data, eul.shape[0])
        return out, raw

    def evaluate_threaded(self, epsilon, n_threads, max_updates=(1 << 62)):
        """update_light_from_queue with the reference's `auto-threads` batches (32 cubes computed in parallel from the
        same stored light, applied in pop order); returns (updates, max difference)."""
        md = C.c_uint8(0)
        n = lib().orc_light_evaluate_threaded(self.handle, epsilon, max_updates, n_threads, C.byref(md))
        return int(n), int(md.value)

    def compute_raw(self, cubes):
        """compute_light: the packed results and the unquantised accumulators (incoming_light rgb, total_rays)."""
        c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
        out = np.zeros((c.shape[0], 4), dtype=np.uint8)
        raw = np.zeros((c.shape[0], 4), dtype=np.float32)
        lib().orc_light_compute_raw(self.handle, c.ctypes.data, c.shape[0], out.ctypes.data, raw.ctypes.data)
        return out, raw

    def field(self):
        out = np.zeros(self.shape + (4,), dtype=np.uint8)
        lib().orc_light_get(self.handle, out.ctypes.data)
        return out

    def set_field(self, field):
        f = np.ascontiguousarray(field, dtype=np.uint8)
        lib().orc_light_set_field(self.handle, f.ctypes.data)

    def get(self, cube):
        c = np.array(cube, dtype=np.int32)
        out = np.zeros(4, dtype=np.uint8)
        lib().orc_light_get_outside(self.handle, c.ctypes.data, out.ctypes.data)
        return tuple(int(v) for v in out)

    def queue_len(self):
        return int(lib().orc_light_queue_len(self.handle))

    def queue_peek(self):
        return int(lib().orc_light_queue_peek(self.handle))
