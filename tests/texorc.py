"""ctypes wrapper over oracle_texture/libtexorc.so — RaytraceToTexture's Split on the raytracer oracle (TEST
INFRASTRUCTURE: the checker, never the product)."""
import ctypes as C
import os
import subprocess

import numpy as np

import orc
from aicb200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "oracle_texture", "libtexorc.so")

LAYER_NONE, LAYER_WORLD, LAYER_UI = 0, 1, -1

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    # built by __graft_entry__.build(); an existing library is loaded as it is
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle_texture"), "-B"], check=True, capture_output=True)
    L = C.CDLL(LIB_PATH)
    L.orc_render_layers_texture.restype = C.c_uint64
    L.orc_render_layers_texture.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_void_p,
                                            C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.orc_texture_trace_samples.restype = C.c_uint64
    L.orc_texture_trace_samples.argtypes = [C.c_void_p, C.POINTER(abi.Options), C.c_void_p, C.POINTER(abi.Options),
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                            C.c_void_p, C.c_void_p]
    L.orc_texture_mean_and_store.restype = None
    L.orc_texture_mean_and_store.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_float,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_f16_from_f32.restype = C.c_uint16
    L.orc_f16_from_f32.argtypes = [C.c_float]
    L.orc_texture_monotonic_violations.restype = C.c_uint64
    L.orc_set_libm.argtypes = [C.c_int]
    L.orc_set_libm.restype = None
    L.orc_scene_create.restype = C.c_void_p
    L.orc_scene_create.argtypes = [C.POINTER(abi.SceneDesc)]
    L.orc_scene_destroy.argtypes = [C.c_void_p]
    L.orc_scene_destroy.restype = None
    _lib = L
    return L


def set_libm(mode):
    """As orc.set_libm, for the copy of the raytracer oracle inside this library."""
    lib().orc_set_libm(int(mode))


class Scene:
    """The raytracer oracle's scene, created in this library (its copy of the oracle has its own scene type)."""

    def __init__(self, space):
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


def _parts(layer):
    if not layer:
        return None, None, None, None
    o = layer[2].to_abi(True)
    return layer[0].handle, C.byref(layer[1].data), C.byref(o), o


def render_layers_texture(world, ui, backdrop, no_world, depth_transform, pixels=None):
    """trace_one for each pixel (raytrace_to_texture.rs:591-683).  world / ui = (texorc.Scene, Camera,
    GraphicsOptions) or None.  Returns (rgba16f bits uint16 [n, 4], depth float32 [n], cubes_traced)."""
    lead = world if world else ui
    w, h = lead[1].data.fb_width, lead[1].data.fb_height
    plist = None if pixels is None else np.ascontiguousarray(pixels, dtype=np.uint32).reshape(-1)
    n = w * h if plist is None else plist.size
    rgba = np.zeros((n, 4), dtype=np.uint16)
    depth = np.zeros(n, dtype=np.float32)
    wh, wc, wo, _k1 = _parts(world)
    uh, uc, uo, _k2 = _parts(ui)
    b = np.array(backdrop, dtype=np.float32) if backdrop is not None else None
    nw = np.array(no_world, dtype=np.float32) if no_world is not None else None
    m = np.ascontiguousarray(depth_transform, dtype=np.float64).reshape(16)
    total = lib().orc_render_layers_texture(wh, wc, wo, uh, uc, uo, b.ctypes.data if b is not None else None,
                                            nw.ctypes.data if nw is not None else None, m.ctypes.data,
                                            plist.ctypes.data if plist is not None else None, n, rgba.ctypes.data,
                                            depth.ctypes.data)
    return rgba, depth, int(total)


def trace_samples(world, ui, backdrop, no_world, world_rays=None, ui_rays=None):
    """trace_ray_through_layers into a fresh Split per ray.  world / ui = (texorc.Scene, GraphicsOptions) or None;
    rays [n, 6] (origin, direction).  Returns dict of colorbuf [n, 4], depth [n], layer [n], cubes_traced."""
    wr = None if world_rays is None else np.ascontiguousarray(world_rays, dtype=np.float64).reshape(-1, 6)
    ur = None if ui_rays is None else np.ascontiguousarray(ui_rays, dtype=np.float64).reshape(-1, 6)
    n = (wr if wr is not None else ur).shape[0]
    cb = np.zeros((n, 4), dtype=np.float32)
    depth = np.zeros(n, dtype=np.float64)
    layer = np.zeros(n, dtype=np.int32)
    wo = world[1].to_abi(True) if world else None
    uo = ui[1].to_abi(True) if ui else None
    b = np.array(backdrop, dtype=np.float32) if backdrop is not None else None
    nw = np.array(no_world, dtype=np.float32) if no_world is not None else None
    total = lib().orc_texture_trace_samples(world[0].handle if world else None, C.byref(wo) if wo else None,
                                            ui[0].handle if ui else None, C.byref(uo) if uo else None,
                                            b.ctypes.data if b is not None else None,
                                            nw.ctypes.data if nw is not None else None,
                                            wr.ctypes.data if wr is not None else None,
                                            ur.ctypes.data if ur is not None else None, n, cb.ctypes.data,
                                            depth.ctypes.data, layer.ctypes.data)
    return {"colorbuf": cb, "depth": depth, "layer": layer, "cubes_traced": int(total)}


def mean_and_store(colorbuf, depth, layer, exposure_world, exposure_ui, depth_transform):
    """Split::mean of the given samples and trace_one's stores: (rgba16f bits [4], depth f32, layer)."""
    cb = np.ascontiguousarray(colorbuf, dtype=np.float32).reshape(-1, 4)
    d = np.ascontiguousarray(depth, dtype=np.float64)
    l = np.ascontiguousarray(layer, dtype=np.int32)
    m = np.ascontiguousarray(depth_transform, dtype=np.float64).reshape(16)
    rgba = np.zeros(4, dtype=np.uint16)
    out_d = np.zeros(1, dtype=np.float32)
    out_l = np.zeros(1, dtype=np.int32)
    lib().orc_texture_mean_and_store(cb.ctypes.data, d.ctypes.data, l.ctypes.data, cb.shape[0], exposure_world,
                                     exposure_ui, m.ctypes.data, rgba.ctypes.data, out_d.ctypes.data, out_l.ctypes.data)
    return rgba, out_d[0], int(out_l[0])


def f16_bits(v):
    return int(lib().orc_f16_from_f32(float(v)))


def monotonic_violations():
    return int(lib().orc_texture_monotonic_violations())


LIBM_CR = orc.LIBM_CR
