"""ctypes wrapper over oracle_terminal/libtermorc.so — the desktop terminal's ColorCharacterBuf on the raytracer oracle
(TEST INFRASTRUCTURE: the checker, never the product)."""
import ctypes as C
import os
import subprocess

import numpy as np

import orc
from aicb200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "oracle_terminal", "libtermorc.so")

# the oracle's Exception numbering (oracle/aic_oracle.cpp); SURFACE = a hit on a block
SURFACE, ENTER_SPACE, SKY, BACKDROP, INCOMPLETE, PAINT, DEBUG_RG = -1, 0, 1, 2, 3, 4, 5

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    # built by __graft_entry__.build(); an existing library is loaded as it is
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle_terminal"), "-B"], check=True, capture_output=True)
    L = C.CDLL(LIB_PATH)
    L.orc_render_layers_terminal.restype = C.c_uint64
    L.orc_render_layers_terminal.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_void_p,
                                             C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_terminal_trace_samples.restype = C.c_uint64
    L.orc_terminal_trace_samples.argtypes = [C.c_void_p, C.POINTER(abi.Options), C.c_void_p, C.POINTER(abi.Options),
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                             C.c_void_p, C.c_void_p]
    L.orc_character_add.restype = None
    L.orc_character_add.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    L.orc_terminal_to_srgb8.restype = None
    L.orc_terminal_to_srgb8.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    L.orc_character_mean.restype = None
    L.orc_character_mean.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
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


def _rgba_arg(v):
    a = np.array(v, dtype=np.float32) if v is not None else None
    return a, (a.ctypes.data if a is not None else None)


def render_layers_terminal(world, ui, backdrop, no_world):
    """The terminal's frame.  world / ui = (termorc.Scene, Camera, GraphicsOptions) or None.  Returns a dict of text
    (int32 [H, W]), layer (int32 [H, W]), rgba (float32 [H, W, 4]) and cubes_traced."""
    lead = world if world else ui
    w, h = lead[1].data.fb_width, lead[1].data.fb_height
    rgba = np.zeros((h, w, 4), dtype=np.float32)
    text = np.zeros((h, w), dtype=np.int32)
    layer = np.zeros((h, w), dtype=np.int32)
    wh, wc, wo, _k1 = _parts(world)
    uh, uc, uo, _k2 = _parts(ui)
    _b, bp = _rgba_arg(backdrop)
    _nw, nwp = _rgba_arg(no_world)
    total = lib().orc_render_layers_terminal(wh, wc, wo, uh, uc, uo, bp, nwp, rgba.ctypes.data, text.ctypes.data,
                                             layer.ctypes.data)
    return {"text": text, "layer": layer, "rgba": rgba, "cubes_traced": int(total)}


def trace_samples(world, ui, backdrop, no_world, world_rays=None, ui_rays=None):
    """trace_ray_through_layers into a fresh ColorCharacterBuf per ray.  world / ui = (termorc.Scene, GraphicsOptions)
    or None; rays [n, 6] (origin, direction).  Returns dict of colorbuf [n, 4], text [n], layer [n], cubes_traced."""
    wr = None if world_rays is None else np.ascontiguousarray(world_rays, dtype=np.float64).reshape(-1, 6)
    ur = None if ui_rays is None else np.ascontiguousarray(ui_rays, dtype=np.float64).reshape(-1, 6)
    n = (wr if wr is not None else ur).shape[0]
    cb = np.zeros((n, 4), dtype=np.float32)
    text = np.zeros(n, dtype=np.int32)
    layer = np.zeros(n, dtype=np.int32)
    wo = world[1].to_abi(True) if world else None
    uo = ui[1].to_abi(True) if ui else None
    _b, bp = _rgba_arg(backdrop)
    _nw, nwp = _rgba_arg(no_world)
    total = lib().orc_terminal_trace_samples(world[0].handle if world else None, C.byref(wo) if wo else None,
                                             ui[0].handle if ui else None, C.byref(uo) if uo else None, bp, nwp,
                                             wr.ctypes.data if wr is not None else None,
                                             ur.ctypes.data if ur is not None else None, n, cb.ctypes.data,
                                             text.ctypes.data, layer.ctypes.data)
    return {"colorbuf": cb, "text": text, "layer": layer, "cubes_traced": int(total)}


def character_add(state, hits):
    """CharacterBuf::add of hits [(exception, block, layer)] in order, from state (text, layer)."""
    st = np.array(state, dtype=np.int32)
    ex = np.array([h[0] for h in hits], dtype=np.int32)
    bl = np.array([h[1] for h in hits], dtype=np.int32)
    ly = np.array([h[2] for h in hits], dtype=np.int32)
    lib().orc_character_add(st.ctypes.data, ex.ctypes.data, bl.ctypes.data, ly.ctypes.data, len(hits))
    return int(st[0]), int(st[1])


def character_mean(states):
    """CharacterBuf::mean of the (text, layer) states, in sample order."""
    s = np.ascontiguousarray(states, dtype=np.int32).reshape(-1, 2)
    out = np.zeros(2, dtype=np.int32)
    lib().orc_character_mean(s.ctypes.data, s.shape[0], out.ctypes.data)
    return int(out[0]), int(out[1])


def to_srgb8(rgba):
    """Rgba::to_srgb8 (color.rs:669-676) of post-processed linear RGBA [..., 4]: draw_rgba's encoder."""
    c = np.ascontiguousarray(rgba, dtype=np.float32).reshape(-1, 4)
    out = np.zeros((c.shape[0], 4), dtype=np.uint8)
    lib().orc_terminal_to_srgb8(c.ctypes.data, c.shape[0], out.ctypes.data)
    return out


LIBM_CR = orc.LIBM_CR
