"""ctypes wrapper over oracle_cursor/libcursororc.so — cursor_raycast and project_cursor on the raytracer oracle (TEST
INFRASTRUCTURE: the checker, never the product)."""
import ctypes as C
import os
import subprocess

import numpy as np

from aicb200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "oracle_cursor", "libcursororc.so")

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    # built by __graft_entry__.build(); an existing library is loaded as it is
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle_cursor"), "-B"], check=True, capture_output=True)
    L = C.CDLL(LIB_PATH)
    L.orc_cursor_scene_create.restype = C.c_void_p
    L.orc_cursor_scene_create.argtypes = [C.POINTER(abi.SceneDesc)]
    L.orc_cursor_scene_destroy.restype = None
    L.orc_cursor_scene_destroy.argtypes = [C.c_void_p]
    L.orc_cursor_raycast.restype = None
    L.orc_cursor_raycast.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.orc_project_cursor.restype = None
    L.orc_project_cursor.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.c_void_p, C.POINTER(abi.CameraData),
                                     C.c_void_p, C.c_size_t, C.c_double, C.c_void_p]
    _lib = L
    return L


class CursorScene:
    """The cursor oracle's scene of an aicb200.Space."""

    def __init__(self, space):
        desc, keep = space.to_desc()
        self.handle = C.c_void_p(lib().orc_cursor_scene_create(C.byref(desc)))
        del keep

    def __del__(self):
        try:
            if self.handle:
                lib().orc_cursor_scene_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def cursor_raycast(self, origin_dir, max_distance=None):
        """cursor_raycast for rays [n, 6]: an abi.CURSOR_DTYPE array."""
        od = np.ascontiguousarray(origin_dir, dtype=np.float64).reshape(-1, 6)
        n = od.shape[0]
        md = None if max_distance is None else np.ascontiguousarray(
            np.broadcast_to(np.asarray(max_distance, dtype=np.float64), (n,)))
        out = np.zeros(n, dtype=abi.CURSOR_DTYPE)
        lib().orc_cursor_raycast(self.handle, od.ctypes.data, None if md is None else md.ctypes.data, n,
                                 out.ctypes.data)
        return out


def project_cursor(world=None, ui=None, ndc=None, world_max_distance=6.0):
    """project_cursor: world / ui = (CursorScene, aicb200.Camera) or None; ndc [n, 2]."""
    p = np.ascontiguousarray(ndc, dtype=np.float64).reshape(-1, 2)
    out = np.zeros(p.shape[0], dtype=abi.CURSOR_DTYPE)
    lib().orc_project_cursor(world[0].handle if world else None, C.byref(world[1].data) if world else None,
                             ui[0].handle if ui else None, C.byref(ui[1].data) if ui else None, p.ctypes.data,
                             p.shape[0], float(world_max_distance), out.ctypes.data)
    return out


def same_bits(a, b):
    """Two abi.CURSOR_DTYPE arrays are byte for byte equal (f64s by their bits)."""
    return np.array_equal(np.asarray(a).reshape(-1).view(np.uint8), np.asarray(b).reshape(-1).view(np.uint8))
