"""ctypes wrapper of orc_light_compute_debug in oracle_light/liblightorc.so (TEST INFRASTRUCTURE: the checker, never the
product): Space::compute_light::<LightUpdateCubeInfo> (space.rs:810, space/light/debug.rs) on the light oracle."""
import ctypes as C

import numpy as np

import lightorc
from aicb200 import LIGHT_RAY_DTYPE


def _lib():
    L = lightorc.lib()
    L.orc_light_compute_debug.restype = C.c_size_t
    L.orc_light_compute_debug.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_size_t, C.c_void_p]
    L.orc_light_compute.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    return L


def compute(oracle: lightorc.LightOracle, cubes):
    """orc_light_compute (compute_light's texels) on the same oracle."""
    c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
    out = np.zeros((c.shape[0], 4), dtype=np.uint8)
    _lib().orc_light_compute(oracle.handle, c.ctypes.data, c.shape[0], out.ctypes.data)
    return out


def compute_debug(oracle: lightorc.LightOracle, cubes):
    """-> (texels [n,4] uint8, rays, nodes): per cube an array of LIGHT_RAY_DTYPE in the order the walk pushes them, and
    the preorder index of the chart node each ray was struck at."""
    L = _lib()
    c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
    n = c.shape[0]
    texels = np.zeros((n, 4), dtype=np.uint8)
    counts = np.zeros(n, dtype=np.uint32)
    total = L.orc_light_compute_debug(oracle.handle, c.ctypes.data, n, texels.ctypes.data, None, None, 0,
                                      counts.ctypes.data)
    rays = np.zeros(total, dtype=LIGHT_RAY_DTYPE)
    nodes = np.zeros(total, dtype=np.uint32)
    L.orc_light_compute_debug(oracle.handle, c.ctypes.data, n, texels.ctypes.data, rays.ctypes.data, nodes.ctypes.data,
                              total, counts.ctypes.data)
    cuts = np.cumsum(counts.astype(np.int64))[:-1]
    return texels, np.split(rays, cuts), np.split(nodes, cuts)
