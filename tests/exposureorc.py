"""ctypes wrapper over oracle_exposure/libexposureorc.so — exposure::State::step on the raytracer oracle (TEST
INFRASTRUCTURE: the checker, never the product).  ln and exp follow the raytracer oracle's libm switch (orc.set_libm)."""
import ctypes as C
import os
import subprocess

import numpy as np

from aicb200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "oracle_exposure", "libexposureorc.so")

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    # built by __graft_entry__.build(); an existing library is loaded as it is
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle_exposure"), "-B"], check=True, capture_output=True)
    L = C.CDLL(LIB_PATH)
    L.orc_exposure_scene_create.restype = C.c_void_p
    L.orc_exposure_scene_create.argtypes = [C.POINTER(abi.SceneDesc)]
    L.orc_exposure_scene_destroy.restype = None
    L.orc_exposure_scene_destroy.argtypes = [C.c_void_p]
    L.orc_exposure_step.restype = None
    L.orc_exposure_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double, C.c_void_p]
    L.orc_exposure_target.restype = C.c_float
    L.orc_exposure_target.argtypes = [C.c_float]
    L.orc_exposure_average.restype = C.c_float
    L.orc_exposure_average.argtypes = [C.c_void_p]
    L.orc_exposure_block_visible.restype = C.c_int
    L.orc_exposure_block_visible.argtypes = [C.c_void_p, C.c_uint32]
    L.orc_set_libm.restype = None
    L.orc_set_libm.argtypes = [C.c_int]
    _lib = L
    return L


def set_libm(mode):
    """0: glibc logf / expf (what Rust's std calls); 1: the correctly rounded ones the device evaluates."""
    lib().orc_set_libm(mode)


class ExposureScene:
    """The exposure oracle's scene of an aicb200.Space."""

    def __init__(self, space):
        desc, keep = space.to_desc()
        self.handle = C.c_void_p(lib().orc_exposure_scene_create(C.byref(desc)))
        del keep

    def __del__(self):
        try:
            if self.handle:
                lib().orc_exposure_scene_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def step(self, states, eye_to_world, dt):
        """State::step for each eye: (states, exposures), as SpaceRaytracer.step_exposure returns them."""
        st = np.ascontiguousarray(states, dtype=abi.EXPOSURE_STATE_DTYPE).copy()
        n = st.shape[0]
        m = np.ascontiguousarray(eye_to_world, dtype=np.float64).reshape(n, 16)
        out = np.zeros(n, dtype=np.float32)
        lib().orc_exposure_step(self.handle, st.ctypes.data, m.ctypes.data, n, float(dt), out.ctypes.data)
        return st, out

    def visible(self, block_id):
        return bool(lib().orc_exposure_block_visible(self.handle, block_id))


def target_exposure(luminance):
    return np.float32(lib().orc_exposure_target(float(np.float32(luminance))))


def luminance_average(state):
    st = np.ascontiguousarray(np.asarray(state, dtype=abi.EXPOSURE_STATE_DTYPE).reshape(1))
    return np.float32(lib().orc_exposure_average(st.ctypes.data))


def same_bytes(a, b):
    """Two arrays are byte for byte equal (floats by their bits)."""
    return np.array_equal(np.ascontiguousarray(a).reshape(-1).view(np.uint8),
                          np.ascontiguousarray(b).reshape(-1).view(np.uint8))
