"""ctypes wrapper over oracle_light/liblightorc.so — the light oracle with a live block table (TEST INFRASTRUCTURE: the
checker, never the product).  LightOracle is orc.OracleLight's light oracle with block definitions that change after
creation (update_blocks, append_blocks) and the light side of a redefinition (relight_blocks)."""
import ctypes as C
import os
import subprocess

import numpy as np

from aicb200 import _block_descs, abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "oracle_light", "liblightorc.so")

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    # built by __graft_entry__.build(); an existing library is loaded as it is
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle_light"), "-B"], check=True, capture_output=True)
    L = C.CDLL(LIB_PATH)
    L.orc_light_create.restype = C.c_void_p
    L.orc_light_create.argtypes = [C.POINTER(abi.SceneDesc)]
    L.orc_light_destroy.argtypes = [C.c_void_p]
    L.orc_light_fast_evaluate.argtypes = [C.c_void_p]
    L.orc_light_set_cubes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    L.orc_light_evaluate.restype = C.c_uint64
    L.orc_light_evaluate.argtypes = [C.c_void_p, C.c_uint8, C.c_uint64, C.c_void_p]
    L.orc_light_get.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_light_queue_len.restype = C.c_size_t
    L.orc_light_queue_len.argtypes = [C.c_void_p]
    L.orc_light_update_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    L.orc_light_append_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.orc_light_relight_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    _lib = L
    return L


class LightOracle:
    """Light propagation oracle over a Space whose block table changes (space/light/updater.rs restatement)."""

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

    def update_blocks(self, indices, blocks):
        idx = np.ascontiguousarray(indices, dtype=np.uint16)
        lib().orc_light_update_blocks(self.handle, idx.ctypes.data, _block_descs(blocks), len(blocks))

    def append_blocks(self, blocks):
        lib().orc_light_append_blocks(self.handle, _block_descs(blocks), len(blocks))

    def relight_blocks(self, indices):
        idx = np.ascontiguousarray(indices, dtype=np.uint16).reshape(-1)
        lib().orc_light_relight_blocks(self.handle, idx.ctypes.data, idx.size)

    def field(self):
        out = np.zeros(self.shape + (4,), dtype=np.uint8)
        lib().orc_light_get(self.handle, out.ctypes.data)
        return out

    def queue_len(self):
        return int(lib().orc_light_queue_len(self.handle))
