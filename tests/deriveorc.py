"""ctypes wrapper over oracle_derive/libderiveorc.so — compute_derived's light fields (TEST INFRASTRUCTURE: the checker,
never the product)."""
import ctypes as C
import os
import subprocess

from aicb200 import BlockLight, _block_descs, abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "oracle_derive", "libderiveorc.so")
LIBM_PLATFORM, LIBM_CR = 0, 1

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    # built by __graft_entry__.build(); an existing library is loaded as it is
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle_derive"), "-B"], check=True, capture_output=True)
    L = C.CDLL(LIB_PATH)
    L.orc_derive_block_light.restype = C.c_int
    L.orc_derive_block_light.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t)]
    L.orc_set_libm.argtypes = [C.c_int]
    L.orc_set_libm.restype = None
    _lib = L
    return L


def set_libm(mode):
    """The f32 powf of apply_transmittance: LIBM_PLATFORM = this host's powf (what Rust's std calls), LIBM_CR = the
    correctly rounded one (what the device computes)."""
    lib().orc_set_libm(int(mode))


class DerivePanic(Exception):
    """compute_derived panics (Rgb::try_from(..).expect(..)) on the block at `position`."""

    def __init__(self, position):
        super().__init__(f"compute_derived panics on block {position}")
        self.position = position


def derive(blocks):
    """compute_derived's light fields of every block, as aicb200.BlockLight; DerivePanic where the reference panics."""
    n = len(blocks)
    descs = _block_descs(blocks)
    out = (abi.BlockLight * max(n, 1))()
    bad = C.c_size_t()
    if lib().orc_derive_block_light(descs, n, out, C.byref(bad)):
        raise DerivePanic(bad.value)
    return [BlockLight.from_abi(out[i]) for i in range(n)]
