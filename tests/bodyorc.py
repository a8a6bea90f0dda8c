"""ctypes wrapper over oracle_body/libbodyorc.so — step_one_body and collide_along_ray on the raytracer oracle (TEST
INFRASTRUCTURE: the checker, never the product)."""
import ctypes as C
import os
import subprocess

import numpy as np

from aicb200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "oracle_body", "libbodyorc.so")

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    # built by __graft_entry__.build(); an existing library is loaded as it is
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle_body"), "-B"], check=True, capture_output=True)
    L = C.CDLL(LIB_PATH)
    L.orc_body_scene_create.restype = C.c_void_p
    L.orc_body_scene_create.argtypes = [C.POINTER(abi.SceneDesc)]
    L.orc_body_scene_destroy.restype = None
    L.orc_body_scene_destroy.argtypes = [C.c_void_p]
    L.orc_block_uniform_collision.restype = C.c_int
    L.orc_block_uniform_collision.argtypes = [C.POINTER(abi.BlockDesc)]
    L.orc_step_bodies.restype = C.c_int
    L.orc_step_bodies.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_uint32, C.c_int]
    L.orc_collide_along_ray.restype = C.c_int
    L.orc_collide_along_ray.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_double),
                                        C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    L.orc_crush_if_colliding.restype = C.c_int
    L.orc_crush_if_colliding.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_uncrush.restype = C.c_int
    L.orc_uncrush.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    _lib = L
    return L


def uniform_collision(block):
    """uniform_collision of an aicb200.Block: 0 Hard, 1 None, 2 mixed."""
    from aicb200 import fill_block_desc
    bd = abi.BlockDesc()
    fill_block_desc(bd, block)
    return lib().orc_block_uniform_collision(C.byref(bd))


class BodyScene:
    """The body oracle's scene of an aicb200.Space."""

    def __init__(self, space):
        desc, keep = space.to_desc()
        self.handle = C.c_void_p(lib().orc_body_scene_create(C.byref(desc)))
        del keep

    def __del__(self):
        try:
            if self.handle:
                lib().orc_body_scene_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def step_bodies(self, bodies, dt, gravity, external_delta_v=None, max_contacts=16, threads=None):
        """step_one_body for an abi.BODY_DTYPE array: (bodies after, info, contacts [n, max_contacts]); None if the
        call is rejected (a body the reference could not hold)."""
        b = np.ascontiguousarray(bodies, dtype=abi.BODY_DTYPE).copy()
        n = b.shape[0]
        edv = None if external_delta_v is None else np.ascontiguousarray(
            np.broadcast_to(np.asarray(external_delta_v, dtype=np.float64), (n, 3)))
        g = np.ascontiguousarray(gravity, dtype=np.float64)
        info = np.zeros(n, dtype=abi.BODY_STEP_INFO_DTYPE)
        contacts = np.zeros((n, max_contacts), dtype=abi.CONTACT_DTYPE)
        nt = threads or os.cpu_count() or 1
        r = lib().orc_step_bodies(self.handle, b.ctypes.data, None if edv is None else edv.ctypes.data, n, float(dt),
                                  g.ctypes.data, info.ctypes.data, contacts.ctypes.data, max_contacts, nt)
        if r != 0:
            return None
        return b, info, contacts

    def crush_if_colliding(self, body):
        """crush_if_colliding alone: (body after, CrushInfo [6], panic status)."""
        b = np.ascontiguousarray(body, dtype=abi.BODY_DTYPE).reshape(1).copy()
        info = np.zeros(6, dtype=np.float64)
        st = lib().orc_crush_if_colliding(self.handle, b.ctypes.data, info.ctypes.data)
        return b[0], info, st

    def uncrush(self, body):
        """uncrush alone: (body after, abi.UNCRUSH_*, axes [3])."""
        b = np.ascontiguousarray(body, dtype=abi.BODY_DTYPE).reshape(1).copy()
        axes = np.zeros(3, dtype=np.uint8)
        r = lib().orc_uncrush(self.handle, b.ctypes.data, axes.ctypes.data)
        return b[0], r, axes

    def collide_along_ray(self, origin_dir, aab, not_already=True, max_reported=64):
        """collide_along_ray on the Space: ((t, contact) or None, reported contacts)."""
        od = np.ascontiguousarray(origin_dir, dtype=np.float64)
        box = np.ascontiguousarray(aab, dtype=np.float64)
        t = C.c_double(0.0)
        contact = np.zeros(1, dtype=abi.CONTACT_DTYPE)
        reported = np.zeros(max_reported, dtype=abi.CONTACT_DTYPE)
        n = C.c_uint32(0)
        hit = lib().orc_collide_along_ray(self.handle, od.ctypes.data, box.ctypes.data, 1 if not_already else 0,
                                          C.byref(t), contact.ctypes.data, reported.ctypes.data, max_reported,
                                          C.byref(n))
        return ((t.value, contact[0]) if hit else None), reported[:n.value]


def contact_tuple(c):
    """A contact as a hashable tuple (kind, cube, face, resolution, voxel)."""
    return (int(c["kind"]), tuple(int(v) for v in c["cube"]), int(c["face"]), int(c["resolution"]),
            tuple(int(v) for v in c["voxel"]))


def same_bits(a, b):
    """Two structured arrays are byte for byte equal (f64s by their bits)."""
    return np.array_equal(np.asarray(a).reshape(-1).view(np.uint8), np.asarray(b).reshape(-1).view(np.uint8))
