"""Space::compute_light::<LightUpdateCubeInfo> on the GPU (aicb_light_compute_debug / aicb_group_light_compute_debug):
the texels, the number of rays of every cube and every field of every ray, bit for bit against the oracle
(orc_light_compute_debug) on the field the GPU converged to, on one context and on a group naming the same device twice.
Rejected calls and the capacity contract leave the volume, the queue and the set of changed cubes as they were."""
import ctypes as C

import numpy as np
import pytest

import lightdebugorc
from aicb200 import LIGHT_RAY_DTYPE, AicbError, GraphicsOptions, SpaceRaytracer, abi
from lightorc import LightOracle
from test_gpu_group_light import group_scene, slab_space, with_field
from test_gpu_light import all_cubes, light_scene
from test_gpu_light_voxels import VOXEL_SCENES

pytestmark = pytest.mark.gpu

SCENES = dict(VOXEL_SCENES, light_scene=light_scene, slab_space=slab_space)
DEVICES = {"ctx": None, "group2": [0, 0]}


def lit_scene(space, devices):
    """A scene of `space` after fast_evaluate + evaluate(1), on one context or a group."""
    if devices is None:
        g, s = None, SpaceRaytracer(space, GraphicsOptions())
    else:
        g, s = group_scene(devices, space)
    s.light_fast_evaluate()
    s.light_evaluate(1)
    return g, s


def state(s):
    return s.light_download(), s.light_download_queue(), s.light_changes_count()


@pytest.mark.parametrize("devices", list(DEVICES.values()), ids=list(DEVICES))
@pytest.mark.parametrize("name", list(SCENES))
def test_rays_are_bit_exact(name, devices):
    space = SCENES[name]()
    g, s = lit_scene(space, devices)
    field = s.light_download()
    cubes = all_cubes(space)
    before = state(s)
    texels, rays = s.light_compute_debug(cubes)
    debug_stats = s.light_stats()
    assert all(np.array_equal(a, b) for a, b in zip(before, state(s)))
    assert np.array_equal(texels, s.light_compute(cubes))
    assert s.light_stats() == debug_stats            # the same counters as aicb_light_compute's
    if name in ("slab_space", "translucent_stack"):
        assert debug_stats["rounds"] > 0             # some cubes took the lockstep walk
    ref_texels, ref_rays, _ = lightdebugorc.compute_debug(LightOracle(with_field(space, field)), cubes)
    assert np.array_equal(texels, ref_texels)
    assert [r.size for r in rays] == [r.size for r in ref_rays]
    got, want = np.concatenate(rays), np.concatenate(ref_rays)
    assert got.size > 0
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), "rays differ from the oracle"
    s.close()


def raw_call(s, cubes, rays, capacity, counts, texels, total):
    c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
    return s._fn("light_compute_debug")(s.handle, c.ctypes.data if c.size else None, c.shape[0],
                                         None if texels is None else texels.ctypes.data,
                                         None if rays is None else rays.ctypes.data, capacity,
                                         None if counts is None else counts.ctypes.data,
                                         None if total is None else C.byref(total))


@pytest.mark.parametrize("devices", list(DEVICES.values()), ids=list(DEVICES))
def test_capacity_and_rejected_calls_change_nothing(devices):
    space = light_scene()
    g, s = lit_scene(space, devices)
    cubes = all_cubes(space)[::7]
    _, rays = s.light_compute_debug(cubes)
    need = sum(r.size for r in rays)
    assert need > 1
    stats, before = s.light_stats(), state(s)
    n = cubes.shape[0]
    buf = np.frombuffer(np.full(need * LIGHT_RAY_DTYPE.itemsize, 0xAB, dtype=np.uint8).tobytes(), dtype=LIGHT_RAY_DTYPE).copy()
    texels, counts = np.full((n, 4), 7, dtype=np.uint8), np.full(n, 7, dtype=np.uint32)
    total = C.c_size_t(0)
    assert raw_call(s, cubes, buf, need - 1, counts, texels, total) == abi.ERR_INVALID
    assert total.value == need
    assert (buf.view(np.uint8) == 0xAB).all() and (texels == 7).all() and (counts == 7).all()
    total = C.c_size_t(0)
    assert raw_call(s, cubes, None, need, counts, texels, total) == abi.ERR_INVALID and total.value == need
    # the argument checks: NULL outputs, a cube out of bounds
    for args in [(None, counts, texels, total), (buf, None, texels, total), (buf, counts, None, total),
                 (buf, counts, texels, None)]:
        assert raw_call(s, cubes, args[0], need, args[1], args[2], args[3]) == abi.ERR_INVALID
    outside = cubes.copy()
    outside[3] = np.array(space.lower) + np.array(space.size)
    total = C.c_size_t(0)
    assert raw_call(s, outside, buf, need, counts, texels, total) == abi.ERR_INVALID and total.value == 0
    assert (buf.view(np.uint8) == 0xAB).all() and (texels == 7).all() and (counts == 7).all()
    with pytest.raises(AicbError):
        s.light_compute_debug(outside)
    assert s.light_stats() == stats
    assert all(np.array_equal(a, b) for a, b in zip(before, state(s)))
    # capacity exactly the total, and no cubes
    total = C.c_size_t(0)
    assert raw_call(s, cubes, buf, need, counts, texels, total) == abi.OK and total.value == need
    assert np.array_equal(buf.view(np.uint8), np.concatenate(rays).view(np.uint8))
    assert raw_call(s, cubes[:0], None, 0, None, None, total) == abi.OK and total.value == 0
    s.close()


def test_light_physics_none_is_rejected():
    space = light_scene()
    unlit = type(space)(space.lower, space.block_ids, space.blocks, light=None, sky_colors=space.sky_colors,
                        light_max_distance=0)
    rt = SpaceRaytracer(unlit, GraphicsOptions())
    with pytest.raises(AicbError):
        rt.light_compute_debug(all_cubes(space)[:4])
    total = C.c_size_t(5)
    assert raw_call(rt, all_cubes(space)[:0], None, 0, None, None, total) == abi.ERR_INVALID
    rt.close()
