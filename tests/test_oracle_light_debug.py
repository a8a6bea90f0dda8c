"""Pins orc_light_compute_debug (oracle_light/aic_light_blocks.cpp), Space::compute_light::<LightUpdateCubeInfo>, against
the reference's light tests (space/light/tests.rs) where they apply, and checks what every cube's ray list must satisfy
on the scenes of the GPU light tests.  CPU only."""
import numpy as np
import pytest

import lightdebugorc
from aicb200 import Block, Space
from lightorc import LightOracle
from test_gpu_group_light import slab_space
from test_gpu_light import NO_RAYS, all_cubes, light_scene
from test_gpu_light_voxels import VOXEL_SCENES
from test_oracle_light import WHITE, some, value

SCENES = dict(VOXEL_SCENES, light_scene=light_scene, slab_space=slab_space)


def lut(v):
    return np.array([value((int(x), 0, 0))[0] for x in v], dtype=np.float32)


# tests.rs:233-261: an opaque emitter in the middle of a 3^3 Space under a black sky
def test_rays_around_an_opaque_emitter():
    light = (0.5, 1.0, 2.0)
    ids = np.zeros((3, 3, 3), dtype=np.uint16)
    field = np.zeros((3, 3, 3, 4), dtype=np.uint8)
    field[..., 3] = NO_RAYS
    space = Space((0, 0, 0), ids, [Block.air(), Block(color=WHITE, emission=light)], light=field,
                  sky_colors=[(0.0, 0.0, 0.0)], light_max_distance=30)
    ol = LightOracle(space)
    ol.set_cubes([(1, 1, 1)], [1])
    ol.evaluate(0)
    cubes = all_cubes(space)
    texels, rays, nodes = lightdebugorc.compute_debug(ol, cubes)
    assert np.array_equal(texels, lightdebugorc.compute(ol, cubes))
    f = ol.field()
    centre = 13
    assert tuple(texels[centre]) == some(light) and rays[centre].size == 0   # opaque origin: no walk
    f32 = np.float32
    expect = {0: (f32(0.13397168), f32(0.26794338), f32(0.53588676)),
              1: (f32(0.1649385), f32(0.32987696), f32(0.6597539)),
              2: (f32(0.21763763), f32(0.43527526), f32(0.8705506))}
    emission = np.array(light, dtype=np.float32)
    for axis in range(3):
        for side in (0, 2):
            c = [1, 1, 1]
            c[axis] = side
            i = (c[0] * 3 + c[1]) * 3 + c[2]
            assert value(texels[i]) == expect[axis], c
            # every ray of a face neighbour ends on the emitter's face toward it and reads the neighbour's own light
            r = rays[i]
            assert r.size > 0
            assert (r["trigger_cube"] == (1, 1, 1)).all() and (r["value_cube"] == c).all()
            assert (r["value"] == f[tuple(c)]).all()
            lf = emission + (f32(1.0) * lut(f[tuple(c)][:3])) * f32(1.0)   # emission + WHITE.reflect(value)
            assert np.array_equal(r["light_from_struck_face"], np.broadcast_to(lf, (r.size, 3)))
    # the emitter is the only visible block: every ray of every cube strikes it
    for r in rays:
        assert (r["trigger_cube"] == (1, 1, 1)).all()


@pytest.mark.parametrize("name", list(SCENES))
def test_every_ray_list_meets_the_invariants(name):
    space = SCENES[name]()
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0, max_updates=300)
    field = ol.field()
    cubes = all_cubes(space)
    texels, rays, nodes = lightdebugorc.compute_debug(ol, cubes)
    assert np.array_equal(texels, lightdebugorc.compute(ol, cubes))
    lower, size = np.array(space.lower), np.array(space.size)
    opaque_faces = np.array([b.light_opaque_faces for b in space.blocks])
    n_rays = 0
    for cube, r, nd in zip(cubes, rays, nodes):
        rel = cube - lower
        if opaque_faces[space.block_ids[tuple(rel)]] == 0x3F:
            assert r.size == 0, cube
            continue
        assert (np.diff(nd.astype(np.int64)) > 0).all(), cube    # preorder = the reference's order
        n_rays += r.size
        for ray in r:
            t, v = ray["trigger_cube"] - lower, ray["value_cube"] - lower
            step = v - t
            assert np.abs(step).sum() == 1
            axis = int(np.flatnonzero(step)[0])
            face = axis + (3 if step[axis] > 0 else 0)             # the struck face, NX..PZ
            assert (opaque_faces[space.block_ids[tuple(t)]] >> face) & 1, (cube, ray)
            if ((v >= 0) & (v < size)).all():
                assert (ray["value"] == field[tuple(v)]).all(), (cube, ray)
    assert n_rays > 0
