"""Volumetric hit records are written when their span closes: the cases where a span closes late, or never, against the
oracle bit for bit (hits, steps, depths, ColorBuf, sRGB8, cubes_traced).  A surface whose ray stops before its span
closes is never shaded and takes no slot of the hit stream; one whose span is closed after its voxel block is left
is written with the inner level's caster state."""
import numpy as np
import pytest

import aicb200
import orc
import texorc
from aicb200 import (FOG_NONE, LIGHT_FLAT, LIGHT_LINEAR, LIGHT_NONE, TRANSPARENCY_VOLUMETRIC, Block, Context,
                     GraphicsOptions, RtRenderer, Space, SpaceRaytracer, scenes)
from test_gpu_parity import compare, render_both, same_srgb8
from test_gpu_resolve import faint_slab
from test_gpu_texture import NO_WORLD, same_texels

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _oracle_rounds_once():
    prev = orc.get_libm()
    orc.set_libm(orc.LIBM_CR)
    texorc.set_libm(texorc.LIBM_CR)
    yield
    orc.set_libm(prev)


def volumetric(**kw):
    opts = GraphicsOptions.unaltered_colors()
    opts.transparency = TRANSPARENCY_VOLUMETRIC
    for k, v in kw.items():
        setattr(opts, k, v)
    return opts


def trace_both(space, opts, rays):
    gpu = SpaceRaytracer(space, opts).trace_rays(rays, want_steps=True, want_hit=True, want_depth=True)
    ref = orc.OracleScene(space).trace_rays(rays, opts)
    compare(gpu, ref)
    assert gpu["info"].cubes_traced == int(ref["steps"].sum())
    return ref


def fan(origin, direction, n=64, spread=0.3, seed=0):
    rng = np.random.default_rng(seed)
    d = np.asarray(direction, dtype=float) + rng.uniform(-spread, spread, size=(n, 3)) * [0.0, 1.0, 1.0]
    return np.column_stack([np.tile(origin, (n, 1)), d])


def test_span_made_opaque_with_a_surface_directly_behind():
    """A row of dense transparent cubes makes the ray opaque inside a span; the opaque and transparent cubes right
    behind it are surfaces whose span never closes."""
    ids = np.zeros((24, 3, 3), dtype=np.uint16)
    ids[2:8, :, :] = 1
    ids[8, :, :] = 2
    ids[9:, :, :] = 3
    space = Space((0, 0, 0), ids, [Block.air(), Block(color=(0.8, 0.3, 0.1, 0.85)), Block(color=(0.1, 0.9, 0.2, 1.0)),
                                   Block(color=(0.2, 0.2, 0.9, 0.5))])
    rays = fan((-0.5, 1.5, 1.5), (1.0, 0.0, 0.0), spread=0.15)
    for kw in (dict(), dict(debug_pixel_cost=True)):
        ref = trace_both(space, volumetric(**kw), rays)
        assert (ref["steps"] < 24).any()   # the opacity cut stopped rays before the end of the row


def test_step_cap_with_an_open_span():
    """A long row of faint res-16 voxel blocks: rays reach the 1000-step cap inside a span."""
    blk = scenes.make_voxel_block(5, resolution=16, alpha=0.02, fill_mask=3, partial_bounds=False)
    space = Space((0, 0, 0), np.ones((80, 2, 2), dtype=np.uint16), [Block.air(), blk])
    rays = fan((-0.5, 1.01, 0.99), (1.0, 0.001, 0.002), n=32, spread=0.01, seed=1)
    ref = trace_both(space, volumetric(), rays)
    assert (ref["steps"] == 1001).any()


@pytest.mark.parametrize("direction", [(1, 0.6, 1), (-1, -0.3, 0.2), (0.3, -1, -0.7), (0, 0, -1)])
def test_inner_spans_closed_on_the_outer_level(direction):
    """Partial-bounds transparent voxel blocks: a ray leaves a block's voxel bounds inside a span (the inner iterator
    ends without an exit step) and the Space level's next step closes it."""
    rng = np.random.default_rng(4)
    n = 10
    ids = rng.integers(0, 4, size=(n, n, n)).astype(np.uint16)
    blocks = [Block.air()] + [scenes.make_voxel_block(s, resolution=r, alpha=a, fill_mask=3, partial_bounds=True)
                              for s, r, a in ((11, 16, 0.4), (12, 8, 0.15), (13, 4, 0.7))]
    space = Space((0, 0, 0), ids, blocks)
    for lighting in (LIGHT_NONE, LIGHT_LINEAR):
        opts = GraphicsOptions(transparency=TRANSPARENCY_VOLUMETRIC, lighting_display=lighting, view_distance=60.0)
        cam = scenes.standard_camera(space, opts, 80, 60, direction=direction)
        gpu, img, ref = render_both(space, cam, opts)
        compare(gpu, ref, f"{direction} l{lighting}")
        same_srgb8(img, ref)
        assert img.info.cubes_traced == ref["cubes_traced"]


def test_ui_layer_already_opaque():
    """Layers: where the UI layer in front made the pixel opaque, the world's rays start opaque and emit nothing."""
    world = scenes.small_mixed_scene(n=12, seed=7)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    wopts = GraphicsOptions(view_distance=40.0, transparency=TRANSPARENCY_VOLUMETRIC)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT)
    wcam = scenes.standard_camera(world, wopts, 64, 48)
    ucam = scenes.standard_camera(ui_space, uopts, 64, 48, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    wrt = SpaceRaytracer(world, wopts)
    urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
    got = aicb200.render_layers((wrt, wcam, wopts), (urt, ucam, uopts), None, NO_WORLD)
    ref = orc.render_layers((orc.OracleScene(world), wcam, wopts), (orc.OracleScene(ui_space), ucam, uopts), None,
                            NO_WORLD)
    assert np.array_equal(got.data.reshape(-1, 4), ref["srgb8"])
    assert got.info.cubes_traced == ref["cubes_traced"]


def test_hit_stream_overflow_retry():
    """19-65 surfaces per ray: the first frame of a fresh context overflows its hit stream and is re-run."""
    space = faint_slab()
    opts = GraphicsOptions(lighting_display=LIGHT_FLAT, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0)
    cam = scenes.standard_camera(space, opts, 64, 32, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    ref = orc.OracleScene(space).render(cam, opts)
    ctx = Context()
    try:
        r = RtRenderer(cam, ctx)
        r.update(space)
        gpu = r.draw_colorbuf()
        assert gpu["info"].counters[2] > 8 * gpu["info"].rays
        compare(gpu, ref, "overflow")
        assert gpu["info"].cubes_traced == ref["cubes_traced"]
        img = r.draw()
        same_srgb8(img, ref)
        r.rt.close()
    finally:
        ctx.close()


def test_pixel_list_texture_batch():
    world = scenes.config_c2(n=24, n_voxel_blocks=4, with_light=True)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    wopts = GraphicsOptions(view_distance=96.0, transparency=TRANSPARENCY_VOLUMETRIC, exposure=1.75)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT, exposure=0.625)
    wcam = scenes.standard_camera(world, wopts, 64, 48)
    ucam = scenes.standard_camera(ui_space, uopts, 64, 48, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    wrt = SpaceRaytracer(world, wopts)
    urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
    m = wcam.depth_transform()
    bd = (0.1, 0.3, 0.6, 0.5)
    px = np.random.default_rng(3).integers(0, 64 * 48, size=777).astype(np.uint32)
    for ui in (None, (urt, ucam, uopts)):
        rgba, depth, info = aicb200.render_layers_texture((wrt, wcam, wopts), ui, bd, NO_WORLD, m, pixels=px)
        ref_rgba, ref_depth, ref_total = texorc.render_layers_texture(
            (texorc.Scene(world), wcam, wopts), None if ui is None else (texorc.Scene(ui_space), ucam, uopts), bd,
            NO_WORLD, m, pixels=px)
        assert same_texels(rgba, depth, ref_rgba, ref_depth)
        assert info.cubes_traced == ref_total
