"""The CPU restatement of RaytraceToTexture's per-pixel work (oracle_texture/aic_texture.cpp): Split's layer rule on
hand-built rays, Split::mean, trace_one's stores, Camera.depth_transform() and pixel_picker_order().  The reference
has no test for this caller (raytrace_to_texture.rs:998), so these pin the restatement against its source."""
import math

import numpy as np
import pytest

import aicb200
import orc
import texorc
from aicb200 import FOG_NONE, LIGHT_NONE, Block, Camera, GraphicsOptions, Space, Viewport, scenes

OPTS = GraphicsOptions(fog=FOG_NONE, lighting_display=LIGHT_NONE, view_distance=50.0)
HIT = (0.5, 0.5, -5.0, 0.0, 0.0, 1.0)    # meets cube (0, 0, 0) at t = 5
MISS = (5.5, 5.5, -5.0, 0.0, 0.0, 1.0)   # passes beside it


def one_cube(color):
    return Space((0, 0, 0), np.ones((1, 1, 1), dtype=np.uint16), [Block.air(), Block(color=color)])


@pytest.fixture(scope="module")
def layers():
    texorc.set_libm(texorc.LIBM_CR)
    ui_partial = texorc.Scene(one_cube((0.2, 0.9, 0.3, 0.5)))
    world = texorc.Scene(one_cube((0.8, 0.1, 0.1, 1.0)))
    return ui_partial, world


def trace(world_scene, ui_scene, backdrop=None, no_world=None, world_ray=HIT, ui_ray=HIT):
    w = (world_scene, OPTS) if world_scene else None
    u = (ui_scene, OPTS) if ui_scene else None
    r = texorc.trace_samples(w, u, backdrop, no_world, [world_ray] if w else None, [ui_ray] if u else None)
    return r["colorbuf"][0], r["depth"][0], int(r["layer"][0])


def test_partial_ui_hit_makes_the_pixel_ui(layers):
    ui, world = layers
    cb, depth, layer = trace(world, ui)
    assert layer == texorc.LAYER_UI
    assert depth == 5.0          # the UI surface is the nearest
    assert cb[3] == 0.0          # the world behind it (and the sky) made it opaque


def test_transparent_ui_over_a_world_hit_is_world(layers):
    ui, world = layers
    cb, depth, layer = trace(world, ui, ui_ray=MISS)
    assert layer == texorc.LAYER_WORLD
    assert depth == 5.0


def test_backdrop_alone_makes_the_pixel_ui(layers):
    ui, world = layers
    cb, depth, layer = trace(world, None, backdrop=(0.1, 0.2, 0.3, 0.5))
    assert layer == texorc.LAYER_UI
    assert depth == 5.0          # the backdrop has no depth; the world's surface does
    cb, depth, layer = trace(world, ui, backdrop=(0.1, 0.2, 0.3, 0.5), ui_ray=MISS)
    assert layer == texorc.LAYER_UI


def test_paint_is_world_at_the_far_plane(layers):
    ui, _ = layers
    cb, depth, layer = trace(None, ui, no_world=(0.5, 0.5, 0.5, 1.0), ui_ray=MISS)
    assert layer == texorc.LAYER_WORLD
    assert depth == math.inf     # P::paint starts a fresh Split
    # and the UI hit of a painted pixel is forgotten: paint replaces the whole accumulator
    cb, depth, layer = trace(None, ui, no_world=(0.5, 0.5, 0.5, 1.0))
    assert (layer, depth) == (texorc.LAYER_WORLD, math.inf)
    cam = Camera(OPTS, Viewport.with_scale(1.0, (8, 8)))
    m = cam.depth_transform()
    rgba, d, l = texorc.mean_and_store([cb], [depth], [layer], 2.0, 3.0, m)
    assert l == texorc.LAYER_WORLD
    assert d == np.float32(1.0)   # +inf clamps to 1: the far plane, positive for the world
    assert rgba[0] == texorc.f16_bits(np.float32(cb[0]) * np.float32(2.0))


def test_nothing_is_none_with_negative_depth_and_unit_exposure(layers):
    ui, _ = layers
    cb, depth, layer = trace(None, ui, ui_ray=MISS)
    assert layer == texorc.LAYER_NONE
    assert cb[3] == 1.0 and depth == math.inf
    cam = Camera(OPTS, Viewport.with_scale(1.0, (8, 8)))
    cb = np.array([0.25, 0.5, 0.75, 1.0], dtype=np.float32)   # an emissive transparent UI leaves light, T = 1
    rgba, d, l = texorc.mean_and_store([cb], [math.inf], [texorc.LAYER_NONE], 2.0, 3.0, cam.depth_transform())
    assert l == texorc.LAYER_NONE
    assert d == np.float32(-1.0)  # InLayer::Ui's sign for no layer
    assert list(rgba) == [texorc.f16_bits(v) for v in (0.25, 0.5, 0.75, 0.0)]   # exposure 1


def test_mean_takes_the_first_tagged_sample_and_the_least_depth():
    cam = Camera(OPTS, Viewport.with_scale(1.0, (8, 8)))
    m = cam.depth_transform()
    cb = np.array([[0.1, 0.2, 0.3, 1.0], [0.4, 0.1, 0.2, 0.5], [0.2, 0.2, 0.2, 0.0], [0.0, 0.0, 0.0, 1.0]],
                  dtype=np.float32)
    depth = [0.7, 0.5, 0.2, math.inf]
    layer = [texorc.LAYER_NONE, texorc.LAYER_UI, texorc.LAYER_WORLD, texorc.LAYER_NONE]
    rgba, d, l = texorc.mean_and_store(cb, depth, layer, 2.0, 3.0, m)
    assert l == texorc.LAYER_UI
    mean = (cb[0] + cb[1] + cb[2] + cb[3]) / np.float32(4.0)
    assert rgba[0] == texorc.f16_bits(mean[0] * np.float32(3.0))   # the UI camera's exposure
    a = np.float32(1.0) - mean[3]
    assert rgba[3] == texorc.f16_bits(a)
    z = (0.0 * m[0, 2] + 0.0 * m[1, 2]) + 0.2 * m[2, 2] + m[3, 2]
    w = (0.0 * m[0, 3] + 0.0 * m[1, 3]) + 0.2 * m[2, 3] + m[3, 3]
    assert d == -np.float32(z / w)


def test_f16_conversion_rounds_like_half():
    rng = np.random.default_rng(5)
    v = np.concatenate([rng.standard_normal(2000).astype(np.float32) * 300,
                        np.array([0.0, -0.0, 65504.0, 65520.0, 1e-8, 6e-8, 3e-5, np.inf, -np.inf], dtype=np.float32)])
    got = np.array([texorc.f16_bits(x) for x in v], dtype=np.uint16)
    assert np.array_equal(got, v.astype(np.float16).view(np.uint16))


def test_depth_transform_maps_the_near_and_far_planes():
    for fov, vd, size in ((90.0, 200.0, (64, 48)), (30.0, 37.5, (100, 20)), (140.0, 10000.0, (3, 7))):
        cam = Camera(GraphicsOptions(fov_y=fov, view_distance=vd), Viewport.with_scale(1.0, size))
        m = cam.depth_transform()
        p = cam.projection_matrix()
        near, far = Camera.NEAR_PLANE_DISTANCE, vd

        def ndc_z(eye_z):   # the projection applied to an eye-space point on the axis
            return (eye_z * p[2, 2] + p[3, 2]) / (eye_z * p[2, 3] + p[3, 3])

        for d, eye_z in ((0.0, -near), (1.0, -far)):
            z = 0.0 * m[0, 2] + 0.0 * m[1, 2] + d * m[2, 2] + m[3, 2]
            w = 0.0 * m[0, 3] + 0.0 * m[1, 3] + d * m[2, 3] + m[3, 3]
            assert math.isclose(z / w, ndc_z(eye_z), rel_tol=1e-12, abs_tol=1e-15), (fov, vd, d)
        assert abs(ndc_z(-near)) < 1e-15 and math.isclose(ndc_z(-far), 1.0, rel_tol=1e-12)


def test_pixel_picker_order_covers_the_frame_centre_first():
    for w, h in ((40, 30), (7, 5), (600, 400)):
        n = w * h
        order = aicb200.pixel_picker_order(w, h)
        central = min(60000, n // 4)
        assert len(order) == max(central, n - central) * 2
        assert set(order.tolist()) == set(range(n))
        first = int(order[0])   # the centre pixel (dither 0) comes first
        assert abs(first % w - (w / 2 - 0.5)) <= 1 and abs(first // w - (h / 2 - 0.5)) <= 1
        if central:   # the centre is revisited: inner picks are every other one
            assert order[0] == order[2 * central]


def test_whole_texture_oracle_agrees_with_the_layers_oracle():
    """With exposure 1 the colour texels are the f16 of the layers oracle's ColorBuf (premultiplied, clamped alpha)."""
    texorc.set_libm(texorc.LIBM_CR)
    prev = orc.get_libm()
    orc.set_libm(orc.LIBM_CR)
    try:
        check_whole_texture()
    finally:
        orc.set_libm(prev)


def check_whole_texture():
    mixed = scenes.small_mixed_scene(n=8, seed=3)
    ui_space = scenes.small_mixed_scene(n=5, seed=11, lower=(0, 0, 0))
    wopts = GraphicsOptions(view_distance=40.0)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_NONE)
    wcam = scenes.standard_camera(mixed, wopts, 24, 16)
    ucam = scenes.standard_camera(ui_space, uopts, 24, 16, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    before = texorc.monotonic_violations()
    rgba, depth, total = texorc.render_layers_texture((texorc.Scene(mixed), wcam, wopts),
                                                      (texorc.Scene(ui_space), ucam, uopts), (0.1, 0.3, 0.6, 0.5),
                                                      None, wcam.depth_transform())
    ref = orc.render_layers((orc.OracleScene(mixed), wcam, wopts), (orc.OracleScene(ui_space), ucam, uopts),
                            (0.1, 0.3, 0.6, 0.5), None)
    cb = ref["colorbuf"]
    a = np.clip(np.float32(1.0) - cb[:, 3], 0.0, 1.0).astype(np.float32)
    want = np.stack([cb[:, 0], cb[:, 1], cb[:, 2], a], axis=1).astype(np.float16).view(np.uint16)
    assert np.array_equal(rgba, want)
    assert total == ref["cubes_traced"]
    assert texorc.monotonic_violations() == before
    assert np.all(np.abs(depth[~np.isnan(depth)]) <= 1.0)   # NDC depth of the clamped ray distance, signed
