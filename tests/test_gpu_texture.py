"""aicb_render_layers_texture — RaytraceToTexture's colour and depth texels (raytrace_to_texture.rs:591-683) for the
whole texture or a batch of pixels — against the CPU restatement (oracle_texture/) and the library's other outputs."""
import numpy as np
import pytest

import aicb200
import orc
import texorc
from aicb200 import (FOG_NONE, LIGHT_FLAT, LIGHT_NONE, TRANSPARENCY_VOLUMETRIC, AicbError, Camera, Context,
                     GraphicsOptions, RtRenderer, SpaceRaytracer, Viewport, abi, scenes)
from test_gpu_resolve import faint_slab

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _oracle_rounds_once():
    prev = orc.get_libm()
    orc.set_libm(orc.LIBM_CR)
    texorc.set_libm(texorc.LIBM_CR)
    yield
    orc.set_libm(prev)


def same_texels(rgba, depth, ref_rgba, ref_depth):
    """f16 bits equal; f32 depth bits equal, a NaN only as a NaN."""
    if not np.array_equal(rgba, ref_rgba):
        return False
    nan = np.isnan(depth)
    return np.array_equal(nan, np.isnan(ref_depth)) and np.array_equal(depth[~nan].view(np.uint32),
                                                                        ref_depth[~nan].view(np.uint32))


NO_WORLD = aicb200.srgb8_to_linear((0xBC, 0xBC, 0xBC)) + (1.0,)
CASES = [
    dict(world=True, ui=True, backdrop=(0.1, 0.3, 0.6, 0.5)),
    dict(world=True, ui=True, backdrop=None),
    dict(world=True, ui=False, backdrop=(0.9, 0.2, 0.1, 0.25)),
    dict(world=False, ui=True, backdrop=(0.0, 0.5, 0.0, 0.3)),
    dict(world=False, ui=True, backdrop=None),
]


def layer_setup(mixed_space, ui_space, aa, debug=False):
    wopts = GraphicsOptions(view_distance=40.0, antialiasing_always=aa, exposure=1.75, debug_pixel_cost=debug)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT, exposure=0.625,
                            antialiasing_always=aa)
    wcam = scenes.standard_camera(mixed_space, wopts, 64, 48)
    ucam = scenes.standard_camera(ui_space, uopts, 64, 48, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    return wopts, uopts, wcam, ucam


@pytest.mark.parametrize("debug", [False, True])
@pytest.mark.parametrize("aa", [False, True])
def test_whole_texture_equals_the_oracle(aa, debug):
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    wopts, uopts, wcam, ucam = layer_setup(mixed, ui_space, aa, debug)
    wrt = SpaceRaytracer(mixed, wopts)
    urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
    wo, uo = texorc.Scene(mixed), texorc.Scene(ui_space)
    m = wcam.depth_transform()
    before = texorc.monotonic_violations()
    for c in CASES:
        gw = (wrt, wcam, wopts) if c["world"] else None
        gu = (urt, ucam, uopts) if c["ui"] else None
        rgba, depth, info = aicb200.render_layers_texture(gw, gu, c["backdrop"], NO_WORLD, m)
        ref_rgba, ref_depth, ref_total = texorc.render_layers_texture(
            (wo, wcam, wopts) if c["world"] else None, (uo, ucam, uopts) if c["ui"] else None, c["backdrop"], NO_WORLD, m)
        assert same_texels(rgba, depth, ref_rgba, ref_depth), f"aa={aa} debug={debug} {c}"
        assert info.cubes_traced == ref_total, f"aa={aa} {c}"
        if c["world"] and c["ui"] and c["backdrop"] is None:   # UI pixels and world pixels side by side
            assert (depth > 0).any() and (depth < 0).any()
    assert texorc.monotonic_violations() == before


def test_pixel_batches_equal_the_whole_texture_and_the_oracle():
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    for aa in (False, True):
        wopts, uopts, wcam, ucam = layer_setup(mixed, ui_space, aa)
        wrt = SpaceRaytracer(mixed, wopts)
        urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
        wo, uo = texorc.Scene(mixed), texorc.Scene(ui_space)
        m = wcam.depth_transform()
        gw, gu = (wrt, wcam, wopts), (urt, ucam, uopts)
        bd = (0.1, 0.3, 0.6, 0.5)
        full_rgba, full_depth, _ = aicb200.render_layers_texture(gw, gu, bd, NO_WORLD, m)
        n = 64 * 48
        rng = np.random.default_rng(3)
        batches = [aicb200.pixel_picker_order(64, 48, 1000), rng.integers(0, n, size=777).astype(np.uint32),
                   np.array([n - 1], dtype=np.uint32)]
        for px in batches:
            rgba, depth, info = aicb200.render_layers_texture(gw, gu, bd, NO_WORLD, m, pixels=px)
            assert same_texels(rgba, depth, full_rgba[px], full_depth[px]), f"aa={aa} batch of {len(px)}"
            ref_rgba, ref_depth, ref_total = texorc.render_layers_texture((wo, wcam, wopts), (uo, ucam, uopts), bd,
                                                                          NO_WORLD, m, pixels=px)
            assert same_texels(rgba, depth, ref_rgba, ref_depth)
            assert info.cubes_traced == ref_total


@pytest.mark.parametrize("lighting", [LIGHT_NONE, LIGHT_FLAT])
def test_deep_batch_overflows_then_matches_through_both_compositing_paths(lighting):
    """19-65 surfaces per ray: the first frame of a fresh context overflows the 8 hit slots per ray and is re-issued;
    then the batch matches the oracle through resolve_kernel and through shade_kernel + encode_kernel."""
    space = faint_slab()
    opts = GraphicsOptions(lighting_display=lighting, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0,
                           exposure=1.5)
    cam = scenes.standard_camera(space, opts, 64, 32, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    m = cam.depth_transform()
    px = aicb200.pixel_picker_order(64, 32, 1500)
    ref_rgba, ref_depth, ref_total = texorc.render_layers_texture((texorc.Scene(space), cam, opts), None, None, NO_WORLD,
                                                                  m, pixels=px)
    ctx = Context()
    try:
        rt = SpaceRaytracer(space, opts, ctx)
        rgba, depth, info = aicb200.render_layers_texture((rt, cam, opts), None, None, NO_WORLD, m, pixels=px)
        assert info.counters[2] > 8 * info.rays   # more surface hits than the first hit stream had slots
        assert same_texels(rgba, depth, ref_rgba, ref_depth)
        assert info.cubes_traced == ref_total
        empty = RtRenderer(cam, ctx)
        empty.update(aicb200.Space((0, 0, 0), np.zeros((4, 4, 4), dtype=np.uint16), [aicb200.Block.air()]))
        empty.draw_colorbuf()   # no surfaces: the next frame is fused
        empty.rt.close()
        for fused in (True, False):
            rgba, depth, info = aicb200.render_layers_texture((rt, cam, opts), None, None, NO_WORLD, m, pixels=px)
            assert (info.stage_ms[3] == 0.0) == fused
            assert same_texels(rgba, depth, ref_rgba, ref_depth), f"fused={fused}"
            assert info.cubes_traced == ref_total
        rt.close()
    finally:
        ctx.close()


def test_world_only_texture_equals_rgba16f_and_colorbuf_depth():
    space = scenes.small_mixed_scene(n=12, seed=7)
    for aa in (False, True):
        opts = GraphicsOptions(view_distance=40.0, antialiasing_always=aa, exposure=2.5)
        cam = scenes.standard_camera(space, opts, 64, 48)
        r = RtRenderer(cam)
        r.update(space)
        m = cam.depth_transform()
        rgba, depth, _ = aicb200.render_layers_texture((r.rt, cam, opts), None, None, None, m)
        assert np.array_equal(rgba, r.draw_rgba16f().reshape(-1, 4).view(np.uint16))
        d = r.draw_colorbuf()["depth"]
        d = np.where(d < 0.0, 0.0, np.where(d > 1.0, 1.0, d))
        z = ((0.0 * m[0, 2] + 0.0 * m[1, 2]) + d * m[2, 2]) + m[3, 2]
        w = ((0.0 * m[0, 3] + 0.0 * m[1, 3]) + d * m[2, 3]) + m[3, 3]
        want = (z / w).astype(np.float32)   # the world layer everywhere: the sky makes every ray opaque
        assert same_texels(depth, depth, want, want)
        assert np.array_equal(depth.view(np.uint32), want.view(np.uint32))


def test_invalid_batches():
    space = scenes.small_mixed_scene(n=8, seed=7)
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(space, opts, 16, 8)
    rt = SpaceRaytracer(space, opts)
    m = cam.depth_transform()
    with pytest.raises(AicbError) as e:
        aicb200.render_layers_texture((rt, cam, opts), None, None, None, m, pixels=np.array([5, 16 * 8], np.uint32))
    assert e.value.status == abi.ERR_INVALID
    lib = aicb200.load_library()
    o = opts.to_abi(True)
    layer = abi.Layer(rt.handle, aicb200.C.pointer(cam.data), aicb200.C.pointer(o))
    mm = np.ascontiguousarray(m, dtype=np.float64).reshape(16)
    rgba = np.zeros((200, 4), dtype=np.uint16)
    depth = np.zeros(200, dtype=np.float32)
    dptr = mm.ctypes.data_as(aicb200.C.POINTER(aicb200.C.c_double))
    # without a list the length must be the texture's
    assert lib.aicb_render_layers_texture(aicb200.C.byref(layer), None, None, None, dptr, None, 127, rgba.ctypes.data,
                                          depth.ctypes.data, None) == abi.ERR_INVALID
    # n_pixels == 0 does nothing
    info = abi.RenderInfo()
    info.cubes_traced = 99
    assert lib.aicb_render_layers_texture(aicb200.C.byref(layer), None, None, None, dptr, None, 0, None, None,
                                          aicb200.C.byref(info)) == abi.OK
    assert info.cubes_traced == 0
    rgba, depth, info = aicb200.render_layers_texture((rt, cam, opts), None, None, None, m,
                                                      pixels=np.zeros(0, np.uint32))
    assert rgba.shape == (0, 4) and depth.shape == (0,)
    rt.close()
