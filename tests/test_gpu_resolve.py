"""resolve_kernel (None / Flat lighting: shading and compositing in one pass, one warp per 32 rays, hit lists in
shared-memory windows of 128 slots): frames in which a warp's hit lists span many windows, against the oracle, the
choice between it and shade_kernel + encode_kernel, and the stage times a frame reports.  Also: every blocking entry
point re-issues a frame that overflowed the hit stream and returns what the warmed context returns, and a context
gives an enlarged hit stream back after a run of shallow frames."""
import ctypes as C

import numpy as np
import pytest

import aicb200
import orc
from aicb200 import (LIGHT_BOUNCE, LIGHT_FLAT, LIGHT_LINEAR, LIGHT_NONE, TRANSPARENCY_SURFACE, TRANSPARENCY_VOLUMETRIC,
                     Block, Context, DeviceGroup, GraphicsOptions, RenderInfo, RtRenderer, Space, abi, scenes)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _oracle_rounds_once():
    prev = orc.get_libm()
    orc.set_libm(orc.LIBM_CR)
    yield
    orc.set_libm(prev)


def faint_slab():
    """40 x 24 x 24 cubes of two faint transparent blocks (alpha 0.03 / 0.02), seen end on from close by: every ray
    meets 19 to 65 surfaces and none becomes opaque, so a warp lists about a thousand slots and most lanes' lists
    straddle a window boundary."""
    n, m = 40, 24
    x, y, z = np.meshgrid(np.arange(n), np.arange(m), np.arange(m), indexing="ij")
    ids = (1 + (x + y + z) % 2).astype(np.uint16)
    return Space((0, 0, 0), ids, [Block.air(), Block(color=(0.9, 0.5, 0.2, 0.03)), Block(color=(0.2, 0.4, 0.9, 0.02))])


def _slab_rays(n=128):
    """n x n explicit rays along the faint slab's length: each crosses its 40 cubes."""
    y, z = np.meshgrid(np.linspace(0.25, 21.75, n), np.linspace(0.25, 21.75, n), indexing="ij")
    d = np.array([1.0, 0.04, 0.03]) / np.linalg.norm([1.0, 0.04, 0.03])
    return np.column_stack([np.full(n * n, -1.0), y.ravel(), z.ravel(), np.tile(d, (n * n, 1))])


def _blocking_call(call, r, group, cam, opts):
    """One blocking entry point on the faint slab: (its outputs, its RenderInfo)."""
    if call == "draw":
        img = r.draw()
    elif call == "draw_shard":
        img = r.draw(shard=(16, 1, 2))
    elif call == "orthographic":
        img = aicb200.render_orthographic(r.rt, 2)
    elif call == "group":
        img = group.draw(cam, opts)
    elif call == "draw_colorbuf" or call == "trace_rays":
        d = r.draw_colorbuf() if call == "draw_colorbuf" else r.rt.trace_rays(_slab_rays(), want_depth=True,
                                                                                want_hit=True, want_steps=True)
        return [d["colorbuf"], d["depth"], d["hit"], d["steps"]], d["info"]
    else:   # aicb_render_rgba16f and aicb_render_text (print_space's entry point): their wrappers drop the info
        lib, info, o, n = aicb200.load_library(), abi.RenderInfo(), r.rt.graphics_options.to_abi(True), r.pixel_count()
        if call == "draw_rgba16f":
            out = np.empty((n, 4), dtype=np.float16)
            st = lib.aicb_render_rgba16f(r.rt.handle, C.byref(cam.data), C.byref(o), None, out.ctypes.data, n,
                                         C.byref(info))
        else:
            out = np.empty(n, dtype=np.int32)
            st = lib.aicb_render_text(r.rt.handle, C.byref(cam.data), C.byref(o), out.ctypes.data, n, C.byref(info))
        assert st == abi.OK
        return [out], RenderInfo.from_abi(info)
    return [img.data], img.info


@pytest.mark.parametrize("call", ["draw", "draw_shard", "draw_rgba16f", "draw_colorbuf", "trace_rays", "orthographic",
                                  "text", "group"])
def test_blocking_call_reissues_an_overflowed_frame(call):
    """Every ray meets 19 to 65 surfaces of the faint slab, more than the 8 hit slots per ray (at least 65536 in all) of
    a fresh context's hit stream: the first frame overflows it, and the blocking call issues the frame again with a
    larger stream before it returns.  What it returns must equal the same call's on the warmed context.  `group` is
    the world-only frame of a two-context DeviceGroup on one device."""
    space = faint_slab()
    opts = GraphicsOptions(lighting_display=LIGHT_NONE, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0)
    cam = scenes.standard_camera(space, opts, 256, 192, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    ctx = Context()
    group = DeviceGroup([0, 0]) if call == "group" else None
    try:
        r = RtRenderer(cam, ctx)
        if group:
            group.update(space)
        else:
            r.update(space)
        first, info = _blocking_call(call, r, group, cam, opts)
        assert info.counters[2] > max(8 * info.rays, 1 << 16), info   # surface hits: more than the first stream held
        again, warm = _blocking_call(call, r, group, cam, opts)
        for a, b in zip(first, again):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), call
        assert (info.cubes_traced, info.rays, info.counters) == (warm.cubes_traced, warm.rays, warm.counters), call
        if r.rt:
            r.rt.close()
    finally:
        if group:
            group.close()
        ctx.close()


@pytest.mark.parametrize("lighting", [LIGHT_FLAT, LIGHT_BOUNCE])
def test_enlarged_hit_stream_is_given_back(lighting):
    """A faint-slab frame overflows a fresh context's hit stream and is re-issued with a larger one; after 16 shallow
    frames in a row the context gives the large hit and ShadedHit buffers back (with Bounce, those of the secondary rays'
    streams too) and lowers the capacity again.  Every shallow frame equals the same frame on a fresh context, and the
    faint-slab frame drawn once more, which overflows the lowered capacity and is re-issued, equals the first.  The
    shallow scene's blocks are opaque: at most one surface per primary ray and one per secondary ray, well under a
    sixteenth of the enlarged capacity per ray."""
    slab, mixed = faint_slab(), scenes.config_c0(n=16)
    opts = GraphicsOptions(lighting_display=lighting, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0)
    slab_cam = scenes.standard_camera(slab, opts, 128, 96, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    mixed_cam = scenes.standard_camera(mixed, opts, 64, 48)
    ctx, fresh = Context(), Context()
    renderers = []
    try:
        deep, shallow, ref = RtRenderer(slab_cam, ctx), RtRenderer(mixed_cam, ctx), RtRenderer(mixed_cam, fresh)
        renderers = [deep, shallow, ref]
        deep.update(slab)
        shallow.update(mixed)
        ref.update(mixed)
        first = deep.draw()
        assert first.info.counters[2] > max(8 * first.info.rays, 1 << 16), first.info   # it overflowed a fresh stream
        want = ref.draw()
        for _ in range(16):
            img = shallow.draw()
            assert np.array_equal(img.data, want.data)
            assert (img.info.cubes_traced, img.info.counters) == (want.info.cubes_traced, want.info.counters)
        again = deep.draw()
        assert np.array_equal(again.data, first.data)
        assert (again.info.cubes_traced, again.info.counters) == (first.info.cubes_traced, first.info.counters)
    finally:
        for r in renderers:
            if r.rt:
                r.rt.close()
        ctx.close()
        fresh.close()


@pytest.mark.parametrize("antialias", [False, True])
@pytest.mark.parametrize("transparency", [TRANSPARENCY_SURFACE, TRANSPARENCY_VOLUMETRIC])
@pytest.mark.parametrize("lighting", [LIGHT_NONE, LIGHT_FLAT])
def test_hit_lists_longer_than_a_window(lighting, transparency, antialias):
    """A frame after a shallow one runs resolve_kernel; having met many surfaces per ray, the next one runs
    shade_kernel + encode_kernel.  Both equal the oracle."""
    space = faint_slab()
    opts = GraphicsOptions(lighting_display=lighting, transparency=transparency, antialiasing_always=antialias,
                           view_distance=200.0)
    cam = scenes.standard_camera(space, opts, 64, 32, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    ref = orc.OracleScene(space).render(cam, opts)
    assert ref["steps"].min() >= 19
    ctx = Context()
    try:
        r = RtRenderer(cam, ctx)
        r.update(space)
        r.draw_colorbuf()   # overflows the hit stream once (the library re-issues it with a larger one)
        empty = RtRenderer(cam, ctx)
        empty.update(Space((0, 0, 0), np.zeros((4, 4, 4), dtype=np.uint16), [Block.air()]))
        empty.draw_colorbuf()   # no surfaces: the next frame is fused
        empty.rt.close()
        for fused in (True, False):
            gpu = r.draw_colorbuf()
            assert (gpu["info"].stage_ms[3] == 0.0) == fused
            assert gpu["info"].counters[2] > 16 * gpu["info"].rays   # surface hits: many windows per warp
            assert np.array_equal(gpu["hit"], ref["hit"])
            assert np.array_equal(gpu["steps"], ref["steps"])
            assert np.array_equal(gpu["depth"], ref["depth"])
            assert orc.max_ulp_diff(gpu["colorbuf"], ref["colorbuf"]) == 0
            assert gpu["info"].cubes_traced == ref["cubes_traced"]
        r.rt.close()
    finally:
        ctx.close()


def test_stage_times_of_fused_and_split_frames():
    """With None / Flat lighting the first frame of a context runs gen -> march -> resolve: stage_ms[2] is the resolve
    kernel and stage_ms[3] is 0.  Interpolated and Bounce lighting keep a separate encode kernel in stage_ms[3]."""
    space = scenes.small_mixed_scene(n=12, seed=7)
    for lighting, fused in ((LIGHT_NONE, True), (LIGHT_FLAT, True), (LIGHT_LINEAR, False), (LIGHT_BOUNCE, False)):
        opts = GraphicsOptions(lighting_display=lighting, view_distance=40.0)
        cam = scenes.standard_camera(space, opts, 64, 48)
        ctx = Context()
        try:
            r = RtRenderer(cam, ctx)
            r.update(space)
            img = r.draw()
            stage = img.info.stage_ms
            assert all(v > 0.0 for v in stage[:3]), stage
            assert (stage[3] == 0.0) == fused, stage
            r.rt.close()
        finally:
            ctx.close()
