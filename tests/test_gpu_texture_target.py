"""aicb_texture_target_* / aicb_group_texture_target_* — RaytraceToTexture's update strategy, dirty_pixels and render
targets kept on the device (raytrace_to_texture.rs) — against the restated PixelPicker (aicb200.pixel_picker_order,
pinned in test_texture_picker.py), the texture oracle (oracle_texture/) and a host model of the state.  Everything is
compared exactly: pick indices, texel bits, counters."""
import ctypes as C

import numpy as np
import pytest

import aicb200
import orc
import texorc
from aicb200 import (TEXTURE_CONSISTENT, TEXTURE_INCREMENTAL, AicbError, Context, DeviceGroup, GraphicsOptions,
                     SpaceRaytracer, TextureTarget, abi, scenes)
from test_gpu_texture import NO_WORLD, layer_setup, same_texels

pytestmark = pytest.mark.gpu

BACKDROP = (0.1, 0.3, 0.6, 0.5)


@pytest.fixture(autouse=True, scope="module")
def _oracle_rounds_once():
    prev = orc.get_libm()
    orc.set_libm(orc.LIBM_CR)
    texorc.set_libm(texorc.LIBM_CR)
    yield
    orc.set_libm(prev)


def cycle_length(w, h, strategy=TEXTURE_INCREMENTAL):
    n = w * h
    c = min(aicb200.CENTRAL_PIXEL_LIMIT, n // 4)
    return 2 * max(c, n - c) if strategy == TEXTURE_INCREMENTAL else n


def planned_picks(w, h, strategy, start, n):
    if strategy == TEXTURE_CONSISTENT:
        return aicb200.consistent_picks(w, h, start, n)
    return aicb200.pixel_picker_order(w, h, start + n)[start:]


@pytest.mark.parametrize("size", [(1, 1), (3, 2), (17, 9), (64, 48), (640, 360), (1920, 1080), (3840, 2160)])
def test_incremental_picks_equal_pixel_picker(size):
    w, h = size
    t = TextureTarget(w, h, TEXTURE_INCREMENTAL)
    try:
        k = 2 * cycle_length(w, h)
        want = aicb200.pixel_picker_order(w, h, k)
        assert np.array_equal(t.picks(0, k), want)
        # from the middle of the sequence, as a batch starts
        s = k // 2 + 1
        assert np.array_equal(t.picks(s, min(1000, k - s)), want[s:s + 1000])
        st = t.state
        assert (st["width"], st["height"], st["strategy"]) == (w, h, TEXTURE_INCREMENTAL)
        assert st["cycle_length"] == cycle_length(w, h) == st["dirty_pixels"] and st["next_pick"] == 0
    finally:
        t.close()


def test_consistent_picks_wrap_like_point_from_pixel_index():
    for w, h in [(1, 1), (17, 9), (640, 360)]:
        t = TextureTarget(w, h, TEXTURE_CONSISTENT)
        n = w * h
        for start in (0, max(n - 5, 1), 3 * n + 1, 2 ** 40 + 11):
            assert np.array_equal(t.picks(start, 40), aicb200.consistent_picks(w, h, start, 40)), (w, h, start)
        assert t.state["cycle_length"] == n
        t.close()


class HostModel:
    """RaytraceToTexture::Inner on the host: the state and the two targets, filled from the oracle's texels."""

    def __init__(self, w, h, strategy):
        self.w, self.h, self.strategy = w, h, strategy
        self.rgba = np.zeros((w * h, 4), np.uint16)
        self.depth = np.zeros(w * h, np.float32)
        self.next = 0
        self.dirty = cycle_length(w, h, strategy)

    def trace(self, oracle_layers, m, n):
        if self.dirty == 0:
            return 0, 0
        px = planned_picks(self.w, self.h, self.strategy, self.next, n)
        total = 0
        if n:
            rgba, depth, total = texorc.render_layers_texture(*oracle_layers, m, pixels=px)
            self.rgba[px] = rgba      # a pixel picked twice has the same bits both times
            self.depth[px] = depth
        self.next += n
        self.dirty -= min(n, self.dirty)
        return n, total

    def check(self, t):
        st = t.state
        assert (st["dirty_pixels"], st["next_pick"]) == (self.dirty, self.next)
        rgba, depth = t.read()
        assert rgba.shape == (self.h, self.w, 4) and depth.shape == (self.h, self.w)
        assert same_texels(rgba.reshape(-1, 4), depth.reshape(-1), self.rgba, self.depth)


def scenes_for(ui):
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0)) if ui else None
    return mixed, ui_space


def run_batches(t, gpu_layers, oracle_layers, m, model, steps):
    """`steps`: batch sizes, or "dirty" for mark_dirty; after each call the target equals the model."""
    for step in steps:
        if step == "dirty":
            t.mark_dirty()
            model.dirty = cycle_length(model.w, model.h, model.strategy)
        else:
            was_clean = model.dirty == 0
            before = t.read() if was_clean else None
            traced, info = t.trace(*gpu_layers, m, step)
            want, total = model.trace(oracle_layers, m, step)
            assert traced == want, step
            assert info.cubes_traced == total, step
            if was_clean:   # nothing traced, not a byte changed
                after = t.read()
                assert np.array_equal(before[0], after[0]) and np.array_equal(before[1].view(np.uint32),
                                                                             after[1].view(np.uint32))
        model.check(t)


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("ui", [False, True])
def test_batches_equal_the_oracle_stored_in_pick_order(ui, aa):
    mixed, ui_space = scenes_for(ui)
    wopts, uopts, wcam, ucam = layer_setup(mixed, ui_space or mixed, aa)
    ctx = Context()
    wrt = SpaceRaytracer(mixed, wopts, ctx)
    urt = SpaceRaytracer(ui_space, uopts, ctx) if ui else None
    try:
        m = wcam.depth_transform()
        gpu_layers = ((wrt, wcam, wopts), (urt, ucam, uopts) if ui else None, BACKDROP, NO_WORLD)
        oracle_layers = ((texorc.Scene(mixed), wcam, wopts),
                         (texorc.Scene(ui_space), ucam, uopts) if ui else None, BACKDROP, NO_WORLD)
        w, h = wcam.data.fb_width, wcam.data.fb_height
        cyc = cycle_length(w, h)
        for strategy in (TEXTURE_INCREMENTAL, TEXTURE_CONSISTENT):
            t = TextureTarget(w, h, strategy, ctx)
            c = cycle_length(w, h, strategy)
            model = HostModel(w, h, strategy)
            model.check(t)   # cleared targets
            steps = [1, 31, 700, cyc + 5, 9, 0, "dirty", 0, 64, c, 40, "dirty", 2 * c + 3]
            run_batches(t, gpu_layers, oracle_layers, m, model, steps)
            t.close()
    finally:
        for rt in (wrt, urt):
            if rt:
                rt.close()
        ctx.close()


def test_resize_makes_a_new_order_and_cleared_targets():
    mixed, _ = scenes_for(False)
    opts = GraphicsOptions(view_distance=40.0, exposure=1.75)
    ctx = Context()
    rt = SpaceRaytracer(mixed, opts, ctx)
    try:
        orc_scene = texorc.Scene(mixed)
        for strategy in (TEXTURE_INCREMENTAL, TEXTURE_CONSISTENT):
            cam = scenes.standard_camera(mixed, opts, 64, 48)
            t = TextureTarget(64, 48, strategy, ctx)
            model = HostModel(64, 48, strategy)
            run_batches(t, ((rt, cam, opts), None, None, NO_WORLD), ((orc_scene, cam, opts), None, None, NO_WORLD),
                        cam.depth_transform(), model, [500])
            # the same size: nothing changes, not even the device buffers
            bufs = t.tensors()
            t.resize(64, 48)
            model.check(t)
            assert t.tensors()[0].data_ptr() == bufs[0].data_ptr()
            # another size: cleared targets, a new order (Incremental from pick 0), dirty_pixels as it was
            dirty, nxt = model.dirty, model.next
            t.resize(40, 30)
            st = t.state
            assert (st["width"], st["height"], st["dirty_pixels"]) == (40, 30, dirty)
            assert st["next_pick"] == (0 if strategy == TEXTURE_INCREMENTAL else nxt)
            assert st["cycle_length"] == cycle_length(40, 30, strategy)
            rgba, depth = t.read()
            assert not rgba.any() and not depth.view(np.uint32).any()
            assert np.array_equal(t.picks(0, 3000), planned_picks(40, 30, strategy, 0, 3000))
            model2 = HostModel(40, 30, strategy)
            model2.dirty, model2.next = st["dirty_pixels"], st["next_pick"]
            cam2 = scenes.standard_camera(mixed, opts, 40, 30)
            run_batches(t, ((rt, cam2, opts), None, None, NO_WORLD), ((orc_scene, cam2, opts), None, None, NO_WORLD),
                        cam2.depth_transform(), model2, [333, "dirty", 1000])
            t.close()
    finally:
        rt.close()
        ctx.close()


def test_tensors_are_the_targets_in_place():
    torch = pytest.importorskip("torch")
    mixed, _ = scenes_for(False)
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(mixed, opts, 64, 48)
    ctx = Context()
    rt = SpaceRaytracer(mixed, opts, ctx)
    try:
        t = TextureTarget(64, 48, TEXTURE_INCREMENTAL, ctx)
        rgba_t, depth_t = t.tensors()
        assert rgba_t.dtype == torch.uint16 and tuple(rgba_t.shape) == (48, 64, 4)
        assert depth_t.dtype == torch.float32 and tuple(depth_t.shape) == (48, 64)
        assert rgba_t.device == torch.device("cuda", ctx.device_id)
        t.trace((rt, cam, opts), None, None, NO_WORLD, cam.depth_transform(), 2000)
        rgba, depth = t.read()
        assert np.array_equal(rgba_t.cpu().numpy(), rgba)   # the tensors see what the trace wrote
        assert np.array_equal(depth_t.cpu().numpy().view(np.uint32), depth.view(np.uint32))
        t.close()
    finally:
        rt.close()
        ctx.close()


def group_device_lists():
    import torch
    n = torch.cuda.device_count()
    lists = [[0], [0, 0], list(range(n))]
    return [d for i, d in enumerate(lists) if d not in lists[:i]]


def test_a_group_equals_one_context():
    mixed, ui_space = scenes_for(True)
    wopts, uopts, wcam, ucam = layer_setup(mixed, ui_space, False)
    m = wcam.depth_transform()
    w, h = wcam.data.fb_width, wcam.data.fb_height
    steps = [1, 31, 700, 2000, "dirty", 96]

    def run(make_target, layers):
        t = make_target()
        out = []
        for s in steps:
            if s == "dirty":
                t.mark_dirty()
            else:
                traced, info = t.trace(*layers, m, s)
                rgba, depth = t.read()
                out.append((traced, info.cubes_traced, t.state, rgba, depth.view(np.uint32)))
        t.resize(40, 30)
        out.append((t.state, t.read()[0], t.picks(0, 500)))
        t.close()
        return out

    for strategy in (TEXTURE_INCREMENTAL, TEXTURE_CONSISTENT):
        ctx = Context()
        wrt = SpaceRaytracer(mixed, wopts, ctx)
        urt = SpaceRaytracer(ui_space, uopts, ctx)
        one = run(lambda: TextureTarget(w, h, strategy, ctx), ((wrt, wcam, wopts), (urt, ucam, uopts), BACKDROP,
                                                               NO_WORLD))
        wrt.close()
        urt.close()
        ctx.close()
        for devices in group_device_lists():
            g = DeviceGroup(devices)
            gw, gu = g.add_scene(mixed), g.add_scene(ui_space)
            got = run(lambda: g.texture_target(w, h, strategy), ((gw, wcam, wopts), (gu, ucam, uopts), BACKDROP,
                                                                 NO_WORLD))
            for a, b in zip(one, got):
                for x, y in zip(a, b):
                    if isinstance(x, np.ndarray):
                        assert np.array_equal(x, y), devices
                    else:
                        assert x == y, devices
            g.close()


def test_invalid_arguments():
    mixed, _ = scenes_for(False)
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(mixed, opts, 64, 48)
    m = cam.depth_transform()
    lib = aicb200.load_library()
    ctx, other = Context(), Context()
    rt = SpaceRaytracer(mixed, opts, ctx)
    rt_other = SpaceRaytracer(mixed, opts, other)
    try:
        for w, h in [(0, 48), (64, 0), (0, 0), (65536, 65536)]:
            with pytest.raises(AicbError) as e:
                TextureTarget(w, h, TEXTURE_INCREMENTAL, ctx)
            assert e.value.status == abi.ERR_INVALID
        with pytest.raises(AicbError) as e:
            TextureTarget(64, 48, 0, ctx)
        assert e.value.status == abi.ERR_INVALID
        t = TextureTarget(64, 48, TEXTURE_INCREMENTAL, ctx)
        before = t.state
        bad_cam = scenes.standard_camera(mixed, opts, 48, 64)   # the same pixel count, another size
        for layers in [((rt, bad_cam, opts), None), ((rt_other, cam, opts), None), (None, None)]:
            with pytest.raises(AicbError) as e:
                t.trace(layers[0], layers[1], None, None, m, 10)
            assert e.value.status == abi.ERR_INVALID
        with pytest.raises(AicbError) as e:    # no depth transform
            t.trace((rt, cam, opts), None, None, NO_WORLD, None, 10)
        assert e.value.status == abi.ERR_INVALID
        assert t.state == before
        # NULL handles and outputs
        h = C.c_void_p()
        assert lib.aicb_texture_target_create(None, 4, 4, TEXTURE_INCREMENTAL, C.byref(h)) == abi.ERR_INVALID
        assert lib.aicb_texture_target_create(ctx.handle, 4, 4, TEXTURE_INCREMENTAL, None) == abi.ERR_INVALID
        assert lib.aicb_texture_target_resize(None, 4, 4) == abi.ERR_INVALID
        assert lib.aicb_texture_target_mark_dirty(None) == abi.ERR_INVALID
        assert lib.aicb_texture_target_state(t.handle, None) == abi.ERR_INVALID
        assert lib.aicb_texture_target_picks(t.handle, 0, 5, None) == abi.ERR_INVALID
        d0 = C.c_void_p()
        assert lib.aicb_texture_target_buffers(t.handle, None, C.byref(d0)) == abi.ERR_INVALID
        assert lib.aicb_texture_target_read(t.handle, None, None, 10) == abi.ERR_INVALID
        assert lib.aicb_texture_target_trace(None, None, None, None, None, None, 1, None, None) == abi.ERR_INVALID
        assert lib.aicb_group_texture_target_create(None, 4, 4, TEXTURE_INCREMENTAL, C.byref(h)) == abi.ERR_INVALID
        with pytest.raises(AicbError) as e:
            t.resize(0, 5)
        assert e.value.status == abi.ERR_INVALID
        assert t.state == before   # a rejected resize changes nothing
        t.close()
    finally:
        rt.close()
        rt_other.close()
        ctx.close()
        other.close()


def test_group_layers_must_be_of_the_targets_group():
    mixed, _ = scenes_for(False)
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(mixed, opts, 64, 48)
    g1, g2 = DeviceGroup([0]), DeviceGroup([0])
    try:
        s2 = g2.add_scene(mixed)
        t = g1.texture_target(64, 48)
        with pytest.raises(AicbError) as e:
            t.trace((s2, cam, opts), None, None, NO_WORLD, cam.depth_transform(), 10)
        assert e.value.status == abi.ERR_INVALID
    finally:
        g1.close()
        g2.close()
