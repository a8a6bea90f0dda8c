"""The world-only outputs of one context on a device group (aicb_group_render_colorbuf / _rgba16f / _text /
_orthographic and aicb_group_trace_rays): each must equal the single-context call on a fresh SpaceRaytracer of the same
Space bit for bit, outputs and counters.  One H100 is enough: the same device is named several times, each name its own
context."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import aicb200
from aicb200 import (FOG_PHYSICAL, LIGHT_BOUNCE, LIGHT_LINEAR, AicbError, Block, GraphicsOptions, RtRenderer,
                     SpaceRaytracer, Space, abi, scenes)

pytestmark = pytest.mark.gpu

DEVICES = ([0], [0, 0], [0, 0, 0])
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def spaces():
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    return {
        "mixed": mixed,
        "c2": scenes.config_c2(n=16, n_voxel_blocks=6),                       # mixed transparent, res-1 and res-16
        "res16": scenes.config_c1(n=16, n_voxel_blocks=8, resolution=16),    # resolution-16 voxel blocks
        "box": Space(mixed.lower, np.ascontiguousarray(mixed.block_ids[:5, :9, :7]), mixed.blocks),   # not a cube
    }


def same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def same_counts(a, b):
    return (a.cubes_traced, a.rays, a.counters, a.algorithmic_bytes) == \
        (b.cubes_traced, b.rays, b.counters, b.algorithmic_bytes)


def text_of(fn, handle, cam, opts):
    w, h = cam.data.fb_width, cam.data.fb_height
    out = np.zeros(w * h, dtype=np.int32)
    info = abi.RenderInfo()
    o = opts.to_abi(True)
    assert fn(handle, C.byref(cam.data), C.byref(o), out.ctypes.data, out.size, C.byref(info)) == abi.OK
    return out, aicb200.RenderInfo.from_abi(info)


# (space, options, framebuffer size)
FRAMES = {
    "c2": ("c2", {}, (48, 40)),
    "res16": ("res16", {}, (40, 33)),
    "aa": ("mixed", dict(antialiasing_always=True), (40, 33)),
    "debug_pixel_cost": ("mixed", dict(debug_pixel_cost=True), (40, 33)),
    "bounce": ("mixed", dict(lighting_display=LIGHT_BOUNCE, bounce_samples=2), (40, 33)),
    "linear_fog": ("mixed", dict(lighting_display=LIGHT_LINEAR, fog=FOG_PHYSICAL), (40, 33)),
    "odd_37x23": ("mixed", dict(antialiasing_always=True), (37, 23)),       # the last strip is partial
    "20_rows": ("c2", {}, (41, 20)),                                        # 3 devices: the third has no strip
    "5_rows": ("mixed", {}, (29, 5)),                                       # one strip: only device 0 draws
}


@pytest.mark.parametrize("case", list(FRAMES))
def test_frames_equal_the_single_context_frames(spaces, case):
    name, kw, (w, h) = FRAMES[case]
    space = spaces[name]
    opts = GraphicsOptions(view_distance=40.0, exposure=1.5, **kw)
    cam = scenes.standard_camera(space, opts, w, h)
    r = RtRenderer(cam)
    r.update(space)
    ref_cb = r.draw_colorbuf()
    ref_16 = r.draw_rgba16f()
    ref_text, ref_text_info = text_of(aicb200.load_library().aicb_render_text, r.rt.handle, cam, opts)
    assert ref_cb["info"].rays == w * h * (4 if kw.get("antialiasing_always") else 1)
    for devices in DEVICES:
        g = aicb200.DeviceGroup(devices)
        g.update(space)
        got = g.draw_colorbuf(cam, cam.options)
        for k in ("colorbuf", "depth", "hit", "steps"):
            assert same_bits(got[k], ref_cb[k]), f"{case} {devices} {k}"
        assert same_counts(got["info"], ref_cb["info"]), f"{case} {devices}"
        assert same_bits(g.draw_rgba16f(cam, cam.options), ref_16), f"{case} {devices} rgba16f"
        text, info = text_of(aicb200.load_library().aicb_group_render_text, g.scene.handle, cam, cam.options)
        assert np.array_equal(text, ref_text), f"{case} {devices} text"
        assert same_counts(info, ref_text_info), f"{case} {devices} text"
        assert np.array_equal(g.render_text(cam, cam.options).ravel(), ref_text)
        # outputs the caller does not want are neither stored nor returned; the others are unchanged
        some = g.draw_colorbuf(cam, cam.options, want_depth=False, want_hit=True, want_steps=False)
        assert some["depth"] is None and some["steps"] is None
        assert same_bits(some["colorbuf"], ref_cb["colorbuf"]) and same_bits(some["hit"], ref_cb["hit"])
        g.close()
    r.rt.close()


def ray_batch(space, n, seed):
    """Rays from around and inside the Space in every direction, some axis-aligned and some of zero length."""
    rng = np.random.default_rng(seed)
    lo, size = np.array(space.lower, np.float64), np.array(space.size, np.float64)
    o = lo + rng.uniform(-0.5, 1.5, size=(n, 3)) * size
    d = rng.normal(size=(n, 3))
    axis = rng.integers(0, 3, size=n)
    aligned = rng.random(n) < 0.2
    d[aligned] = 0.0
    d[aligned, axis[aligned]] = rng.choice([-1.0, 1.0], size=aligned.sum())
    d[rng.random(n) < 0.01] = 0.0
    return np.concatenate([o, d], axis=1)


WANTS = [(a, b, c) for a in (False, True) for b in (False, True) for c in (False, True)]


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 95, 100_003])
def test_ray_batches_equal_the_single_context_batch(spaces, n):
    space = spaces["mixed"]
    opts = GraphicsOptions(view_distance=40.0)
    rays = ray_batch(space, n, seed=n + 1)
    rt = SpaceRaytracer(space, opts)
    refs = {(sky, want): rt.trace_rays(rays, sky, *want) for sky in (True, False) for want in WANTS}
    for devices in DEVICES:
        g = aicb200.DeviceGroup(devices)
        g.update(space)
        for (sky, want), ref in refs.items():
            got = g.trace_rays(rays, rt.graphics_options, sky, *want)
            for k in ("colorbuf", "depth", "hit", "steps"):
                assert same_bits(got[k], ref[k]), f"n={n} {devices} sky={sky} want={want} {k}"
            assert same_counts(got["info"], ref["info"]), f"n={n} {devices} sky={sky} want={want}"
        g.close()
    rt.close()


def test_print_space_through_a_group_scene(spaces):
    """raytracer/text.rs:196-258, 265-341: the reference's two 80x40 golden images through aicb_group_render_text, and a
    mixed Space's image equal to the single-context one."""
    golden = json.load(open(os.path.join(GOLDEN, "text_images.json")))
    grey = lambda i, n: (i / (n - 1),) * 3 + (1.0,) if n > 1 else (0.5, 0.5, 0.5, 1.0)
    ramp = Space((0, 0, 0), np.array([1, 2, 3], dtype=np.uint16).reshape(3, 1, 1),
                 [Block.air()] + [Block(color=grey(i, 3)) for i in range(3)])
    idx = np.zeros((4, 2, 4), dtype=np.uint16)
    pal = np.zeros((1, 8), dtype=np.float32)
    pal[0, :4] = (1, 1, 1, 1)
    partial = Space((0, 0, 0), np.array([1, 2], dtype=np.uint16).reshape(2, 1, 1),
                    [Block.air(), Block(color=grey(0, 1)), Block(resolution=4, indices=idx, palette=pal)])
    mixed = spaces["mixed"]
    chars = {i: chr(ord("a") + i % 26) for i in range(len(mixed.blocks))}
    alone = aicb200.print_space(mixed, (1.0, 0.4, -0.7), chars)
    for devices in DEVICES:
        g = aicb200.DeviceGroup(devices)
        for space, c, want in ((ramp, {1: "0", 2: "1", 3: "2"}, golden["print_space_test"]),
                               (partial, {1: "0", 2: "P"}, golden["partial_voxels"]),
                               (mixed, chars, alone)):
            g.update(space)
            assert aicb200.print_space(space, (1.0, 1.0, 1.0) if space is not mixed else (1.0, 0.4, -0.7), c,
                                       g.scene) == want, f"{devices}"
        g.close()


@pytest.mark.parametrize("res", [1, 16, 32])
def test_orthographic_images_equal_the_single_context_image(spaces, res):
    for name in ("mixed", "box"):
        space = spaces[name]
        rt = SpaceRaytracer(space, GraphicsOptions.unaltered_colors())
        ref = aicb200.render_orthographic(rt, res)
        sx, sy, sz = (space.size[a] * res for a in range(3))
        assert ref.size == (sz + sx + sz + 2, sz + sy + sz + 2)
        assert (ref.data[sz, :, 3] == 0).all() and (ref.data[:, sz, 3] == 0).all()   # the gaps are transparent
        assert (ref.data[:sz, :sz] == 0).all()                                         # and the corners
        assert ref.info.rays == sx * sz * 2 + sy * (sz * 2 + sx)
        for devices in DEVICES:
            g = aicb200.DeviceGroup(devices)
            g.update(space)
            w, h, gw, gh = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
            lib = aicb200.load_library()
            assert lib.aicb_ortho_image_size(rt.handle, res, C.byref(w), C.byref(h)) == abi.OK
            assert lib.aicb_group_ortho_image_size(g.scene.handle, res, C.byref(gw), C.byref(gh)) == abi.OK
            assert (gw.value, gh.value) == (w.value, h.value) == ref.size
            img = g.render_orthographic(res)
            assert img.size == ref.size
            assert np.array_equal(img.data, ref.data), f"{name} res={res} {devices}"
            assert same_counts(img.info, ref.info), f"{name} res={res} {devices}"
            g.close()
        rt.close()


def test_rejected_input_changes_nothing(spaces):
    space = spaces["mixed"]
    opts = GraphicsOptions(view_distance=40.0)
    w, h = 40, 33
    cam = scenes.standard_camera(space, opts, w, h)
    g = aicb200.DeviceGroup([0, 0])
    g.update(space)
    before = g.draw_colorbuf(cam, cam.options)
    before_ortho = g.render_orthographic(4)
    lib = aicb200.load_library()
    gs = g.scene.handle
    n = w * h
    o = cam.options.to_abi(True)
    bad = GraphicsOptions(view_distance=40.0, fog=99).to_abi(True)   # validate_options rejects it
    cb, depth = np.zeros((n, 4), np.float32), np.zeros(n, np.float64)
    hit, steps = np.zeros((n, 8), np.int32), np.zeros(n, np.uint32)
    px16, text, srgb = np.zeros((n, 4), np.uint16), np.zeros(n, np.int32), np.zeros((4 * n, 4), np.uint8)
    rays = ray_batch(space, 64, seed=3)
    info = abi.RenderInfo()

    def colorbuf(opt, out, length):
        return lib.aicb_group_render_colorbuf(gs, C.byref(cam.data), C.byref(opt), out, depth.ctypes.data,
                                              hit.ctypes.data, steps.ctypes.data, length, C.byref(info))

    def trace(opt, src, out, count):
        return lib.aicb_group_trace_rays(gs, src, count, C.byref(opt), out, None, None, None, None)

    calls = [
        colorbuf(o, cb.ctypes.data, n - 1), colorbuf(o, None, n), colorbuf(bad, cb.ctypes.data, n),
        lib.aicb_group_render_colorbuf(gs, None, C.byref(o), cb.ctypes.data, None, None, None, n, None),
        lib.aicb_group_render_rgba16f(gs, C.byref(cam.data), C.byref(o), px16.ctypes.data, n + 1, None),
        lib.aicb_group_render_rgba16f(gs, C.byref(cam.data), C.byref(o), None, n, None),
        lib.aicb_group_render_rgba16f(gs, C.byref(cam.data), C.byref(bad), px16.ctypes.data, n, None),
        lib.aicb_group_render_text(gs, C.byref(cam.data), C.byref(o), text.ctypes.data, 0, None),
        lib.aicb_group_render_text(gs, C.byref(cam.data), C.byref(o), None, n, None),
        lib.aicb_group_render_text(gs, C.byref(cam.data), C.byref(bad), text.ctypes.data, n, None),
        trace(o, None, cb.ctypes.data, 64), trace(o, rays.ctypes.data, None, 64), trace(bad, rays.ctypes.data,
                                                                                        cb.ctypes.data, 64),
        lib.aicb_group_trace_rays(None, rays.ctypes.data, 64, C.byref(o), cb.ctypes.data, None, None, None, None),
    ]
    iw, ih = C.c_uint32(), C.c_uint32()
    for res in (0, 3, 12, 256):
        calls.append(lib.aicb_group_ortho_image_size(gs, res, C.byref(iw), C.byref(ih)))
        calls.append(lib.aicb_group_render_orthographic(gs, res, srgb.ctypes.data, 1, None))
    assert lib.aicb_group_ortho_image_size(gs, 4, C.byref(iw), C.byref(ih)) == abi.OK
    calls.append(lib.aicb_group_render_orthographic(gs, 4, srgb.ctypes.data, iw.value * ih.value - 1, None))
    calls.append(lib.aicb_group_render_orthographic(gs, 4, None, iw.value * ih.value, None))
    calls.append(lib.aicb_group_ortho_image_size(None, 4, C.byref(iw), C.byref(ih)))
    assert all(st == abi.ERR_INVALID for st in calls), calls
    # the same inputs on one context are rejected with the same status
    rt = SpaceRaytracer(space, opts)
    assert lib.aicb_render_colorbuf(rt.handle, C.byref(cam.data), C.byref(o), None, cb.ctypes.data, None, None, None,
                                    n - 1, None) == abi.ERR_INVALID
    assert lib.aicb_trace_rays(rt.handle, rays.ctypes.data, 64, C.byref(bad), cb.ctypes.data, None, None, None,
                               None) == abi.ERR_INVALID
    assert lib.aicb_render_orthographic(rt.handle, 3, srgb.ctypes.data, 1, None) == abi.ERR_INVALID
    rt.close()
    after = g.draw_colorbuf(cam, cam.options)
    for k in ("colorbuf", "depth", "hit", "steps"):
        assert same_bits(after[k], before[k]), k
    assert same_counts(after["info"], before["info"])
    assert np.array_equal(g.render_orthographic(4).data, before_ortho.data)
    with pytest.raises(AicbError):
        aicb200.DeviceGroup([0]).trace_rays(rays, opts)   # no scene yet
    g.close()
