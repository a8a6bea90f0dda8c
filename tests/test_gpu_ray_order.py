"""Ray order: a frame that repeats its context's previous frame's view and layout hands the marching kernel its rays in
order of the steps its tiles took then, and any other frame in order of the rays' chords.  The order is a scheduling
choice only, so every output of every output kind must be byte for byte the output of a fresh context, whatever frame
came before: one of the same view and layout (the order is used), one whose scene was edited since (the order is used,
one frame stale), a layered frame (its world pass, the last, has the same view and layout: the order is used), and a
moved camera, a different framebuffer size, a different shard or a texture batch (the chord order).  A layered frame's
own passes follow each other's scenes, so they use the chord order.  aicb_render_info::ray_order tells which order a
frame used.  On one context and on a device group of one."""
import ctypes as C

import numpy as np
import pytest

import aicb200
from aicb200 import Context, DeviceGroup, GraphicsOptions, SpaceRaytracer, TextureTarget, abi, scenes

pytestmark = pytest.mark.gpu

W, H = 96, 64
KINDS = ("srgb8", "colorbuf", "text")
EDIT_CUBES = np.array([[3, 4, 5], [8, 8, 8], [10, 2, 7]], dtype=np.int32)


@pytest.fixture(scope="module")
def setup():
    space = scenes.config_c2(n=16, n_voxel_blocks=6, with_light=True)
    opts = GraphicsOptions(view_distance=200.0)   # GraphicsOptions::default(): Volumetric, Linear light, fog
    cam = scenes.standard_camera(space, opts, W, H)
    moved = scenes.standard_camera(space, opts, W, H, direction=(1.0, 0.55, 1.05))
    other_size = scenes.standard_camera(space, opts, W + 8, H)
    ui = scenes.small_mixed_scene(n=6, seed=3)
    return space, opts, cam, moved, other_size, ui


def edit(scene, space, block):
    cubes = EDIT_CUBES + np.array(space.lower, dtype=np.int32)
    scene.update_cubes(cubes, np.full(len(cubes), block, dtype=np.uint16))


def frame(rt, cam, opts, kind, shard=None):
    """One frame of `kind` on a SpaceRaytracer: (outputs as bytes, cubes_traced, ray_order)."""
    lib = aicb200.load_library()
    s = abi.Shard(*shard) if shard else None
    sp = C.byref(s) if s else None
    n = lib.aicb_shard_pixel_count(C.byref(cam.data), sp)
    info = abi.RenderInfo()
    o = opts.to_abi(True)
    if kind == "colorbuf":
        cb, depth = np.empty((n, 4), np.float32), np.empty(n, np.float64)
        hit, steps = np.empty((n, 8), np.int32), np.empty(n, np.uint32)
        st = lib.aicb_render_colorbuf(rt.handle, C.byref(cam.data), C.byref(o), sp, cb.ctypes.data, depth.ctypes.data,
                                      hit.ctypes.data, steps.ctypes.data, n, C.byref(info))
        out = [cb, depth, hit, steps]
    elif kind == "srgb8":
        out = [np.empty((n, 4), np.uint8)]
        st = lib.aicb_render_srgb8(rt.handle, C.byref(cam.data), C.byref(o), sp, out[0].ctypes.data, n, C.byref(info))
    else:
        out = [np.empty(n, np.int32)]
        st = lib.aicb_render_text(rt.handle, C.byref(cam.data), C.byref(o), out[0].ctypes.data, n, C.byref(info))
    assert st == abi.OK, lib.aicb_last_error()
    return [a.tobytes() for a in out], int(info.cubes_traced), int(info.ray_order)


def group_frame(g, cam, opts, kind):
    """The same on a device group; its text call reports no info."""
    if kind == "colorbuf":
        r = g.draw_colorbuf(cam, opts)
        return [r[k].tobytes() for k in ("colorbuf", "depth", "hit", "steps")], r["info"].cubes_traced, r["info"].ray_order
    if kind == "srgb8":
        r = g.draw(cam, opts)
        return [r.data.tobytes()], r.info.cubes_traced, r.info.ray_order
    return [g.render_text(cam, opts).tobytes()], None, None


def check(got, ref, order, label):
    assert got[0] == ref[0], f"{label}: outputs differ"
    if got[1] is not None:
        assert got[1] == ref[1], f"{label}: cubes_traced {got[1]} != {ref[1]}"
        assert got[2] == order, f"{label}: ray_order {got[2]}, expected {order}"


def check_layered(r):
    assert r.info.ray_order == 0, "a layered frame's passes use the chord order"


def test_one_context(setup):
    space, opts, cam, moved, other_size, ui_space = setup

    def fresh(edited=False):
        ctx = Context(0)
        rt = SpaceRaytracer(space, opts, ctx)
        if edited:
            edit(rt, space, 0)
        return ctx, rt

    refs, refs_edited = {}, {}
    for kind in KINDS:
        ctx, rt = fresh()
        refs[kind] = frame(rt, cam, opts, kind)
        check(refs[kind], refs[kind], 0, f"fresh {kind}")
        ctx, rt = fresh(edited=True)
        refs_edited[kind] = frame(rt, cam, opts, kind)

    ctx, rt = fresh()
    ui = SpaceRaytracer(ui_space, opts, ctx)
    target = TextureTarget(W, H, aicb200.TEXTURE_INCREMENTAL, ctx)
    before = {
        "same layout": (lambda: frame(rt, cam, opts, "srgb8"), 1),
        "camera moved": (lambda: frame(rt, moved, opts, "colorbuf"), 0),
        "other size": (lambda: frame(rt, other_size, opts, "srgb8"), 0),
        "other shard": (lambda: frame(rt, cam, opts, "srgb8", shard=(4, 1, 2)), 0),
        "layered": (lambda: check_layered(aicb200.render_layers(world=(rt, cam, opts), ui=(ui, cam, opts))), 1),
        "texture batch": (lambda: target.trace(world=(rt, cam, opts), depth_transform=cam.depth_transform(),
                                                n=W * H // 3), 0),
    }
    for label, (prev, order) in before.items():
        for kind in KINDS:
            prev()
            check(frame(rt, cam, opts, kind), refs[kind], order, f"{label}, {kind}")
    for kind in KINDS:   # cubes edited after the frame whose steps order the rays
        edit(rt, space, 1)
        frame(rt, cam, opts, "srgb8")
        edit(rt, space, 0)
        check(frame(rt, cam, opts, kind), refs_edited[kind], 1, f"scene edited, {kind}")
    target.close()


def test_group_of_one(setup):
    space, opts, cam, moved, other_size, ui_space = setup

    def fresh():
        g = DeviceGroup([0])
        g.update(space)
        return g

    refs = {}
    for kind in KINDS:
        g = fresh()
        refs[kind] = group_frame(g, cam, opts, kind)
        check(refs[kind], refs[kind], 0, f"group: fresh {kind}")
        g.close()

    g = fresh()
    ui = g.add_scene(ui_space)
    target = g.texture_target(W, H)
    before = {
        "same layout": (lambda: group_frame(g, cam, opts, "srgb8"), 1),
        "camera moved": (lambda: group_frame(g, moved, opts, "colorbuf"), 0),
        "other size": (lambda: group_frame(g, other_size, opts, "srgb8"), 0),
        "layered": (lambda: check_layered(g.render_layers(world=(g.scene, cam, opts), ui=(ui, cam, opts))), 1),
        "texture batch": (lambda: target.trace(world=(g.scene, cam, opts), depth_transform=cam.depth_transform(),
                                                n=W * H // 3), 0),
    }
    for label, (prev, order) in before.items():
        for kind in KINDS:
            prev()
            check(group_frame(g, cam, opts, kind), refs[kind], order, f"group: {label}, {kind}")
    g.close()
