"""Layered frames and RaytraceToTexture targets on a device group (aicb_group_render_layers_*), and group scenes kept
current (aicb_group_scene_update_blocks / _upload_light): every output must equal the single-context call's byte for
byte.  One H100 is enough: the same device is named several times, each name its own context."""
import ctypes as C
import re

import numpy as np
import pytest

import aicb200
from aicb200 import (FOG_NONE, LIGHT_BOUNCE, LIGHT_FLAT, LIGHT_NONE, TRANSPARENCY_VOLUMETRIC, AicbError, Block, Context,
                     GraphicsOptions, RtRenderer, SpaceRaytracer, abi, scenes)
from test_gpu_resolve import faint_slab

pytestmark = pytest.mark.gpu

DEVICES = ([0], [0, 0], [0, 0, 0])
NO_WORLD = aicb200.srgb8_to_linear((0xBC, 0xBC, 0xBC)) + (1.0,)
CASES = [
    dict(world=True, ui=True, backdrop=(0.1, 0.3, 0.6, 0.5)),
    dict(world=True, ui=True, backdrop=None),
    dict(world=True, ui=False, backdrop=(0.9, 0.2, 0.1, 0.25)),
    dict(world=False, ui=True, backdrop=(0.0, 0.5, 0.0, 0.3)),   # NO_WORLD_TO_SHOW
    dict(world=False, ui=True, backdrop=None),                   # NO_WORLD_TO_SHOW
]
W, H = 64, 45   # 45 rows: not a multiple of 16 x devices (nor of the 4-row tile)


@pytest.fixture(scope="module")
def spaces():
    return scenes.small_mixed_scene(n=12, seed=7), scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))


def setup(world_space, ui_space, aa, debug=False, w=W, h=H, bounce=False):
    # bounce: the world layer with LightingOption::Bounce, whose frames run a secondary pass per sample
    lighting = dict(lighting_display=LIGHT_BOUNCE, bounce_samples=2) if bounce else {}
    wopts = GraphicsOptions(view_distance=40.0, antialiasing_always=aa, exposure=1.75, debug_pixel_cost=debug,
                            **lighting)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT, exposure=0.625,
                            antialiasing_always=aa)
    wcam = scenes.standard_camera(world_space, wopts, w, h)
    ucam = scenes.standard_camera(ui_space, uopts, w, h, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    return wopts, uopts, wcam, ucam


def layers(c, world, ui):
    return (world if c["world"] else None), (ui if c["ui"] else None)


def same_info(a, b):
    return a.cubes_traced == b.cubes_traced and a.rays == b.rays


@pytest.mark.parametrize("aa,debug,bounce", [(False, False, False), (True, False, False), (False, True, False),
                                             (False, False, True)],
                         ids=["False-False", "True-False", "False-True", "bounce"])
def test_layered_frames_equal_the_single_context_frame(spaces, aa, debug, bounce):
    mixed, ui_space = spaces
    wopts, uopts, wcam, ucam = setup(mixed, ui_space, aa, debug, bounce=bounce)
    wrt = SpaceRaytracer(mixed, wopts)
    urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
    alone = [aicb200.render_layers(*layers(c, (wrt, wcam, wopts), (urt, ucam, uopts)), c["backdrop"], NO_WORLD)
             for c in CASES]
    for devices in DEVICES:
        g = aicb200.DeviceGroup(devices)
        gw, gu = g.add_scene(mixed), g.add_scene(ui_space)
        for c, ref in zip(CASES, alone):
            got = g.render_layers(*layers(c, (gw, wcam, wopts), (gu, ucam, uopts)), c["backdrop"], NO_WORLD)
            assert np.array_equal(got.data, ref.data), f"{devices} aa={aa} debug={debug} bounce={bounce} {c}"
            assert same_info(got.info, ref.info), f"{devices} {c}"
        g.close()
    if bounce:   # the world alone, no backdrop, no paint: the frame of aicb_render_srgb8 (with the sky)
        r = RtRenderer(wcam, wrt.ctx)
        r.update(mixed)
        assert np.array_equal(aicb200.render_layers((wrt, wcam, wopts)).data, r.draw().data)
        r.rt.close()
    urt.close()
    wrt.close()


@pytest.mark.parametrize("aa,bounce", [(False, False), (True, False), (False, True)], ids=["False", "True", "bounce"])
def test_texture_targets_equal_the_single_context_texels(spaces, aa, bounce):
    mixed, ui_space = spaces
    wopts, uopts, wcam, ucam = setup(mixed, ui_space, aa, bounce=bounce)
    wrt = SpaceRaytracer(mixed, wopts)
    urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
    m = wcam.depth_transform()
    n = W * H
    rng = np.random.default_rng(5)
    # None = the whole texture; a PixelPicker batch; shuffled with repeats; fewer than 32; fewer than 32 x 3
    batches = [None, aicb200.pixel_picker_order(W, H, 1000), rng.integers(0, n, size=777).astype(np.uint32),
               rng.permutation(n)[:20].astype(np.uint32), rng.integers(0, n, size=70).astype(np.uint32)]
    runs = [(c, None) for c in CASES] + [(CASES[0], px) for px in batches[1:]]
    alone = [aicb200.render_layers_texture(*layers(c, (wrt, wcam, wopts), (urt, ucam, uopts)), c["backdrop"], NO_WORLD,
                                           m, pixels=px) for c, px in runs]
    for devices in DEVICES:
        g = aicb200.DeviceGroup(devices)
        gw, gu = g.add_scene(mixed), g.add_scene(ui_space)
        for (c, px), (rgba, depth, info) in zip(runs, alone):
            got = g.render_layers_texture(*layers(c, (gw, wcam, wopts), (gu, ucam, uopts)), c["backdrop"], NO_WORLD, m,
                                          pixels=px)
            label = f"{devices} aa={aa} bounce={bounce} {c} {'whole' if px is None else len(px)}"
            assert np.array_equal(got[0], rgba), label
            assert np.array_equal(got[1].view(np.uint32), depth.view(np.uint32)), label
            assert same_info(got[2], info), label
        rgba, depth, info = g.render_layers_texture((gw, wcam, wopts), (gu, ucam, uopts), None, NO_WORLD, m,
                                                    pixels=np.zeros(0, np.uint32))
        assert rgba.shape == (0, 4) and depth.shape == (0,) and info.rays == 0
        g.close()
    urt.close()
    wrt.close()


PASS_LINE = re.compile(r"^\[aicb200\] gen .*\(hits (\d+)\)$", re.M)


@pytest.mark.parametrize("lighting", [LIGHT_NONE, LIGHT_FLAT])
def test_world_pass_overflow_is_reissued_alone(spaces, lighting, monkeypatch, capfd):
    """19-65 surfaces per ray in the world layer: every device's first world pass overflows the hit stream of its fresh
    context and only that pass is issued again; the UI pass (about one surface per ray) is issued once per device.
    AICB_PROFILE_KERNELS makes each finished pass print one line."""
    _, ui_space = spaces
    world = faint_slab()
    wopts = GraphicsOptions(lighting_display=lighting, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT)
    w, h = 128, 96   # every device's share of the frame has more hits than its first stream (>= 65536 slots) holds
    wcam = scenes.standard_camera(world, wopts, w, h, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    ucam = scenes.standard_camera(ui_space, uopts, w, h, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    m = wcam.depth_transform()
    bd = (0.1, 0.3, 0.6, 0.5)
    monkeypatch.setenv("AICB_PROFILE_KERNELS", "1")
    capfd.readouterr()
    ctx = Context()
    wrt = SpaceRaytracer(world, wopts, ctx)
    urt = SpaceRaytracer(ui_space, uopts, ctx)
    ref = aicb200.render_layers((wrt, wcam, wopts), (urt, ucam, uopts), bd, NO_WORLD)
    hits = [int(v) for v in PASS_LINE.findall(capfd.readouterr().err)]
    assert len(hits) >= 3 and min(hits[1:]) > 2 * hits[0], hits   # UI once, then the world until it fits
    assert ref.info.counters[2] > 8 * ref.info.rays
    ctx2 = Context()
    wrt2, urt2 = SpaceRaytracer(world, wopts, ctx2), SpaceRaytracer(ui_space, uopts, ctx2)
    ref_tex = aicb200.render_layers_texture((wrt2, wcam, wopts), (urt2, ucam, uopts), bd, NO_WORLD, m)
    capfd.readouterr()
    for devices in DEVICES[1:]:
        n = len(devices)
        for texture in (False, True):
            g = aicb200.DeviceGroup(devices)
            gw, gu = g.add_scene(world), g.add_scene(ui_space)
            if texture:
                rgba, depth, info = g.render_layers_texture((gw, wcam, wopts), (gu, ucam, uopts), bd, NO_WORLD, m)
                assert np.array_equal(rgba, ref_tex[0]) and np.array_equal(depth.view(np.uint32), ref_tex[1].view(np.uint32))
            else:
                got = g.render_layers((gw, wcam, wopts), (gu, ucam, uopts), bd, NO_WORLD)
                assert np.array_equal(got.data, ref.data)
                info = got.info
            assert info.cubes_traced == ref.info.cubes_traced
            hits = [int(v) for v in PASS_LINE.findall(capfd.readouterr().err)]
            # pass-major: the n UI passes, the n world passes that overflowed, then only world passes again
            assert len(hits) >= 3 * n, f"{devices} texture={texture}: {hits}"
            assert min(hits[n:]) > 2 * max(hits[:n]), f"{devices} texture={texture}: {hits}"
            g.close()
    for s in (wrt, urt, wrt2, urt2):
        s.close()
    ctx.close()
    ctx2.close()


def test_update_blocks_and_upload_light_equal_a_fresh_snapshot(spaces):
    mixed, ui_space = spaces
    wopts, uopts, wcam, ucam = setup(mixed, ui_space, False)
    blocks = list(mixed.blocks)
    singles = [i for i, b in enumerate(blocks) if i and b.indices is None and not b.is_air]
    voxels = [i for i, b in enumerate(blocks) if b.indices is not None]
    new = {singles[0]: Block(color=(0.2, 0.9, 0.4, 1.0)),                          # recoloured
           singles[1]: scenes.make_voxel_block(11, resolution=8, alpha=0.5),      # single voxel -> brick
           voxels[0]: Block(color=(0.0, 0.0, 0.0, 0.0))}                          # brick -> invisible single voxel
    for i, b in new.items():
        blocks[i] = b
    changed = aicb200.Space(mixed.lower, mixed.block_ids, blocks, light=mixed.light, sky_colors=mixed.sky_colors)
    light = np.random.default_rng(9).integers(0, 256, size=mixed.light.shape).astype(np.uint8)
    light[..., 3] = 255
    relit = aicb200.Space(mixed.lower, mixed.block_ids, blocks, light=light, sky_colors=mixed.sky_colors)
    bd = (0.1, 0.3, 0.6, 0.5)
    fresh = []
    for space in (changed, relit):
        wrt = SpaceRaytracer(space, wopts)
        urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
        fresh.append(aicb200.render_layers((wrt, wcam, wopts), (urt, ucam, uopts), bd, NO_WORLD))
        urt.close()
        wrt.close()
    assert not np.array_equal(fresh[0].data, fresh[1].data)
    for devices in DEVICES:
        g = aicb200.DeviceGroup(devices)
        gw, gu = g.add_scene(mixed), g.add_scene(ui_space)
        gw.update_blocks(list(new.keys()), list(new.values()))
        got = g.render_layers((gw, wcam, wopts), (gu, ucam, uopts), bd, NO_WORLD)
        assert np.array_equal(got.data, fresh[0].data), f"{devices} after update_blocks"
        gw.upload_light(light)
        got = g.render_layers((gw, wcam, wopts), (gu, ucam, uopts), bd, NO_WORLD)
        assert np.array_equal(got.data, fresh[1].data), f"{devices} after upload_light"
        g.close()


def test_rejected_input_changes_no_replica(spaces):
    mixed, ui_space = spaces
    wopts, uopts, wcam, ucam = setup(mixed, ui_space, False)
    m = wcam.depth_transform()
    g, other = aicb200.DeviceGroup([0, 0]), aicb200.DeviceGroup([0, 0])
    gw, gu, ou = g.add_scene(mixed), g.add_scene(ui_space), other.add_scene(ui_space)
    bd = (0.1, 0.3, 0.6, 0.5)
    before = g.render_layers((gw, wcam, wopts), (gu, ucam, uopts), bd, NO_WORLD)

    def rejected(call):
        with pytest.raises(AicbError) as e:
            call()
        assert e.value.status == abi.ERR_INVALID

    # layers from two groups
    rejected(lambda: g.render_layers((gw, wcam, wopts), (ou, ucam, uopts), bd, NO_WORLD))
    rejected(lambda: g.render_layers_texture((gw, wcam, wopts), (ou, ucam, uopts), bd, NO_WORLD, m))
    # a length mismatch
    lib = aicb200.load_library()
    o = wopts.to_abi(True)
    layer = abi.GroupLayer(gw.handle, C.pointer(wcam.data), C.pointer(o))
    out = np.zeros((W * H, 4), dtype=np.uint8)
    assert lib.aicb_group_render_layers_srgb8(C.byref(layer), None, None, None, out.ctypes.data, W * H - 1,
                                              None) == abi.ERR_INVALID
    rgba, depth = np.zeros((W * H, 4), dtype=np.uint16), np.zeros(W * H, dtype=np.float32)
    mm = np.ascontiguousarray(m, dtype=np.float64).reshape(16)
    assert lib.aicb_group_render_layers_texture(C.byref(layer), None, None, None, mm.ctypes.data_as(C.POINTER(C.c_double)),
                                                None, W * H - 1, rgba.ctypes.data, depth.ctypes.data,
                                                None) == abi.ERR_INVALID
    # a pixel index beyond the framebuffer
    rejected(lambda: g.render_layers_texture((gw, wcam, wopts), None, None, None, m,
                                             pixels=np.array([3, W * H], np.uint32)))
    # an update_blocks index beyond the table, after a valid one: nothing is applied to any replica
    rejected(lambda: gw.update_blocks([1, len(mixed.blocks)], [Block(color=(1.0, 0.0, 0.0, 1.0))] * 2))
    # a light volume of the wrong size
    rejected(lambda: gw.upload_light(np.zeros((5, 4), np.uint8)))
    after = g.render_layers((gw, wcam, wopts), (gu, ucam, uopts), bd, NO_WORLD)
    assert np.array_equal(after.data, before.data)
    assert after.info.cubes_traced == before.info.cubes_traced   # (both replicas drew strips of it)
    g.close()
    other.close()
