"""Blocks with more than 32768 palette entries on the GPU: a scene's brick pool takes u32 words for them (wide), from
aicb_scene_create or, when update_blocks / append_blocks places the first such block, by widening on the device.

Frames of a wide scene are checked two ways: against the round-once oracle (the frame's ColorBuf, depth, hit, steps,
sRGB8 and CharacterBuf, a layered sRGB8 frame, aicb_trace_rays), and byte for byte against the same Space holding the
block's twin, whose palette is deduplicated below 32768 entries and which is therefore drawn from a narrow pool (every
output, rgba16f, the texture and terminal targets with the wide scene as either layer, orthographic views).
tests/test_oracle_wide_palette.py shows that the oracle draws the two Spaces identically."""
import numpy as np
import pytest

import aicb200
import orc
import widepal
from aicb200 import (LIGHT_BOUNCE, LIGHT_FLAT, LIGHT_LINEAR, LIGHT_NONE, TRANSPARENCY_SURFACE, TRANSPARENCY_THRESHOLD,
                     TRANSPARENCY_VOLUMETRIC, AicbError, Block, GraphicsOptions, RtRenderer, Space, SpaceRaytracer, abi,
                     scenes)
from test_gpu_append_blocks import (DEVICES, NO_WORLD, OPTIONS, W, H, assert_same, every_output, narrow_space, placed,
                                    placements, wide_blocks)
from test_gpu_parity import compare

pytestmark = pytest.mark.gpu
BACKDROP = (0.1, 0.3, 0.6, 0.5)


@pytest.fixture(autouse=True, scope="module")
def _oracle_rounds_once():
    """The oracle of this module evaluates powf / expf in f64 and rounds once, like the device."""
    prev = orc.get_libm()
    orc.set_libm(orc.LIBM_CR)
    yield
    orc.set_libm(prev)


@pytest.fixture(scope="module")
def wide64():
    return widepal.wide_block(11, 64, 40000)


@pytest.fixture(scope="module")
def wide128():
    return widepal.wide_block(12, 128, 65536)


@pytest.fixture(scope="module")
def ui_space():
    return scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))


def ui_camera(space, opts):
    return scenes.standard_camera(space, opts, W, H, direction=(0.2, 0.1, 1.0), distance_scale=1.6)


def oracle_text(space, cam, opts):
    text = orc.OracleScene(space).render(cam, opts, accum_mode=1)["text"]
    return np.where(text == -4, -3, text)


def against_oracle(rt, space, opts, cam, label):
    """The frame outputs of `rt` (a scene of `space`) against the oracle; returns every output of the frame."""
    got = every_output(rt, opts, cam)
    ref = orc.OracleScene(space).render(cam, opts)
    compare(got, ref, label)
    assert np.array_equal(got["srgb8"].reshape(-1, 4), ref["srgb8"]), f"{label}: sRGB8 differs"
    assert np.array_equal(got["text"], oracle_text(space, cam, opts)), f"{label}: CharacterBuf differs"
    return got


def shows_wide_block(got, resolution):
    return (got["hit"][:, 6] == resolution).sum() > 50


def every_layer_output(rt, twin, opts, cam, other, ocam, oopts):
    """every_output of the scene and of its twin with `other` as the UI layer, and of `other` with each of them as the
    UI layer; rgba16f; all byte for byte."""
    assert_same(every_output(rt, opts, cam, (other, ocam, oopts)), every_output(twin, opts, cam, (other, ocam, oopts)),
                "wide scene as the world layer")
    got = every_output(other, oopts, ocam, (rt, cam, opts))
    want = every_output(other, oopts, ocam, (twin, cam, opts))
    assert_same(got, want, "wide scene as the UI layer")
    for s in (rt, twin):
        s.graphics_options = opts.repair()
    r1, r2 = RtRenderer(cam, rt.ctx), RtRenderer(cam, rt.ctx)
    r1.rt, r2.rt = rt, twin
    assert r1.draw_rgba16f().tobytes() == r2.draw_rgba16f().tobytes()


MATRIX = [(t, l) for t in (TRANSPARENCY_SURFACE, TRANSPARENCY_VOLUMETRIC, TRANSPARENCY_THRESHOLD)
          for l in (LIGHT_NONE, LIGHT_FLAT, LIGHT_LINEAR, LIGHT_BOUNCE)]


@pytest.mark.parametrize("transparency,lighting", MATRIX, ids=[f"t{t}-l{l}" for t, l in MATRIX])
def test_created_wide_scene_frames(wide64, ui_space, transparency, lighting):
    wide, twin = wide64
    ws, ts = widepal.space_with(wide), widepal.space_with(twin)
    opts = GraphicsOptions(view_distance=40.0, transparency=transparency, lighting_display=lighting,
                           transparency_threshold=0.3, bounce_samples=2)
    rt = SpaceRaytracer(ws, opts)
    trt = SpaceRaytracer(ts, opts, rt.ctx)
    uopts = GraphicsOptions(lighting_display=LIGHT_FLAT)
    urt = SpaceRaytracer(ui_space, uopts, rt.ctx)
    cam = scenes.standard_camera(ws, opts, W, H)
    ucam = ui_camera(ui_space, uopts)
    got = against_oracle(rt, ws, opts, cam, f"t{transparency} l{lighting}")
    assert shows_wide_block(got, 64)
    every_layer_output(rt, trt, opts, cam, urt, ucam, uopts)
    # the layered sRGB8 frame, the wide scene as either layer
    for world, ui, ow, ou in (((rt, cam, opts), (urt, ucam, uopts), (ws, cam, opts), (ui_space, ucam, uopts)),
                              ((urt, ucam, uopts), (rt, cam, opts), (ui_space, ucam, uopts), (ws, cam, opts))):
        frame = aicb200.render_layers(world, ui, BACKDROP, NO_WORLD).data.reshape(-1, 4)
        ref = orc.render_layers((orc.OracleScene(ow[0]), ow[1], ow[2]), (orc.OracleScene(ou[0]), ou[1], ou[2]),
                                BACKDROP, NO_WORLD)
        assert np.array_equal(frame, ref["srgb8"]), "layered sRGB8 differs"
    for s in (urt, trt, rt):
        s.close()


def test_created_wide_scene_65536_entries(wide128, ui_space):
    """A resolution-128 block that uses palette entry 65535: frames, orthographic views and aicb_trace_rays."""
    wide, twin = wide128
    ws, ts = widepal.space_with(wide), widepal.space_with(twin)
    uopts = GraphicsOptions(lighting_display=LIGHT_FLAT)
    for opts in OPTIONS:
        rt = SpaceRaytracer(ws, opts)
        trt = SpaceRaytracer(ts, opts, rt.ctx)
        urt = SpaceRaytracer(ui_space, uopts, rt.ctx)
        cam = scenes.standard_camera(ws, opts, W, H)
        got = against_oracle(rt, ws, opts, cam, f"res 128, t{opts.transparency}")
        assert shows_wide_block(got, 128)
        every_layer_output(rt, trt, opts, cam, urt, ui_camera(ui_space, uopts), uopts)
        ortho = aicb200.render_orthographic(rt, 2).data
        assert ortho.tobytes() == aicb200.render_orthographic(trt, 2).data.tobytes()
        rng = np.random.default_rng(3)
        lo, size = np.array(ws.lower, np.float64), np.array(ws.size, np.float64)
        o = lo + rng.uniform(-0.5, 1.5, (3000, 3)) * size
        target = lo + rng.uniform(0.6, 1.0, (3000, 3)) * size   # towards the wide block's cubes
        rays = np.concatenate([o, target - o], axis=1)
        g = rt.trace_rays(rays, want_depth=True, want_hit=True, want_steps=True)
        compare(g, orc.OracleScene(ws).trace_rays(rays, opts), "trace_rays")
        assert (g["hit"][:, 6] == 128).sum() > 50
        for s in (urt, trt, rt):
            s.close()


def test_update_blocks_widens_the_pool(wide64):
    """A narrow scene whose block at an id in use is redefined as a wide block: every output equals a scene created
    with the wide block, and the oracle."""
    wide, _ = wide64
    ws = widepal.space_with(wide)
    wid = len(ws.blocks) - 1
    narrow = widepal.space_with(scenes.make_voxel_block(5, resolution=16, alpha=0.5))
    opts = OPTIONS[0]
    rt = SpaceRaytracer(narrow, opts)
    before = rt.device_bytes
    rt.update_blocks([wid], [wide])
    assert rt.device_bytes > before
    fresh = SpaceRaytracer(ws, opts, rt.ctx)
    for o in OPTIONS:
        cam = scenes.standard_camera(ws, o, W, H)
        got = against_oracle(rt, ws, o, cam, f"widened by update_blocks, t{o.transparency}")
        assert shows_wide_block(got, 64)
        assert_same(got, every_output(fresh, o, cam), "fresh wide scene")
    fresh.close()
    rt.close()


def test_append_blocks_widens_the_pool(wide64):
    """A narrow scene that appends a wide block, then places it: every output equals a fresh scene and the oracle."""
    wide, _ = wide64
    base = scenes.small_mixed_scene(n=8, seed=7)
    opts = OPTIONS[0]
    rt = SpaceRaytracer(base, opts)
    rt.append_blocks([wide])
    wid = len(base.blocks)
    at = np.array([(7, 7, 7), (7, 5, 6), (6, 7, 4), (5, 6, 7)], np.int32) + np.array(base.lower, np.int32)
    ids = np.full(len(at), wid, np.uint16)
    rt.update_cubes(at, ids)
    final = placed(base, base.blocks + [wide], at, ids)
    fresh = SpaceRaytracer(final, opts, rt.ctx)
    assert rt.device_bytes == fresh.device_bytes
    for o in OPTIONS:
        cam = scenes.standard_camera(final, o, W, H)
        got = against_oracle(rt, final, o, cam, f"widened by append_blocks, t{o.transparency}")
        assert shows_wide_block(got, 64)
        assert_same(got, every_output(fresh, o, cam), "fresh wide scene")
    fresh.close()
    rt.close()


def test_append_widens_the_cells_and_the_pool(wide64):
    """One append past 16384 ids that holds a wide block: the cells become u32 and the pool wide in the same call."""
    wide, _ = wide64
    space = narrow_space()
    new = wide_blocks() + [wide]
    n0 = len(space.blocks)
    wid = n0 + len(new) - 1
    opts = GraphicsOptions(view_distance=80.0)
    rt = SpaceRaytracer(space, opts)
    rt.append_blocks(new)
    cubes, ids = placements(space, [16000, 16300, n0, 16384, n0 + 5, wid, wid, wid], 120, seed=5)
    near = np.array([(9, 9, 9), (9, 8, 7), (8, 9, 6), (7, 7, 9), (9, 6, 8)], np.int32) + np.array(space.lower, np.int32)
    cubes, ids = np.concatenate([cubes, near]), np.concatenate([ids, np.full(len(near), wid, np.uint16)])   # in view
    rt.update_cubes(cubes, ids)
    final = placed(space, space.blocks + new, cubes, ids)
    fresh = SpaceRaytracer(final, opts, rt.ctx)
    assert rt.device_bytes == fresh.device_bytes
    for o in (opts, GraphicsOptions(view_distance=80.0, transparency=TRANSPARENCY_SURFACE, lighting_display=LIGHT_FLAT)):
        cam = scenes.standard_camera(space, o, 96, 64)
        got = against_oracle(rt, final, o, cam, "cells and pool widened")
        assert shows_wide_block(got, 64) and got["text"].max() >= 16384
        assert_same(got, every_output(fresh, o, cam), "fresh wide scene")
    fresh.close()
    rt.close()


def test_unused_wide_block_leaves_frames_unchanged(wide64, ui_space):
    """Widening the pool re-encodes every brick word: a narrow scene's outputs are byte-identical before and after."""
    wide, _ = wide64
    space = scenes.small_mixed_scene(n=12, seed=7)
    uopts = GraphicsOptions(lighting_display=LIGHT_FLAT)
    rt = SpaceRaytracer(space, OPTIONS[0])
    urt = SpaceRaytracer(ui_space, uopts, rt.ctx)
    ucam = ui_camera(ui_space, uopts)
    cams = [scenes.standard_camera(space, o, W, H) for o in OPTIONS]
    before = [every_output(rt, o, c, (urt, ucam, uopts)) for o, c in zip(OPTIONS, cams)]
    narrow_bytes = rt.device_bytes
    rt.append_blocks([wide])
    assert rt.device_bytes > narrow_bytes + 64 ** 3 * 4 - 1
    for o, c, b in zip(OPTIONS, cams, before):
        assert_same(every_output(rt, o, c, (urt, ucam, uopts)), b, f"after widening, t{o.transparency}")
    urt.close()
    rt.close()


def test_redefinitions_compact_and_fill_uniform_narrows(wide64, wide128):
    """Redefinitions of a wide scene's blocks compact its wide pool: device_bytes stays within a fresh scene's plus its
    voxel data once more.  fill_uniform builds a narrow table again, unless its one block needs a wide one."""
    defs = [wide64[0], widepal.wide_block(21, 64, 33000)[0], widepal.wide_block(22, 32, 50000)[0]]
    space = widepal.space_with(defs[0])
    wid = len(space.blocks) - 1
    opts = OPTIONS[0]
    rt = SpaceRaytracer(space, opts)
    blocks = list(space.blocks)

    def with_blocks(bl):
        return Space(space.lower, space.block_ids, list(bl), light=space.light, sky_colors=space.sky_colors)

    bare = SpaceRaytracer(with_blocks([Block.air()] * len(blocks)), opts, rt.ctx)
    bare_bytes = bare.device_bytes
    bare.close()
    rng = np.random.default_rng(4)
    drops, last = 0, None
    for k in range(24):
        i = wid if k % 2 == 0 else int(rng.integers(1, wid))
        b = defs[(k // 2 + 1) % 3] if i == wid else scenes.make_voxel_block(200 + k, resolution=int(rng.choice([4, 16])))
        rt.update_blocks([i], [b])
        blocks[i] = b
        fresh = SpaceRaytracer(with_blocks(blocks), opts, rt.ctx)
        assert rt.device_bytes <= fresh.device_bytes + (fresh.device_bytes - bare_bytes), f"redefinition {k}"
        fresh.close()
        drops += last is not None and rt.device_bytes < last
        last = rt.device_bytes
    assert drops >= 2, "fewer compactions than expected"
    fresh = SpaceRaytracer(with_blocks(blocks), opts, rt.ctx)
    for o in OPTIONS:
        cam = scenes.standard_camera(space, o, W, H)
        assert_same(every_output(rt, o, cam), every_output(fresh, o, cam), f"after redefinitions, t{o.transparency}")
    fresh.close()
    # fill_uniform: a narrow block gives a narrow pool (2 bytes per word), a wide one a wide pool
    for block in (scenes.make_voxel_block(9, resolution=16), wide128[0]):
        rt.fill_uniform(block)
        uniform = Space(space.lower, np.zeros_like(space.block_ids), [block], light=space.light,
                        sky_colors=space.sky_colors)
        fresh = SpaceRaytracer(uniform, opts, rt.ctx)
        assert rt.device_bytes == fresh.device_bytes
        cam = scenes.standard_camera(space, opts, W, H)
        assert_same(every_output(rt, opts, cam), every_output(fresh, opts, cam), "after fill_uniform")
        fresh.close()
    rt.close()


def light_space(block):
    s = widepal.space_with(block)
    return Space(s.lower, s.block_ids, s.blocks, light=None, sky_colors=s.sky_colors, light_max_distance=30)


def test_light_propagation_equals_the_twin(wide64):
    wide, twin = wide64
    fields = []
    for b in (wide, twin):
        rt = SpaceRaytracer(light_space(b), GraphicsOptions())
        rt.light_fast_evaluate()
        rt.light_evaluate(0)
        fields.append(rt.light_download())
        rt.close()
    assert np.array_equal(fields[0], fields[1])


@pytest.mark.parametrize("devices", DEVICES, ids=[str(d) for d in DEVICES])
def test_group(wide64, devices):
    """A group scene created wide, and one widened by append_blocks and by update_blocks: the frames of a single
    context; light propagation on a wide group scene: every replica equal to the twin's field."""
    wide, twin = wide64
    ws = widepal.space_with(wide)
    wid = len(ws.blocks) - 1
    narrow = widepal.space_with(scenes.make_voxel_block(5, resolution=16, alpha=0.5))
    opts = OPTIONS[0]
    cam = scenes.standard_camera(ws, opts, W, H)
    rt = SpaceRaytracer(ws, opts)
    want = aicb200.render_layers((rt, cam, opts), None, BACKDROP, NO_WORLD).data
    want_t = aicb200.render_layers_terminal((rt, cam, opts), None, None, NO_WORLD)
    g = aicb200.DeviceGroup(devices)
    created, updated, appended = g.add_scene(ws), g.add_scene(narrow), g.add_scene(narrow)
    updated.update_blocks([wid], [wide])
    appended.append_blocks([wide])
    appended.update_cubes(*_all_cubes_of(narrow, wid, wid + 1))
    for gs in (created, updated, appended):
        assert np.array_equal(g.render_layers((gs, cam, opts), None, BACKDROP, NO_WORLD).data, want)
        got_t = g.render_layers_terminal((gs, cam, opts), None, None, NO_WORLD)
        # `appended` holds the wide block at the next id
        assert np.array_equal(np.where(got_t["text"] == wid + 1, wid, got_t["text"]), want_t["text"])
        assert np.array_equal(got_t["rgba"], want_t["rgba"])
    g.close()
    rt.close()
    tw = SpaceRaytracer(light_space(twin), GraphicsOptions())
    tw.light_fast_evaluate()
    tw.light_evaluate(0)
    field = tw.light_download()
    tw.close()
    g = aicb200.DeviceGroup(devices)
    gs = g.add_scene(light_space(wide))
    gs.light_fast_evaluate()
    gs.light_evaluate(0)
    for i in range(len(devices)):
        assert np.array_equal(gs.light_download(i), field), f"replica {i}"
    g.close()


def _all_cubes_of(space, old_id, new_id):
    """Every cube of `space` that holds old_id, with new_id for each."""
    cubes = (np.argwhere(space.block_ids == old_id) + np.array(space.lower)).astype(np.int32)
    return cubes, np.full(len(cubes), new_id, np.uint16)


def test_rejected_palettes_change_nothing(wide64):
    """A palette of 65537 entries cannot be indexed by a u16 VoxelIndex: AICB_ERR_UNSUPPORTED from create, update and
    append, on a narrow and a wide scene and on a group, with the same frames and device_bytes afterwards."""
    wide, _ = wide64
    pal = np.zeros((65537, 8), np.float32)
    pal[:, :4] = (0.5, 0.4, 0.3, 1.0)
    idx = np.zeros((4, 4, 4), np.uint16)
    idx[1, 2, 3] = 65535
    bad = Block(resolution=4, indices=idx, palette=pal)
    opts = OPTIONS[0]

    def unsupported(call):
        with pytest.raises(AicbError) as e:
            call()
        assert e.value.status == abi.ERR_UNSUPPORTED

    unsupported(lambda: SpaceRaytracer(widepal.space_with(bad), opts))
    for block in (scenes.make_voxel_block(5, resolution=16), wide):
        space = widepal.space_with(block)
        wid = len(space.blocks) - 1
        cam = scenes.standard_camera(space, opts, W, H)
        rt = SpaceRaytracer(space, opts)
        before, nbytes = every_output(rt, opts, cam), rt.device_bytes
        unsupported(lambda: rt.update_blocks([wid], [bad]))
        unsupported(lambda: rt.append_blocks([Block(color=(0.1, 0.2, 0.3, 1.0)), bad]))
        assert rt.device_bytes == nbytes
        assert_same(every_output(rt, opts, cam), before, "after the rejected calls")
        g = aicb200.DeviceGroup([0, 0])
        gs = g.add_scene(space)
        frame = g.render_layers((gs, cam, opts)).data
        unsupported(lambda: gs.update_blocks([wid], [bad]))
        unsupported(lambda: gs.append_blocks([bad]))
        assert np.array_equal(g.render_layers((gs, cam, opts)).data, frame)
        assert np.array_equal(frame, aicb200.render_layers((rt, cam, opts)).data)
        g.close()
        rt.close()
