"""New block indices on a live scene (aicb_scene_append_blocks / aicb_group_scene_append_blocks): SpaceChange::BlockIndex
past the table, as UpdatingSpaceRaytracer::update appends TracingBlock::from_block for it (updating.rs:145-151).  Every
output of a scene that grew must equal, byte for byte, the output of a scene created with the longer table: frames of
every kind, light propagation through the new ids, group replicas, and a table that grows past 16384 blocks (u16 cells
re-encoded as u32 cells on the device)."""
import ctypes as C

import numpy as np
import pytest
import torch

import aicb200
import orc
from aicb200 import (FOG_NONE, LIGHT_FLAT, LIGHT_LINEAR, TRANSPARENCY_SURFACE, TRANSPARENCY_THRESHOLD,
                     TRANSPARENCY_VOLUMETRIC, AicbError, Block, GraphicsOptions, RtRenderer, Space, SpaceRaytracer, abi,
                     scenes)
from test_gpu_light import all_cubes, compare_fields, light_scene
from test_gpu_light_changes import cubes_set_opaque
from test_gpu_parity import compare, same_srgb8

pytestmark = pytest.mark.gpu
DEVICES = ([0], [0, 0], [0, 0, 0])
NO_WORLD = aicb200.srgb8_to_linear((0xBC, 0xBC, 0xBC)) + (1.0,)
OPTIONS = [GraphicsOptions(view_distance=40.0, transparency=TRANSPARENCY_VOLUMETRIC, lighting_display=LIGHT_LINEAR),
           GraphicsOptions(view_distance=40.0, transparency=TRANSPARENCY_SURFACE, lighting_display=LIGHT_FLAT),
           GraphicsOptions(view_distance=40.0, transparency=TRANSPARENCY_THRESHOLD, transparency_threshold=0.25)]
W, H = 64, 48


@pytest.fixture(autouse=True, scope="module")
def _oracle_rounds_once():
    """The oracle of this module evaluates powf / expf in f64 and rounds once, like the device."""
    prev = orc.get_libm()
    orc.set_libm(orc.LIBM_CR)
    yield
    orc.set_libm(prev)


@pytest.fixture(scope="module")
def spaces():
    return scenes.small_mixed_scene(n=12, seed=7), scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))


def new_blocks():
    """One of each kind a new palette entry can be."""
    brick = scenes.make_voxel_block(5, resolution=8, alpha=0.5)
    assert brick.voxel_lower != (0, 0, 0) and brick.voxel_size != (8, 8, 8)   # partial voxel_bounds
    return [Block(color=(0.9, 0.35, 0.1, 1.0)),      # opaque single voxel
            Block(color=(0.2, 0.5, 0.9, 0.375)),     # translucent single voxel
            brick,                                   # res-8 brick, alpha 0.5
            Block.air(),
            Block(color=(0.0, 0.0, 0.0, 0.0))]       # invisible (not AIR)


def placements(space, ids, n, seed):
    """n random cubes of `space` (some over blocks already there) with ids drawn from `ids`."""
    rng = np.random.default_rng(seed)
    cubes = np.stack([rng.integers(0, space.size[a], n) + space.lower[a] for a in range(3)], axis=1).astype(np.int32)
    filled = np.argwhere(space.block_ids != 0)[: n // 3] + np.array(space.lower)
    cubes[: len(filled)] = filled
    return cubes, rng.choice(np.asarray(ids, dtype=np.uint16), n).astype(np.uint16)


def placed(space, blocks, cubes, ids):
    """The Space a scene holds after the cube updates: what a fresh scene is created from."""
    out = space.block_ids.copy()
    for c, i in zip(cubes, ids):
        out[tuple(np.asarray(c) - np.array(space.lower))] = i
    return Space(space.lower, out, blocks, light=space.light, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


def text_of(rt, cam, opts):
    out = np.zeros(cam.data.fb_width * cam.data.fb_height, dtype=np.int32)
    o = opts.to_abi(True)
    assert aicb200.load_library().aicb_render_text(rt.handle, C.byref(cam.data), C.byref(o), out.ctypes.data, out.size,
                                                   None) == abi.OK
    return out


def every_output(rt, opts, cam, ui=None):
    """sRGB8, ColorBuf / depth / hit / steps, CharacterBuf, and a layered texture and terminal frame of `rt`."""
    rt.graphics_options = opts.repair()
    r = RtRenderer(cam, rt.ctx)
    r.rt = rt
    out = {"srgb8": r.draw().data, "text": text_of(rt, cam, opts)}
    cb = r.draw_colorbuf()
    out.update({k: cb[k] for k in ("colorbuf", "depth", "hit", "steps")})
    world = (rt, cam, opts)
    rgba, depth, _ = aicb200.render_layers_texture(world, ui, (0.1, 0.3, 0.6, 0.5), NO_WORLD, cam.depth_transform())
    term = aicb200.render_layers_terminal(world, ui, None, NO_WORLD)
    out.update({"tex_rgba": rgba, "tex_depth": depth, "term_text": term["text"], "term_layer": term["layer"],
                "term_rgba": term["rgba"]})
    return out


def assert_same(a, b, label=""):
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), f"{label}: {k} differs"


def test_append_place_render_equals_fresh_snapshot(spaces):
    mixed, ui_space = spaces
    new = new_blocks()
    n0 = len(mixed.blocks)
    rt = SpaceRaytracer(mixed, OPTIONS[0])
    urt = SpaceRaytracer(ui_space, GraphicsOptions(fog=FOG_NONE, lighting_display=LIGHT_FLAT), rt.ctx)
    rt.append_blocks(new)
    cubes, ids = placements(mixed, range(n0, n0 + len(new)), 80, seed=3)
    rt.update_cubes(cubes, ids)
    fresh = SpaceRaytracer(placed(mixed, mixed.blocks + new, cubes, ids), OPTIONS[0], rt.ctx)
    assert rt.device_bytes == fresh.device_bytes
    for opts in OPTIONS:
        cam = scenes.standard_camera(mixed, opts, W, H)
        ucam = scenes.standard_camera(ui_space, urt.graphics_options, W, H, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
        ui = (urt, ucam, urt.graphics_options)
        got, want = every_output(rt, opts, cam, ui), every_output(fresh, opts, cam, ui)
        assert_same(got, want, f"transparency {opts.transparency}")
        assert np.isin(got["text"], np.arange(n0, n0 + len(new))).any(), "no new block index in the CharacterBuf"
    for s in (fresh, urt, rt):
        s.close()


def test_many_small_appends_equal_fresh_snapshot(spaces):
    """300 appends of one block each: the device tables reallocate several times (geometric growth) on the way."""
    mixed, _ = spaces
    opts = OPTIONS[0]
    rt = SpaceRaytracer(mixed, opts)
    blocks = list(mixed.blocks)
    rng = np.random.default_rng(8)
    kinds = new_blocks()
    ids = mixed.block_ids.copy()
    for k in range(300):
        b = kinds[k % len(kinds)] if k % 7 else Block(color=tuple(rng.uniform(0.05, 1.0, 3)) + (1.0,))
        rt.append_blocks([b])
        blocks.append(b)
        if k % 3 == 0:
            cubes, new_ids = placements(mixed, [len(blocks) - 1, int(rng.integers(0, len(blocks)))], 4, seed=k)
            rt.update_cubes(cubes, new_ids)
            for c, i in zip(cubes, new_ids):
                ids[tuple(c - np.array(mixed.lower))] = i
    fresh = SpaceRaytracer(Space(mixed.lower, ids, blocks, light=mixed.light, sky_colors=mixed.sky_colors), opts, rt.ctx)
    assert rt.device_bytes == fresh.device_bytes
    cam = scenes.standard_camera(mixed, opts, W, H)
    assert_same(every_output(rt, opts, cam), every_output(fresh, opts, cam))
    rt.close()
    fresh.close()


def narrow_space(n_blocks=16380, n=10, seed=29):
    """A small Space with a table just below 16384 blocks (u16 cells), ids from every part of it."""
    rng = np.random.default_rng(seed)
    cols = rng.uniform(0.05, 1.0, (n_blocks, 3))
    blocks = [Block.air()] + [Block(color=(cols[i, 0], cols[i, 1], cols[i, 2], 0.5 if i % 7 == 0 else 1.0))
                              for i in range(1, n_blocks)]
    blocks[16300] = scenes.make_voxel_block(16300, resolution=8, alpha=0.5)
    h = scenes.grid_hash(31, (n, n, n))
    ids = np.where((h & np.uint64(7)) < 2, (h >> np.uint64(8)) % np.uint64(n_blocks), 0).astype(np.uint16)
    return Space((-2, 1, 0), ids, blocks, light=scenes.noise_light(5, ids, blocks), sky_colors=scenes.OCTANT_SKY)


def wide_blocks(n=40, seed=30):
    rng = np.random.default_rng(seed)
    cols = rng.uniform(0.05, 1.0, (n, 3))
    out = [Block(color=(cols[i, 0], cols[i, 1], cols[i, 2], (1.0, 0.5, 0.25)[i % 3])) for i in range(n)]
    out[5] = scenes.make_voxel_block(77, resolution=4, alpha=0.5)
    out[9] = Block(color=(0.0, 0.0, 0.0, 0.0))
    return out


def test_crossing_16384_blocks_widens_the_cells():
    """40 blocks appended to a table of 16380 in one call: the cells are re-encoded from u16 to u32 on the device.
    Every output equals a fresh wide scene and the oracle (0 ULP); further cube and block updates keep it so."""
    space = narrow_space()
    new = wide_blocks()
    n0 = len(space.blocks)
    opts = GraphicsOptions(view_distance=80.0)
    rt = SpaceRaytracer(space, opts)
    narrow_bytes = rt.device_bytes
    rt.append_blocks(new)
    assert rt.device_bytes > narrow_bytes + space.block_ids.size * 2 - 1   # the cells take 4 bytes each now
    blocks = space.blocks + new
    cubes, ids = placements(space, [16000, 16383, n0, 16384, 16385, n0 + 5, n0 + 9, n0 + 39], 120, seed=5)
    rt.update_cubes(cubes, ids)
    final = placed(space, blocks, cubes, ids)
    fresh = SpaceRaytracer(final, opts, rt.ctx)
    assert rt.device_bytes == fresh.device_bytes
    for o in (opts, GraphicsOptions(view_distance=80.0, transparency=TRANSPARENCY_SURFACE, lighting_display=LIGHT_FLAT)):
        cam = scenes.standard_camera(space, o, 96, 64)
        got = every_output(rt, o, cam)
        assert_same(got, every_output(fresh, o, cam), "fresh wide scene")
        ref = orc.OracleScene(final).render(cam, o)
        compare(got, ref, "appended past 16384")
        rendering = aicb200.Rendering((96, 64), got["srgb8"], 0, None)
        same_srgb8(rendering, ref)
        text = orc.OracleScene(final).render(cam, o, accum_mode=1)["text"]
        assert np.array_equal(got["text"], np.where(text == -4, -3, text))
        assert got["text"].max() >= 16384
    # SpaceChange::CubeBlock and BlockEvaluation on the widened scene
    cubes2, ids2 = placements(space, [3, n0 + 1, n0 + 20, 16384], 40, seed=6)
    rt.update_cubes(cubes2, ids2)
    changed = {n0 + 1: scenes.make_voxel_block(12, resolution=8, alpha=1.0), 16384: Block(color=(0.3, 0.8, 0.2, 1.0)),
               100: Block(color=(0.0, 0.0, 0.0, 0.0))}
    rt.update_blocks(list(changed), list(changed.values()))
    blocks2 = list(blocks)
    for i, b in changed.items():
        blocks2[i] = b
    again = SpaceRaytracer(placed(final, blocks2, cubes2, ids2), opts, rt.ctx)
    cam = scenes.standard_camera(space, opts, 96, 64)
    assert_same(every_output(rt, opts, cam), every_output(again, opts, cam), "updates after widening")
    for s in (again, fresh, rt):
        s.close()


@pytest.mark.parametrize("widen", [False, True], ids=["reallocate", "widen"])
def test_append_while_a_frame_is_in_flight(spaces, widen):
    """A frame issued before an append that moves the device tables (or widens the cells) is the frame of the table
    it was issued on."""
    space = narrow_space() if widen else spaces[0]
    new = wide_blocks() if widen else new_blocks()
    opts = GraphicsOptions(view_distance=80.0)
    cam = scenes.standard_camera(space, opts, 320, 240)
    rt = SpaceRaytracer(space, opts)
    r = RtRenderer(cam, rt.ctx)
    r.rt = rt
    before = r.draw().data.reshape(-1, 4)
    lib = aicb200.load_library()
    n = cam.data.fb_width * cam.data.fb_height
    d_out = torch.zeros((n, 4), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    o = opts.to_abi(True)
    assert lib.aicb_render_srgb8_device(rt.handle, C.byref(cam.data), C.byref(o), None, d_out.data_ptr(), n,
                                        C.c_void_p(stream.cuda_stream)) == abi.OK
    rt.append_blocks(new)   # every device table moves: the scene was created with exact-size tables
    info = abi.RenderInfo()
    assert lib.aicb_render_finish(rt.handle, C.byref(info)) == abi.OK
    torch.cuda.synchronize()
    assert np.array_equal(d_out.cpu().numpy(), before)
    after = r.draw().data.reshape(-1, 4)   # nothing holds a new id yet
    assert np.array_equal(after, before)
    rt.close()


def test_light_edits_place_appended_blocks():
    """On a converged light scene: append an emissive and an opaque block, place them with a propagating edit."""
    space = light_scene(seed=9)
    new = [Block(color=(0.1, 0.1, 0.1, 1.0), emission=(3.0, 1.5, 0.5)), Block(color=(0.7, 0.6, 0.9, 1.0))]
    n0 = len(space.blocks)
    longer = Space(space.lower, space.block_ids, space.blocks + new, light=space.light, sky_colors=space.sky_colors,
                   light_max_distance=space.light_max_distance)
    rt = SpaceRaytracer(space, GraphicsOptions())
    rt.light_fast_evaluate()
    rt.light_evaluate(0)
    rt.light_take_changes(discard=True)
    before = rt.light_download()
    rt.append_blocks(new)
    cubes, ids = placements(space, [n0, n0 + 1, n0, 0, 2], 40, seed=11)
    updates, _ = rt.light_edit_and_propagate(cubes, ids, 0)
    assert updates > 0
    field = rt.light_download()
    # compute_light on the edited cubes and their neighbours, against the resulting field, is the oracle's
    edited = placed(longer, longer.blocks, cubes, ids)
    near = {tuple(c + d) for c in cubes for d in [(0, 0, 0)] + [tuple(v) for v in np.vstack([np.eye(3), -np.eye(3)]).astype(int)]}
    lo, hi = np.array(space.lower), np.array(space.lower) + np.array(space.size)
    near = np.array([c for c in sorted(near) if (np.array(c) >= lo).all() and (np.array(c) < hi).all()], dtype=np.int32)
    on_field = orc.OracleLight(Space(edited.lower, edited.block_ids, edited.blocks, light=field,
                                     sky_colors=space.sky_colors, light_max_distance=space.light_max_distance))
    assert np.array_equal(rt.light_compute(near), on_field.compute(near))
    # the converged field meets the light contract against the same edits on a scene created with the longer table
    ol = orc.OracleLight(longer)
    ol.fast_evaluate()
    ol.evaluate(0)
    ol.set_cubes(cubes, ids)
    ol.evaluate(0)
    compare_fields(field, ol.field())
    fresh = SpaceRaytracer(longer, GraphicsOptions(), rt.ctx)
    fresh.light_fast_evaluate()
    fresh.light_evaluate(0)
    fresh.light_edit_and_propagate(cubes, ids, 0)
    compare_fields(field, fresh.light_download())
    # SpaceChange::CubeLight lists the edited cubes
    idx, tx = rt.light_take_changes()
    taken = set(idx.tolist())
    changed = np.flatnonzero((before.reshape(-1, 4) != field.reshape(-1, 4)).any(axis=1))
    assert all(int(i) in taken for i in changed)
    assert np.array_equal(tx, field.reshape(-1, 4)[idx])
    opaque = cubes_set_opaque(longer, cubes, ids)
    assert opaque and opaque <= taken
    fresh.close()
    rt.close()


@pytest.mark.parametrize("devices", DEVICES, ids=[str(d) for d in DEVICES])
def test_group_append_equals_the_single_context(spaces, devices):
    mixed, ui_space = spaces
    new = new_blocks()
    n0 = len(mixed.blocks)
    wopts, uopts = OPTIONS[0], GraphicsOptions(fog=FOG_NONE, lighting_display=LIGHT_FLAT)
    wcam = scenes.standard_camera(mixed, wopts, W, H)
    ucam = scenes.standard_camera(ui_space, uopts, W, H, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    cubes, ids = placements(mixed, range(n0, n0 + len(new)), 60, seed=4)
    rt = SpaceRaytracer(mixed, wopts)
    urt = SpaceRaytracer(ui_space, uopts, rt.ctx)
    rt.append_blocks(new)
    rt.update_cubes(cubes, ids)
    g = aicb200.DeviceGroup(devices)
    gw, gu = g.add_scene(mixed), g.add_scene(ui_space)
    gw.append_blocks(new)
    gw.update_cubes(cubes, ids)
    bd = (0.1, 0.3, 0.6, 0.5)
    want = aicb200.render_layers((rt, wcam, wopts), (urt, ucam, uopts), bd, NO_WORLD)
    got = g.render_layers((gw, wcam, wopts), (gu, ucam, uopts), bd, NO_WORLD)
    assert np.array_equal(got.data, want.data)
    want_t = aicb200.render_layers_terminal((rt, wcam, wopts), None, None, NO_WORLD)
    got_t = g.render_layers_terminal((gw, wcam, wopts), None, None, NO_WORLD)
    assert np.array_equal(got_t["text"], want_t["text"]) and np.array_equal(got_t["rgba"], want_t["rgba"])
    g.close()
    urt.close()
    rt.close()
    # past 16384 blocks: every replica widens its own cells
    space = narrow_space()
    new = wide_blocks()
    opts = GraphicsOptions(view_distance=80.0)
    cam = scenes.standard_camera(space, opts, W, H)
    cubes, ids = placements(space, [16383, 16384, 16400, 16419], 60, seed=9)
    rt = SpaceRaytracer(space, opts)
    rt.append_blocks(new[:2])
    rt.append_blocks(new[2:])
    rt.update_cubes(cubes, ids)
    g = aicb200.DeviceGroup(devices)
    gw = g.add_scene(space)
    gw.append_blocks(new[:2])
    gw.append_blocks(new[2:])
    gw.update_cubes(cubes, ids)
    assert np.array_equal(g.render_layers((gw, cam, opts)).data, aicb200.render_layers((rt, cam, opts)).data)
    g.close()
    rt.close()
    # light: a propagating edit with a new id leaves every replica identical
    space = light_scene(seed=9)
    n0 = len(space.blocks)
    g = aicb200.DeviceGroup(devices)
    gs = g.add_scene(space)
    gs.light_fast_evaluate()
    gs.light_evaluate(0)
    gs.append_blocks([Block(color=(0.1, 0.1, 0.1, 1.0), emission=(3.0, 1.5, 0.5)), Block(color=(0.7, 0.6, 0.9, 1.0))])
    cubes, ids = placements(space, [n0, n0 + 1], 20, seed=12)
    assert gs.light_edit_and_propagate(cubes, ids, 0)[0] > 0
    first = gs.light_download(0)
    for i in range(1, len(devices)):
        assert np.array_equal(gs.light_download(i), first), f"replica {i} differs from replica 0"
    ol = orc.OracleLight(Space(space.lower, space.block_ids, space.blocks + [Block(color=(0.1, 0.1, 0.1, 1.0),
                                                                                    emission=(3.0, 1.5, 0.5)),
                                                                              Block(color=(0.7, 0.6, 0.9, 1.0))],
                               light=space.light, sky_colors=space.sky_colors,
                               light_max_distance=space.light_max_distance))
    ol.fast_evaluate()
    ol.evaluate(0)
    ol.set_cubes(cubes, ids)
    ol.evaluate(0)
    compare_fields(first, ol.field())
    g.close()


def test_rejected_appends_change_nothing(spaces):
    mixed, _ = spaces
    n0 = len(mixed.blocks)
    opts = OPTIONS[0]
    cam = scenes.standard_camera(mixed, opts, W, H)
    bad = Block(resolution=3, indices=np.zeros((1, 1, 1), np.uint16), palette=np.zeros((1, 8), np.float32))
    good = Block(color=(0.9, 0.35, 0.1, 1.0))
    too_many = [good] * (65536 - n0 + 1)
    lib = aicb200.load_library()

    def rejected(call):
        with pytest.raises(AicbError) as e:
            call()
        assert e.value.status == abi.ERR_INVALID

    rt = SpaceRaytracer(mixed, opts)
    r = RtRenderer(cam, rt.ctx)
    r.rt = rt
    before = r.draw().data
    rejected(lambda: rt.append_blocks([good, good, bad]))
    rejected(lambda: rt.append_blocks(too_many))
    assert lib.aicb_scene_append_blocks(rt.handle, None, 3) == abi.ERR_INVALID
    rejected(lambda: rt.update_cubes([mixed.lower], [n0]))
    assert np.array_equal(r.draw().data, before)
    assert lib.aicb_scene_append_blocks(rt.handle, None, 0) == abi.OK   # n == 0 does nothing
    rt.append_blocks([good])   # and the table still takes the next index
    rt.update_cubes([mixed.lower], [n0])
    rt.close()
    g = aicb200.DeviceGroup([0, 0])
    gw = g.add_scene(mixed)
    frame = g.render_layers((gw, cam, opts)).data
    rejected(lambda: gw.append_blocks([good, good, bad]))
    rejected(lambda: gw.append_blocks(too_many))
    assert lib.aicb_group_scene_append_blocks(gw.handle, None, 3) == abi.ERR_INVALID
    rejected(lambda: gw.update_cubes([mixed.lower], [n0]))
    assert np.array_equal(g.render_layers((gw, cam, opts)).data, frame)
    g.close()
