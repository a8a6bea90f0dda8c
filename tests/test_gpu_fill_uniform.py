"""SpaceChange::EveryBlock on a live scene (aicb_scene_fill_uniform / aicb_group_scene_fill_uniform): Mutation::fill_uniform
over the whole bounds (space.rs:1461-1474).  The table becomes [block] and every cube holds id 0, and every output, and
device_bytes, equals a scene created from the filled Space; light is not touched, and the host's
light_queue_region(bounds, 210) then queues every cube as the reference does."""
import ctypes as C

import numpy as np
import pytest
import torch

import aicb200
from aicb200 import AicbError, Block, GraphicsOptions, RtRenderer, Space, SpaceRaytracer, abi, scenes
from resumeorc import LightOracle
from test_gpu_append_blocks import (DEVICES, OPTIONS, W, H, assert_same, every_output, narrow_space, new_blocks, placed,
                                    placements, wide_blocks)
from test_gpu_light import compare_fields
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit
from test_oracle_light_resume import fill_uniform_space

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def spaces():
    return scenes.small_mixed_scene(n=12, seed=7), scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))


def fill_blocks():
    """An opaque block, a translucent single voxel, a resolution-8 partial brick and AIR."""
    opaque, translucent, brick, air = new_blocks()[:4]
    return {"opaque": opaque, "translucent": translucent, "brick": brick, "air": air}


def filled(space, block):
    """The Space after fill_uniform(bounds, block), with the light the scene still holds."""
    return Space(space.lower, np.zeros_like(space.block_ids), [block], light=space.light, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


@pytest.mark.parametrize("kind", list(fill_blocks()))
def test_fill_equals_fresh_scene(spaces, kind):
    mixed, _ = spaces
    block = fill_blocks()[kind]
    rt = SpaceRaytracer(mixed, OPTIONS[0])
    rt.fill_uniform(block)
    fresh = SpaceRaytracer(filled(mixed, block), OPTIONS[0], rt.ctx)
    assert rt.device_bytes == fresh.device_bytes
    for opts in OPTIONS:
        cam = scenes.standard_camera(mixed, opts, W, H)
        assert_same(every_output(rt, opts, cam), every_output(fresh, opts, cam), f"{kind}, transparency {opts.transparency}")
    fresh.close()
    rt.close()


@pytest.mark.parametrize("devices", DEVICES, ids=[str(d) for d in DEVICES])
def test_group_fill_equals_fresh_scene(spaces, devices):
    mixed, _ = spaces
    opts = OPTIONS[0]
    cam = scenes.standard_camera(mixed, opts, W, H)
    g = aicb200.DeviceGroup(devices)
    gw = g.add_scene(mixed)
    for kind, block in fill_blocks().items():
        gw.fill_uniform(block)
        fresh = SpaceRaytracer(filled(mixed, block), opts)
        assert np.array_equal(g.render_layers((gw, cam, opts)).data, aicb200.render_layers((fresh, cam, opts)).data), kind
        got_t, want_t = g.render_layers_terminal((gw, cam, opts)), aicb200.render_layers_terminal((fresh, cam, opts))
        assert np.array_equal(got_t["text"], want_t["text"]) and np.array_equal(got_t["rgba"], want_t["rgba"]), kind
        fresh.close()
    g.close()


@pytest.mark.parametrize("devices", [None] + list(DEVICES), ids=["ctx"] + [str(d) for d in DEVICES])
def test_fill_narrows_wide_cells(devices):
    """A table grown past 16384 blocks has u32 cells; the fill leaves a one-block table with u16 cells."""
    space = narrow_space()
    opts = GraphicsOptions(view_distance=80.0)
    cam = scenes.standard_camera(space, opts, W, H)
    block = fill_blocks()["brick"]
    if devices is None:
        rt = SpaceRaytracer(space, opts)
        rt.append_blocks(wide_blocks())
        rt.fill_uniform(block)
        fresh = SpaceRaytracer(filled(space, block), opts, rt.ctx)
        assert rt.device_bytes == fresh.device_bytes
        assert_same(every_output(rt, opts, cam), every_output(fresh, opts, cam), "narrowed")
        fresh.close()
        rt.close()
        return
    g = aicb200.DeviceGroup(devices)
    gw = g.add_scene(space)
    gw.append_blocks(wide_blocks())
    gw.fill_uniform(block)
    fresh = SpaceRaytracer(filled(space, block), opts)
    assert np.array_equal(g.render_layers((gw, cam, opts)).data, aicb200.render_layers((fresh, cam, opts)).data)
    fresh.close()
    g.close()


def after_fill(target, space, seed):
    """fill -> append -> cube updates -> update of the filled and an appended id, on `target`; the Space it holds."""
    target.fill_uniform(Block.air())
    new = new_blocks()
    target.append_blocks(new)
    cubes, ids = placements(filled(space, Block.air()), range(0, 1 + len(new)), 80, seed)
    target.update_cubes(cubes, ids)
    changed = {0: Block(color=(0.2, 0.6, 0.3, 0.5)), 3: scenes.make_voxel_block(41, resolution=4)}
    target.update_blocks(list(changed), list(changed.values()))
    blocks = [Block.air()] + new
    for i, b in changed.items():
        blocks[i] = b
    return placed(filled(space, Block.air()), blocks, cubes, ids)


def test_updates_after_a_fill_equal_fresh_scene(spaces):
    mixed, _ = spaces
    rt = SpaceRaytracer(mixed, OPTIONS[0])
    fresh = SpaceRaytracer(after_fill(rt, mixed, seed=21), OPTIONS[0], rt.ctx)
    for opts in OPTIONS:
        cam = scenes.standard_camera(mixed, opts, W, H)
        assert_same(every_output(rt, opts, cam), every_output(fresh, opts, cam), f"transparency {opts.transparency}")
    fresh.close()
    rt.close()


@pytest.mark.parametrize("devices", DEVICES, ids=[str(d) for d in DEVICES])
def test_group_updates_after_a_fill_equal_fresh_scene(spaces, devices):
    mixed, _ = spaces
    opts = OPTIONS[0]
    cam = scenes.standard_camera(mixed, opts, W, H)
    g = aicb200.DeviceGroup(devices)
    gw = g.add_scene(mixed)
    fresh = SpaceRaytracer(after_fill(gw, mixed, seed=22), opts)
    assert np.array_equal(g.render_layers((gw, cam, opts)).data, aicb200.render_layers((fresh, cam, opts)).data)
    fresh.close()
    g.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_lit_fill_keeps_the_light_and_queues_the_bounds(devices):
    """fill_uniform_entire_space (space/tests.rs:411-434) on a lit scene: the fill writes no texel and adds no changed
    cube; light_queue_region(bounds, 210) raises every cube to at least 210; light_evaluate then meets the light
    contract against the oracle started from the same field and queue."""
    space = fill_uniform_space()
    lit = Lit(devices, space)
    lit.light_fast_evaluate()
    lit.light_evaluate(0)
    high = ((5, 3, 0), (10, 4, 2), 230)
    lit.light_queue_region(*high)
    field, queue, changed = lit.field(), lit.light_download_queue(), lit.light_changes_count()
    assert (queue == 230).sum() == 10 * 4 * 2 and (queue != 230).sum() == (queue == 0).sum()
    lit.fill_uniform(Block.air())
    assert np.array_equal(lit.field(), field)
    assert np.array_equal(lit.light_download_queue(), queue)
    assert lit.light_changes_count() == changed
    lit.light_queue_region(space.lower, space.size, 210)
    assert np.array_equal(lit.field(), field)
    assert lit.light_changes_count() == changed
    after = lit.light_download_queue()
    assert np.array_equal(after, np.maximum(queue, 210))
    ol = LightOracle(Space(space.lower, np.zeros_like(space.block_ids), [Block.air()], light=field,
                           light_max_distance=space.light_max_distance))
    ol.queue_region(*high)
    ol.queue_region(space.lower, space.size, 210)
    assert np.array_equal(ol.queue(), after)
    assert lit.light_evaluate(0)[0] > 0
    ol.evaluate(0)
    compare_fields(lit.field(), ol.field())
    assert not lit.light_download_queue().any()
    lit.close()


def test_fill_while_a_frame_is_in_flight(spaces):
    """A frame issued on a caller's stream before the fill is the old scene's frame; the next one is the filled
    scene's."""
    mixed, _ = spaces
    opts = GraphicsOptions(view_distance=80.0)
    cam = scenes.standard_camera(mixed, opts, 320, 240)
    rt = SpaceRaytracer(mixed, opts)
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
    block = fill_blocks()["translucent"]
    rt.fill_uniform(block)
    info = abi.RenderInfo()
    assert lib.aicb_render_finish(rt.handle, C.byref(info)) == abi.OK
    torch.cuda.synchronize()
    assert np.array_equal(d_out.cpu().numpy(), before)
    fresh = SpaceRaytracer(filled(mixed, block), opts, rt.ctx)
    rf = RtRenderer(cam, rt.ctx)
    rf.rt = fresh
    after = r.draw().data
    assert np.array_equal(after, rf.draw().data)
    assert not np.array_equal(after.reshape(-1, 4), before)
    fresh.close()
    rt.close()


def test_rejected_fills_change_nothing(spaces):
    mixed, _ = spaces
    opts = OPTIONS[0]
    cam = scenes.standard_camera(mixed, opts, W, H)
    bad = Block(resolution=3, indices=np.zeros((1, 1, 1), np.uint16), palette=np.zeros((1, 8), np.float32))
    lib = aicb200.load_library()
    rt = SpaceRaytracer(mixed, opts)
    r = RtRenderer(cam, rt.ctx)
    r.rt = rt
    before, nbytes = r.draw().data, rt.device_bytes
    with pytest.raises(AicbError) as e:
        rt.fill_uniform(bad)
    assert e.value.status == abi.ERR_INVALID
    assert lib.aicb_scene_fill_uniform(rt.handle, None) == abi.ERR_INVALID
    assert lib.aicb_scene_fill_uniform(None, aicb200._block_descs([Block.air()])) == abi.ERR_INVALID
    assert np.array_equal(r.draw().data, before)
    assert rt.device_bytes == nbytes
    rt.close()
    g = aicb200.DeviceGroup([0, 0])
    gw = g.add_scene(mixed)
    frame = g.render_layers((gw, cam, opts)).data
    with pytest.raises(AicbError) as e:
        gw.fill_uniform(bad)
    assert e.value.status == abi.ERR_INVALID
    assert lib.aicb_group_scene_fill_uniform(gw.handle, None) == abi.ERR_INVALID
    assert np.array_equal(g.render_layers((gw, cam, opts)).data, frame)
    g.close()
