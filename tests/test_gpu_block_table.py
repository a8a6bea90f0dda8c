"""A scene's block table written through its three entry points (aicb_scene_create, aicb_scene_update_blocks,
aicb_scene_append_blocks, and their group forms), in any order: every frame equals, byte for byte, the frame of a scene
created from the final Space.  Also an update while frames that read the old table are in flight, rejected updates,
and a table that starts empty."""
import ctypes as C

import numpy as np
import pytest
import torch

import aicb200
from aicb200 import AicbError, Block, GraphicsOptions, RtRenderer, Space, SpaceRaytracer, abi, scenes
from test_gpu_light import light_scene
from test_gpu_append_blocks import DEVICES, OPTIONS, W, H, assert_same, every_output, new_blocks, placed, placements

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def spaces():
    return scenes.small_mixed_scene(n=12, seed=7), scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))


def with_blocks(space, changed):
    blocks = list(space.blocks)
    for i, b in changed.items():
        blocks[i] = b
    return Space(space.lower, space.block_ids, blocks, light=space.light, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


def kind_changes():
    """small_mixed_scene's 1-7 are single voxels, 9 invisible, 10-14 bricks.  Index 1 is named twice: the second
    definition is the one that stays."""
    return ([1, 3, 9, 10, 1, 5],
            [scenes.make_voxel_block(31, resolution=8, alpha=0.5),   # (replaced below)
             scenes.make_voxel_block(32, resolution=4),               # single voxel -> brick
             Block(color=(0.3, 0.8, 0.2, 1.0)),                       # invisible -> single voxel
             Block(color=(0.0, 0.0, 0.0, 0.0)),                       # brick -> invisible
             Block(color=(0.0, 0.0, 0.0, 0.0)),                       # single voxel -> invisible, last wins
             Block(color=(0.9, 0.6, 0.1, 0.25))])                     # single voxel, recoloured


def final_definitions(indices, blocks):
    return {i: b for i, b in zip(indices, blocks)}   # a later entry replaces an earlier one


def test_one_update_names_an_index_twice_and_changes_every_kind(spaces):
    mixed, _ = spaces
    indices, blocks = kind_changes()
    rt = SpaceRaytracer(mixed, OPTIONS[0])
    rt.update_blocks(indices, blocks)
    fresh = SpaceRaytracer(with_blocks(mixed, final_definitions(indices, blocks)), OPTIONS[0], rt.ctx)
    for opts in OPTIONS:
        cam = scenes.standard_camera(mixed, opts, W, H)
        assert_same(every_output(rt, opts, cam), every_output(fresh, opts, cam), f"transparency {opts.transparency}")
    fresh.close()
    rt.close()


def interleaved(target, space, seed):
    """update -> append -> update of appended ids -> cube updates on `target` (a SpaceRaytracer or a GroupScene).
    Returns the Space it then holds."""
    n0 = len(space.blocks)
    first = {2: scenes.make_voxel_block(21, resolution=8, alpha=0.5), 9: Block(color=(0.6, 0.2, 0.7, 1.0))}
    target.update_blocks(list(first), list(first.values()))
    new = new_blocks()
    target.append_blocks(new)
    second = {n0: scenes.make_voxel_block(22, resolution=4), n0 + 2: Block(color=(0.1, 0.9, 0.9, 0.5)),
              n0 + 3: Block(color=(0.8, 0.8, 0.1, 1.0))}   # brick -> single voxel, brick recoloured, AIR -> single
    target.update_blocks(list(second), list(second.values()))
    cubes, ids = placements(space, list(range(n0, n0 + len(new))) + [2, 9], 60, seed)
    target.update_cubes(cubes, ids)
    blocks = list(space.blocks) + new
    for i, b in {**first, **second}.items():
        blocks[i] = b
    return placed(space, blocks, cubes, ids)


def test_interleaved_updates_and_appends_equal_fresh_snapshot(spaces):
    mixed, _ = spaces
    rt = SpaceRaytracer(mixed, OPTIONS[0])
    fresh = SpaceRaytracer(interleaved(rt, mixed, seed=13), OPTIONS[0], rt.ctx)
    for opts in OPTIONS:
        cam = scenes.standard_camera(mixed, opts, W, H)
        assert_same(every_output(rt, opts, cam), every_output(fresh, opts, cam), f"transparency {opts.transparency}")
    fresh.close()
    rt.close()


@pytest.mark.parametrize("devices", DEVICES, ids=[str(d) for d in DEVICES])
def test_group_interleaved_updates_and_appends_equal_fresh_snapshot(spaces, devices):
    mixed, _ = spaces
    opts = OPTIONS[0]
    cam = scenes.standard_camera(mixed, opts, W, H)
    g = aicb200.DeviceGroup(devices)
    gw = g.add_scene(mixed)
    fresh = SpaceRaytracer(interleaved(gw, mixed, seed=14), opts)
    assert np.array_equal(g.render_layers((gw, cam, opts)).data, aicb200.render_layers((fresh, cam, opts)).data)
    got_t = g.render_layers_terminal((gw, cam, opts))
    want_t = aicb200.render_layers_terminal((fresh, cam, opts))
    assert np.array_equal(got_t["text"], want_t["text"]) and np.array_equal(got_t["rgba"], want_t["rgba"])
    fresh.close()
    g.close()


@pytest.mark.parametrize("between", ["nothing", "other-scene-frame", "light-propagation"])
def test_update_while_a_frame_is_in_flight(spaces, between):
    """Frames issued on a caller's stream before an update that writes the block records over in place (and re-encodes
    cells) are the frames of the table they were issued on; the next frame is the new table's.  Between the frame and
    the update, another scene of the context may issue a frame on that stream (the context's last frame is then not
    this scene's), or propagate light on the context's stream (which times itself with events of its own)."""
    mixed, ui_space = spaces
    opts = GraphicsOptions(view_distance=80.0)
    cam = scenes.standard_camera(mixed, opts, 320, 240)
    ocam = scenes.standard_camera(ui_space, opts, 320, 240)
    rt = SpaceRaytracer(mixed, opts)
    other = SpaceRaytracer(ui_space, opts, rt.ctx)
    lit = SpaceRaytracer(light_scene(seed=9), GraphicsOptions(), rt.ctx)
    r = RtRenderer(cam, rt.ctx)
    r.rt = rt
    before = r.draw().data.reshape(-1, 4)
    ro = RtRenderer(ocam, rt.ctx)
    ro.rt = other
    other_frame_data = ro.draw().data.reshape(-1, 4)
    lib = aicb200.load_library()
    n = cam.data.fb_width * cam.data.fb_height
    d_out = torch.zeros((n, 4), dtype=torch.uint8, device="cuda")
    o_out = torch.zeros((n, 4), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    o = opts.to_abi(True)
    assert lib.aicb_render_srgb8_device(rt.handle, C.byref(cam.data), C.byref(o), None, d_out.data_ptr(), n,
                                        C.c_void_p(stream.cuda_stream)) == abi.OK
    if between == "other-scene-frame":
        assert lib.aicb_render_srgb8_device(other.handle, C.byref(ocam.data), C.byref(o), None, o_out.data_ptr(), n,
                                            C.c_void_p(stream.cuda_stream)) == abi.OK
    elif between == "light-propagation":
        lit.light_fast_evaluate()
        lit.light_evaluate(0)
    indices, blocks = kind_changes()
    rt.update_blocks(indices, blocks)
    info = abi.RenderInfo()
    last = other if between == "other-scene-frame" else rt
    assert lib.aicb_render_finish(last.handle, C.byref(info)) == abi.OK
    torch.cuda.synchronize()
    assert np.array_equal(d_out.cpu().numpy(), before)
    if between == "other-scene-frame":
        assert np.array_equal(o_out.cpu().numpy(), other_frame_data)
    fresh = SpaceRaytracer(with_blocks(mixed, final_definitions(indices, blocks)), opts, rt.ctx)
    rf = RtRenderer(cam, rt.ctx)
    rf.rt = fresh
    after = r.draw().data
    assert np.array_equal(after, rf.draw().data)
    assert not np.array_equal(after.reshape(-1, 4), before)
    for s in (fresh, lit, other, rt):
        s.close()


def test_rejected_updates_change_nothing(spaces):
    mixed, _ = spaces
    n0 = len(mixed.blocks)
    opts = OPTIONS[0]
    cam = scenes.standard_camera(mixed, opts, W, H)
    good = Block(color=(0.9, 0.35, 0.1, 1.0))
    bad = Block(resolution=3, indices=np.zeros((1, 1, 1), np.uint16), palette=np.zeros((1, 8), np.float32))
    rt = SpaceRaytracer(mixed, opts)
    r = RtRenderer(cam, rt.ctx)
    r.rt = rt
    before, nbytes = r.draw().data, rt.device_bytes
    for indices, blocks in (([1, n0], [good, good]),     # an index past the table after a valid entry
                            ([1, 10], [good, bad])):     # a bad descriptor after a valid entry
        with pytest.raises(AicbError) as e:
            rt.update_blocks(indices, blocks)
        assert e.value.status == abi.ERR_INVALID
        assert np.array_equal(r.draw().data, before)
        assert rt.device_bytes == nbytes
    rt.close()


def test_empty_scene_grows_to_a_fresh_scene(spaces):
    """A scene created with no blocks and an empty volume takes its whole table from appends.  With no cube to hold a
    block, the frames are sky alone: the table itself is compared through device_bytes."""
    mixed, _ = spaces
    opts = OPTIONS[0]
    empty_ids = np.zeros((0, 0, 0), np.uint16)
    new = new_blocks()
    rt = SpaceRaytracer(Space((0, 0, 0), empty_ids, []), opts)
    assert rt.device_bytes == 0
    rt.append_blocks(new[:2])
    rt.append_blocks(new[2:])
    fresh = SpaceRaytracer(Space((0, 0, 0), empty_ids, new), opts, rt.ctx)
    assert rt.device_bytes == fresh.device_bytes
    cam = scenes.standard_camera(mixed, opts, W, H)
    r, rf = RtRenderer(cam, rt.ctx), RtRenderer(cam, rt.ctx)
    r.rt, rf.rt = rt, fresh
    assert np.array_equal(r.draw().data, rf.draw().data)
    fresh.close()
    rt.close()
