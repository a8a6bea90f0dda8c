"""Replaced block definitions give their device memory back: aicb_scene_update_blocks marks a redefined id's voxel data
dead and compacts a pool on the device once its dead part exceeds its live part.  Every output stays byte for byte a
fresh scene's; a pool never holds more than twice its live data; the 2^32-voxel limit counts live data only; and a frame
in flight across a compacting update is the old table's frame."""
import ctypes as C

import numpy as np
import pytest
import torch

import aicb200
from aicb200 import Block, GraphicsOptions, RtRenderer, Space, SpaceRaytracer, abi, scenes
from test_gpu_append_blocks import DEVICES, OPTIONS, W, H, assert_same, every_output

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mixed():
    return scenes.small_mixed_scene(n=12, seed=7)


def with_blocks(space, blocks):
    return Space(space.lower, space.block_ids, list(blocks), light=space.light, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


def redefinitions(n_blocks, n, seed):
    """n (index, definition) pairs at random indices, mixing AIR, invisible, opaque and translucent single voxels, and
    bricks of resolution 2 to 16 (some partial)."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        r = int(rng.integers(0, 7))
        if r == 0:
            b = Block.air()
        elif r == 1:
            b = Block(color=(0.0, 0.0, 0.0, 0.0))
        elif r in (2, 3):
            b = Block(color=tuple(rng.uniform(0.05, 1.0, 3)) + ((1.0, 0.5)[r - 2],))
        else:
            b = scenes.make_voxel_block(100 + k, resolution=int(rng.choice([2, 4, 8, 16])), alpha=(1.0, 0.5)[k % 2],
                                        partial_bounds=bool(k % 3))
        out.append((int(rng.integers(0, n_blocks)), b))
    return out


@pytest.mark.parametrize("devices", [None] + list(DEVICES), ids=["ctx"] + [str(d) for d in DEVICES])
def test_many_redefinitions_equal_fresh_scene(mixed, devices):
    """300 redefinitions, one call each: the pools compact several times on the way, and device_bytes never exceeds a
    fresh scene's plus its voxel data once more."""
    opts = OPTIONS[0]
    cam = scenes.standard_camera(mixed, opts, W, H)
    blocks = list(mixed.blocks)
    if devices is None:
        rt = SpaceRaytracer(mixed, opts)
        target = rt
    else:
        g = aicb200.DeviceGroup(devices)
        target = g.add_scene(mixed)
    # a scene with the same table size and no voxel data: what device_bytes counts besides the pools
    bare = SpaceRaytracer(with_blocks(mixed, [Block.air()] * len(blocks)), opts)
    bare_bytes = bare.device_bytes
    bare.close()
    drops, last = 0, None
    for k, (i, b) in enumerate(redefinitions(len(blocks), 300, seed=5)):
        target.update_blocks([i], [b])
        blocks[i] = b
        if devices is None:
            fresh = SpaceRaytracer(with_blocks(mixed, blocks), opts, rt.ctx)
            fresh_bytes = fresh.device_bytes
            fresh.close()
            assert rt.device_bytes <= fresh_bytes + (fresh_bytes - bare_bytes), f"redefinition {k}"
            drops += last is not None and rt.device_bytes < last
            last = rt.device_bytes
    fresh = SpaceRaytracer(with_blocks(mixed, blocks), opts)
    if devices is None:
        assert drops >= 3, "fewer compactions than expected"
        for o in OPTIONS:
            c = scenes.standard_camera(mixed, o, W, H)
            assert_same(every_output(rt, o, c), every_output(fresh, o, c), f"transparency {o.transparency}")
        rt.close()
    else:
        assert np.array_equal(g.render_layers((target, cam, opts)).data, aicb200.render_layers((fresh, cam, opts)).data)
        got_t = g.render_layers_terminal((target, cam, opts))
        want_t = aicb200.render_layers_terminal((fresh, cam, opts))
        assert np.array_equal(got_t["text"], want_t["text"]) and np.array_equal(got_t["rgba"], want_t["rgba"])
        g.close()
    fresh.close()


def big_block_space(block):
    """A 6^3 Space of AIR with one full resolution-128 block at a few cubes."""
    ids = np.zeros((6, 6, 6), np.uint16)
    ids[1, 1, 1] = ids[3, 2, 4] = ids[4, 4, 1] = 1
    return Space((0, 0, 0), ids, [Block.air(), block], sky_colors=scenes.OCTANT_SKY)


def test_repeated_redefinitions_of_a_resolution_128_block():
    """2100 redefinitions of a full resolution-128 block (2^21 voxels each) pass 2^32 voxels written in all; only
    the live data counts against the brick pool's limit."""
    defs = [scenes.make_voxel_block(s, resolution=128, alpha=1.0, partial_bounds=False) for s in (3, 4)]
    assert defs[0].indices.size == 128 ** 3
    opts = GraphicsOptions(view_distance=40.0)
    rt = SpaceRaytracer(big_block_space(defs[0]), opts)
    for k in range(2100):
        rt.update_blocks([1], [defs[(k + 1) % 2]])
    fresh = SpaceRaytracer(big_block_space(defs[2100 % 2]), opts, rt.ctx)
    assert rt.device_bytes <= 2 * fresh.device_bytes
    cam = scenes.standard_camera(fresh.space, opts, W, H)
    assert_same(every_output(rt, opts, cam), every_output(fresh, opts, cam))
    fresh.close()
    rt.close()


def test_compacting_update_while_a_frame_is_in_flight(mixed):
    """An update that compacts both pools (an index redefined 16 times in one call: its dead data exceeds the live data)
    while a frame issued on a caller's stream still runs: that frame is the old table's."""
    opts = GraphicsOptions(view_distance=80.0)
    old = scenes.make_voxel_block(7, resolution=16, alpha=0.5, partial_bounds=False)
    space = with_blocks(mixed, list(mixed.blocks))
    blocks = list(space.blocks)
    bricks = [i for i, b in enumerate(blocks) if b.resolution > 1]
    big = bricks[0]
    blocks[big] = old
    space = with_blocks(mixed, blocks)
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
    new = [scenes.make_voxel_block(s, resolution=16, alpha=1.0, partial_bounds=False) for s in range(8, 24)]
    rt.update_blocks([big] * len(new), new)
    info = abi.RenderInfo()
    assert lib.aicb_render_finish(rt.handle, C.byref(info)) == abi.OK
    torch.cuda.synchronize()
    assert np.array_equal(d_out.cpu().numpy(), before)
    blocks[big] = new[-1]
    fresh = SpaceRaytracer(with_blocks(mixed, blocks), opts, rt.ctx)
    assert rt.device_bytes == fresh.device_bytes   # compacted: the pools hold exactly the live data
    rf = RtRenderer(cam, rt.ctx)
    rf.rt = fresh
    after = r.draw().data
    assert np.array_equal(after, rf.draw().data)
    assert not np.array_equal(after.reshape(-1, 4), before)
    fresh.close()
    rt.close()
