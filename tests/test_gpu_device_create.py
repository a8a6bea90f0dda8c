"""Scenes created and refilled from device memory (aicb_scene_create_device, aicb_scene_fill_uniform_device and their
group forms): with the Space's block ids, light and voxels as CUDA tensors, the new scene must be byte for byte the one
its host twin (aicb_scene_create / aicb_scene_fill_uniform with the same data) builds, with the same errors.  Every
check builds two scenes from one Space on the same target (one context, groups of 1, 2 and 3 contexts of one device),
one through the host call and one through the device call, and compares them after every step: block ids, every frame
output (the group frame on groups), device_bytes (on one context) and the light volume."""
import ctypes as C

import numpy as np
import pytest
import torch

import aicb200
from aicb200 import AicbError, Block, DeviceSpace, GraphicsOptions, Space, abi, scenes
from test_gpu_append_blocks import assert_same, every_output, narrow_space, wide_blocks
from test_gpu_device_blocks import on_device
from test_gpu_device_inputs import T, unlit
from test_gpu_light import light_scene
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
OPTS = GraphicsOptions(view_distance=60.0, lighting_display=aicb200.LIGHT_LINEAR)
W, H = 48, 40


def device_space(space, derive=False):
    """The same Space with its ids, light and voxels as CUDA tensors on device 0."""
    blocks, keep = [], {}
    for b in space.blocks:   # (a block listed many times goes to the device once)
        if id(b) not in keep:
            keep[id(b)] = on_device(b, derive)
        blocks.append(keep[id(b)])
    return DeviceSpace(space.lower, T(space.block_ids), blocks, light=None if space.light is None else T(space.light),
                       sky_colors=space.sky_colors, light_max_distance=space.light_max_distance)


class Twin:
    """Two scenes of one Space on one target: `host` created by the host call, `dev` by the device call (or, with
    dev_space=False, by the host call too, for the fill tests)."""

    def __init__(self, target, space, dev_space=None, cam_space=None):
        self.target, self.space = target, space
        self.host = Lit(target, space)
        self.dev = Lit(target, device_space(space) if dev_space is None else (dev_space or space))
        self.cam = scenes.standard_camera(cam_space or space, OPTS, W, H)

    def state(self, lit):
        s = lit.scene
        out = {"frame": lit.frame(self.cam, OPTS)}
        if np.prod(s.space.size):
            out["ids"] = s.block_ids()
        if lit.group is None:
            out.update(every_output(s, OPTS, self.cam))
            out["device_bytes"] = np.array([s.device_bytes])
        if s.space.light is not None or s.space.light_max_distance:
            out["light"] = lit.field()
        return out

    def check(self, label):
        a, b = self.state(self.host), self.state(self.dev)
        assert a.keys() == b.keys(), label
        assert_same(a, b, label)
        return a

    def close(self):
        self.host.close()
        self.dev.close()


@pytest.fixture(params=TARGETS, ids=TARGET_IDS)
def target(request):
    return request.param


def big_palette_block(seed=11):
    rng = np.random.default_rng(seed)
    pal = np.zeros((40000, 8), np.float32)
    pal[:, :3] = rng.uniform(0, 1, (40000, 3))
    pal[:, 3] = rng.choice(np.array([0.0, 0.5, 1.0], np.float32), 40000)
    return Block(resolution=16, indices=rng.integers(0, 40000, (16, 16, 16)).astype(np.uint16), palette=pal)


def spaces(kind):
    if kind == "mixed":   # lit, octant sky, negative lower corner
        return scenes.small_mixed_scene(n=12, seed=7)
    if kind == "c1":      # partial-bounds resolution-16 blocks over a ground slab
        return scenes.config_c1(n=20, seed=2, n_voxel_blocks=6, with_light=True)
    if kind == "unlit":
        return unlit(scenes.small_mixed_scene(n=12, seed=7))
    if kind == "u32":     # more than 16384 blocks: 32-bit cells
        s = narrow_space()
        ids = s.block_ids.copy()
        ids[1, 2, :5] = [16383, 16384, 16390, 16400, 16419]
        return Space(s.lower, ids, s.blocks + wide_blocks(), light=s.light, sky_colors=s.sky_colors)
    if kind == "wide":    # a block of more than 32768 palette entries: wide brick words
        s = scenes.small_mixed_scene(n=12, seed=7)
        s.blocks[11] = big_palette_block()
        return s
    assert kind == "empty"
    return Space((4, -2, 1), np.zeros((0, 3, 5), np.uint16), [Block.air(), Block(color=(0.3, 0.5, 0.7, 1.0))])


@pytest.mark.parametrize("kind", ["mixed", "c1", "unlit", "u32", "wide", "empty"])
def test_created_scene_equals_the_host_twin(target, kind):
    space = spaces(kind)
    t = Twin(target, space, cam_space=scenes.small_mixed_scene() if kind == "empty" else None)
    t.check(kind)
    t.close()


def test_light_after_creation(target):
    t = Twin(target, light_scene(seed=9))
    t.check("created")
    for lit in (t.host, t.dev):
        lit.light_fast_evaluate()
        lit.light_evaluate(0)
    t.check("fast_evaluate, evaluate(0)")
    t.close()


def test_derived_light_equals_derive_then_host_twin(target):
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    lit = Space(mixed.lower, mixed.block_ids, mixed.blocks, light=np.zeros(mixed.size + (4,), np.uint8),
                sky_colors=mixed.sky_colors, light_max_distance=12)
    dspace = device_space(lit, derive=True)
    for b, d in zip(lit.blocks, aicb200.Context.default().derive_block_light(lit.blocks)):
        b.set_light_data(d)   # (after the device twin took the voxels: its light is derived on the device)
    t = Twin(target, lit, dev_space=dspace)
    t.check("derived")
    for s in (t.host, t.dev):
        s.light_fast_evaluate()
        s.light_evaluate(0)
    t.check("propagated")
    t.close()


def test_stale_mirror_after_creation(target):
    space = light_scene(seed=9)
    t = Twin(target, space)
    rng = np.random.default_rng(3)
    lo, size = np.array(space.lower), np.array(space.size)
    cubes = (rng.integers(0, size, (300, 3)) + lo).astype(np.int32)
    ids = rng.integers(0, len(space.blocks), 300).astype(np.uint16)
    # host calls that read the mirror: the device twin's is rebuilt from its cells first
    assert t.host.light_edit_cubes(cubes[:100], ids[:100]) == t.dev.light_edit_cubes(cubes[:100], ids[:100])
    t.check("light_edit_cubes")
    for lit in (t.host, t.dev):
        lit.update_blocks([1], [Block(color=(0.0, 0.0, 0.0, 0.0))])   # opaque to invisible: a kind change
        lit.update_cubes(cubes[100:200], ids[100:200])
    t.check("update_blocks, update_cubes")
    # device updates on top, then a host call again
    for lit in (t.host, t.dev):
        lit.update_cubes(T(cubes[200:]), T(ids[200:]))
        lit.light_edit_cubes(cubes[:50], ids[50:100])
        lit.light_evaluate(0)
    t.check("device update, light edit")
    t.close()


def _create(lib, desc, device, group=None):
    """The raw creation call (host form if device is False) -> (status, message, out is NULL)."""
    out = C.c_void_p()
    if group is None:
        ctx = aicb200.Context.default().handle
        st = (lib.aicb_scene_create_device(ctx, C.byref(desc), 0, None, C.byref(out)) if device
              else lib.aicb_scene_create(ctx, C.byref(desc), C.byref(out)))
    else:
        st = (lib.aicb_group_scene_create_device(group.handle, C.byref(desc), 0, None, C.byref(out)) if device
              else lib.aicb_group_scene_create(group.handle, C.byref(desc), C.byref(out)))
    msg = lib.aicb_last_error().decode()
    if out.value:   # (a test failure, not a leak)
        (lib.aicb_scene_destroy if group is None else lib.aicb_group_scene_destroy)(out)
    return st, msg, out.value is None


def rejections(space):
    """(label, the Space spoiled, a change of the desc) of each host-twin failure."""
    n = len(space.blocks)

    def with_ids(edit):
        ids = space.block_ids.copy()
        edit(ids)
        return Space(space.lower, ids, space.blocks, light=space.light, sky_colors=space.sky_colors)

    def with_blocks(edit, ids=None):
        blocks = list(space.blocks)
        edit(blocks)
        return Space(space.lower, space.block_ids if ids is None else ids, blocks, light=space.light,
                     sky_colors=space.sky_colors)

    def first(ids):
        ids[0, 0, 0] = n

    def last(ids):
        ids[-1, -1, -1] = n + 7

    def bad_voxel(blocks):
        b = scenes.make_voxel_block(99, resolution=4)
        b.indices = b.indices.copy()
        b.indices.flat[5] = b.palette.shape[0]
        blocks[12] = b

    bad_ids = space.block_ids.copy()
    first(bad_ids)

    def oversized(blocks):
        blocks[11] = Block(resolution=4, indices=np.zeros((4, 4, 4), np.uint16), palette=np.zeros((65537, 8), np.float32))

    def no_blocks(d):
        d.n_blocks = 0

    def far(d):
        d.bounds.lower[0] = (1 << 30) - 5

    return [("id out of range at the first cube", with_ids(first), None),
            ("id out of range at the last cube", with_ids(last), None),
            ("a bad voxel index in a later block, and a bad id", with_blocks(bad_voxel, bad_ids), None),
            ("a palette over 65536 entries", with_blocks(oversized), None),
            ("an empty table for a non-empty volume", space, no_blocks),
            ("bounds beyond 2^30", space, far)]


@pytest.mark.parametrize("devices", [None, [0, 0]], ids=["ctx", "group2"])
def test_rejections_match_the_host_twin(devices):
    space = scenes.small_mixed_scene(n=12, seed=7)
    lib = aicb200.load_library()
    group = None if devices is None else aicb200.DeviceGroup(devices)
    for label, bad, spoil in rejections(space):
        hd, keep_h = bad.to_desc()
        dd, keep_d = device_space(bad).to_desc(DEV)
        if spoil:
            spoil(hd)
            spoil(dd)
        st_h, msg_h, null_h = _create(lib, hd, False, group)
        st_d, msg_d, null_d = _create(lib, dd, True, group)
        assert st_h != abi.OK, label
        assert (st_d, msg_d) == (st_h, msg_h), label
        assert null_h and null_d, label
    # device-only: host memory for the ids, misaligned pointers
    ds = device_space(space)
    for label, spoil, words in [("numpy ids", lambda d: setattr(d, "block_ids", space.block_ids.ctypes.data),
                                 "not device memory"),
                                ("misaligned ids", lambda d: setattr(d, "block_ids", ds.block_ids.data_ptr() + 1),
                                 "aligned"),
                                ("misaligned light", lambda d: setattr(d, "light", ds.light.data_ptr() + 2),
                                 "aligned")]:
        dd, keep = ds.to_desc(DEV)
        spoil(dd)
        st, msg, null = _create(lib, dd, True, group)
        assert st == abi.ERR_INVALID and words in msg and null, label
    with pytest.raises(ValueError):
        DeviceSpace(space.lower, T(space.block_ids).view(torch.int16), ds.blocks)
    with pytest.raises(ValueError):
        DeviceSpace(space.lower, T(space.block_ids), ds.blocks, light=T(space.light)[:, :, :4])
    with pytest.raises(ValueError):
        DeviceSpace(space.lower, T(space.block_ids), ds.blocks[:-1] + [on_device(space.blocks[-1], derive=True)])
    with pytest.raises(ValueError):
        DeviceSpace(space.lower, T(space.block_ids).transpose(0, 2), ds.blocks)
    if group is not None:
        group.close()


def test_inputs_written_on_a_side_stream_are_read_in_stream_order(target):
    """Torch kernels on a side stream write the ids and the light after a delay; the creation issued with that stream
    current reads them without a host synchronise in between."""
    space = scenes.small_mixed_scene(n=12, seed=7)
    ds = device_space(space)
    ids, light = T(space.block_ids), T(space.light)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        out_ids = torch.zeros(space.size, dtype=torch.int16, device=DEV)
        out_light = torch.zeros(space.size + (4,), dtype=torch.uint8, device=DEV)
        torch.cuda._sleep(50_000_000)   # tens of milliseconds of GPU time before the inputs exist
        out_ids.copy_(ids.view(torch.int16))
        out_light.copy_(light)
        late = DeviceSpace(space.lower, out_ids.view(torch.uint16), ds.blocks, light=out_light,
                           sky_colors=space.sky_colors)
        t = Twin(target, space, dev_space=late)
    t.check("side stream")
    t.close()


def fills():
    """(label, the block, derive its light on the device)."""
    derived = scenes.make_voxel_block(13, resolution=8, alpha=0.5, emissive_every=2)
    derived.set_light_data(aicb200.Context.default().derive_block_light([derived])[0])
    return [("single voxel", Block(color=(0.9, 0.35, 0.1, 1.0)), False),
            ("resolution-16 brick", scenes.make_voxel_block(21, resolution=16), False),
            ("wide block", big_palette_block(), False),
            ("derived light", derived, True)]


def test_fill_uniform_device_equals_the_host_twin(target):
    space = light_scene(seed=9)
    t = Twin(target, space, dev_space=False)
    for label, block, derive in fills():
        t.host.fill_uniform(block)
        t.dev.fill_uniform(on_device(block, derive))
        t.check(label)
        for lit in (t.host, t.dev):
            lit.light_queue_region(space.lower, space.size, 210)
            lit.light_evaluate(0)
        t.check(label + ", relit")
    t.close()


def test_fill_uniform_device_on_u32_cells(target):
    space = spaces("u32")
    t = Twin(target, space)
    t.check("created")
    b = scenes.make_voxel_block(22, resolution=16)
    t.host.fill_uniform(b)
    t.dev.fill_uniform(on_device(b))
    t.check("filled")
    t.close()


def test_rejected_fill_uniform_device_changes_nothing(target):
    space = scenes.small_mixed_scene(n=12, seed=7)
    t = Twin(target, space, dev_space=False)
    before = t.state(t.dev)
    lib = aicb200.load_library()
    bad_res = Block(resolution=3, indices=np.zeros((1, 1, 1), np.uint16), palette=np.zeros((1, 8), np.float32))
    bad_idx = scenes.make_voxel_block(4, resolution=4)
    bad_idx.indices = bad_idx.indices.copy()
    bad_idx.indices.flat[5] = bad_idx.palette.shape[0]
    for label, block in [("resolution", bad_res), ("voxel index", bad_idx)]:
        with pytest.raises(AicbError) as want:
            t.host.fill_uniform(block)
        with pytest.raises(AicbError) as got:
            t.dev.fill_uniform(on_device(block))
        assert (got.value.status, str(got.value)) == (want.value.status, str(want.value)), label
    host_desc = aicb200._block_descs([scenes.make_voxel_block(3, resolution=4)])
    assert t.dev.scene._fn("scene_fill_uniform_device")(t.dev.scene.handle, host_desc, 0, None) == abi.ERR_INVALID
    assert "not device memory" in lib.aicb_last_error().decode()
    assert t.dev.scene._fn("scene_fill_uniform_device")(t.dev.scene.handle, None, 0, None) == abi.ERR_INVALID
    assert_same(t.state(t.dev), before, "rejected")
    t.close()
