"""Block definitions fed from device memory (aicb_scene_update_blocks_device, aicb_scene_append_blocks_device and their
group forms): with each definition's indices and palette as CUDA tensors, a call must leave the scene byte for byte as
its host twin (aicb_scene_update_blocks / append_blocks with the same data) does.  Every check builds two scenes from
one Space on the same target (one context; groups of 1, 2 and 3 contexts of one device), updates one through the host
calls and the other through the device calls, and compares after every step: block ids, frames, device_bytes and, on
lit scenes, light_relight_blocks followed by light_evaluate."""
import numpy as np
import pytest
import torch

import aicb200
from aicb200 import AicbError, Block, BlockLight, DeviceBlock, GraphicsOptions, abi, scenes
from test_gpu_append_blocks import assert_same, every_output, narrow_space, new_blocks, placements, wide_blocks
from test_gpu_block_table import kind_changes
from test_gpu_light import light_scene
from test_gpu_light_changes import Lit

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
TARGETS = [None, [0], [0, 0], [0, 0, 0]]
TARGET_IDS = ["ctx", "group1", "group2", "group3"]
OPTS = GraphicsOptions(view_distance=40.0, lighting_display=aicb200.LIGHT_LINEAR)
W, H = 48, 40


def light_of(b: Block) -> BlockLight:
    return BlockLight(face_colors=tuple(tuple(c) for c in b.light_face_colors), color=tuple(b.light_color),
                      emission=tuple(b.light_emission), opaque_faces=int(b.light_opaque_faces),
                      visible=bool(b.light_visible))


def on_device(b: Block, derive=False, visible=False) -> DeviceBlock:
    """The same definition with its voxels as CUDA tensors; light as given, or derived on the device."""
    idx = None
    if b.indices is not None:
        idx = torch.from_numpy(b.indices.view(np.int16)).to(DEV).view(torch.uint16)
    pal = torch.from_numpy(np.ascontiguousarray(b.palette, dtype=np.float32).reshape(-1, 8)).to(DEV)
    return DeviceBlock(b.resolution, b.voxel_lower, idx, pal, is_air=b.is_air,
                       light=None if derive else light_of(b), visible=visible)


class Twin:
    """Two scenes of one Space on one target: `host` fed the host calls, `dev` the device calls."""

    def __init__(self, target, space):
        self.target, self.space = target, space
        self.host, self.dev = Lit(target, space), Lit(target, space)
        self.cam = scenes.standard_camera(space, OPTS, W, H)

    def update(self, indices, blocks, derive=False):
        self.host.update_blocks(indices, blocks)
        self.dev.update_blocks(indices, [on_device(b, derive) for b in blocks])

    def append(self, blocks, derive=False):
        self.host.append_blocks(blocks)
        self.dev.append_blocks([on_device(b, derive) for b in blocks])

    def state(self, lit):
        s = lit.scene
        out = {"ids": s.block_ids(), "frame": lit.frame(self.cam, OPTS)}
        if lit.group is None:
            out.update(every_output(s, OPTS, self.cam))
            out["device_bytes"] = np.array([s.device_bytes])
        return out

    def check(self, label, relight=None):
        assert_same(self.state(self.host), self.state(self.dev), label)
        if relight is not None and self.space.light_max_distance:
            for lit in (self.host, self.dev):
                lit.light_relight_blocks(relight)
                lit.light_evaluate(0)
            assert self.host.field().tobytes() == self.dev.field().tobytes(), f"{label}: light differs"

    def close(self):
        self.host.close()
        self.dev.close()


@pytest.fixture(params=TARGETS, ids=TARGET_IDS)
def target(request):
    return request.param


def test_kind_changes_and_appends(target):
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    t = Twin(target, mixed)
    indices, blocks = kind_changes()   # every kind transition, index 1 named twice
    t.update(indices, blocks)
    t.check("kind changes")
    n0 = len(mixed.blocks)
    t.append(new_blocks())
    cubes, ids = placements(mixed, range(n0, n0 + 5), 60, seed=4)
    t.host.update_cubes(cubes, ids)
    t.dev.update_cubes(cubes, ids)
    t.check("appended and placed")
    t.update([n0 + 2, n0, 3], [Block(color=(0.1, 0.2, 0.9, 1.0)), scenes.make_voxel_block(41, resolution=16),
                               scenes.make_voxel_block(42, resolution=2, alpha=0.5)])
    t.check("appended ids redefined")
    t.close()


def single_voxels():
    """indices=None; resolution 1 with one index at the origin; one index of a resolution-2 block, not at the origin
    (a brick, not a single voxel); n_palette == 0 (AIR)."""
    pal = np.array([[0.9, 0.1, 0.1, 1.0, 0, 0, 0, 0], [0.2, 0.7, 0.3, 0.5, 0.5, 0.5, 0.0, 0]], np.float32)
    at_origin = Block(resolution=1, indices=np.array([[[1]]], np.uint16), palette=pal)
    off_origin = Block(resolution=2, voxel_lower=(1, 0, 0), indices=np.array([[[0]]], np.uint16), palette=pal)
    empty = Block(color=(0.5, 0.5, 0.5, 1.0))
    empty.palette = np.zeros((0, 8), np.float32)
    empty.light_visible = False
    empty.light_color = (0.0, 0.0, 0.0, 0.0)
    empty.light_face_colors = [(0.0, 0.0, 0.0, 0.0)] * 6
    empty.light_emission = (0.0, 0.0, 0.0)
    empty.light_opaque_faces = 0
    return [Block(color=(0.3, 0.6, 0.9, 0.75)), at_origin, off_origin, empty]


def odd_palettes():
    """Partial voxel_bounds, and palettes with unused and duplicate entries."""
    rng = np.random.default_rng(5)
    pal = np.zeros((12, 8), np.float32)
    pal[:, :4] = rng.uniform(0, 1, (12, 4))
    pal[3] = pal[1]   # duplicate
    pal[5, 3] = 0.0   # invisible, unused
    pal[7, :] = 0.0
    idx = rng.choice(np.array([0, 1, 2, 3, 7], np.uint16), (5, 3, 6)).astype(np.uint16)
    return [Block(resolution=8, voxel_lower=(1, 2, 0), indices=idx, palette=pal),
            scenes.make_voxel_block(9, resolution=8, alpha=0.5, transparent_palette_entry=True, emissive_every=3)]


def test_single_voxels_partial_bounds_and_odd_palettes(target):
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    t = Twin(target, mixed)
    t.update([1, 2, 3, 10], single_voxels())
    t.check("single voxels")
    t.update([4, 11], odd_palettes())
    t.check("odd palettes")
    t.append(single_voxels() + odd_palettes())
    t.check("appended")
    t.close()


def test_lit_scene_relights_the_same(target):
    space = light_scene(seed=9)
    t = Twin(target, space)
    t.update([3, 1], [Block(color=(0.1, 0.9, 0.2, 0.25)), scenes.make_voxel_block(3, resolution=4, alpha=0.5)])
    t.check("lit update", relight=[3, 1])
    t.update([2], [Block.air()])
    t.check("opaque to air", relight=[2])
    t.close()


def test_wide_palette_and_wide_cells(target):
    rng = np.random.default_rng(11)
    pal = np.zeros((40000, 8), np.float32)
    pal[:, :3] = rng.uniform(0, 1, (40000, 3))
    pal[:, 3] = rng.choice(np.array([0.0, 0.5, 1.0], np.float32), 40000)
    big = Block(resolution=16, indices=rng.integers(0, 40000, (16, 16, 16)).astype(np.uint16), palette=pal)
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    t = Twin(target, mixed)
    t.update([11], [big])   # a palette over 32768 entries widens the narrow brick pool
    t.check("wide bricks")
    t.close()
    space = narrow_space()
    t = Twin(target, space)
    t.append(wide_blocks()[:2])
    t.append(wide_blocks()[2:])   # past 16384 ids: 32-bit cells
    cubes, ids = placements(space, [16383, 16384, 16400, 16419], 60, seed=9)
    t.host.update_cubes(cubes, ids)
    t.dev.update_cubes(cubes, ids)
    t.check("wide cells")
    t.update([16400, 5], [Block(color=(0.0, 0.0, 0.0, 0.0)), scenes.make_voxel_block(6, resolution=4)])
    t.check("kind changes in 32-bit cells")
    t.close()


def test_repeated_redefinitions_compact_both_pools():
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    t = Twin(None, mixed)
    for k in range(6):
        t.update([10 + k % 3], [scenes.make_voxel_block(60 + k, resolution=64, palette_size=24 + k)])
        t.check(f"redefinition {k}")
    t.close()


def test_derived_light_equals_derive_then_host_twin(target):
    space = light_scene(seed=9)
    t = Twin(target, space)
    blocks = [scenes.make_voxel_block(13, resolution=8, alpha=0.5, emissive_every=2),
              Block(color=(0.4, 0.4, 0.9, 0.5), emission=(0.2, 0.0, 0.1)), scenes.make_voxel_block(14, resolution=4)]
    derived = aicb200.Context.default().derive_block_light(blocks)
    for b, d in zip(blocks, derived):
        b.set_light_data(d)
    t.host.update_blocks([1, 3, 4], blocks)
    t.dev.update_blocks([1, 3, 4], [on_device(b, derive=True) for b in blocks])
    t.check("derived", relight=[1, 3, 4])
    # light_visible ORs in an animation hint: an invisible voxel block that is visible_or_animated
    inv = Block(resolution=2, indices=np.zeros((2, 2, 2), np.uint16), palette=np.zeros((1, 8), np.float32))
    inv.set_light_data(aicb200.Context.default().derive_block_light([inv])[0])
    assert not inv.light_visible
    inv.light_visible = True
    t.host.update_blocks([2], [inv])
    t.dev.update_blocks([2], [on_device(inv, derive=True, visible=True)])
    t.check("animation hint", relight=[2])
    t.close()


def _raw_call(lit, indices, descs, flags=0):
    """The device call with descriptors as given (the Python layer's checks bypassed)."""
    arr = (abi.BlockDesc * len(descs))(*descs)
    if indices is None:
        return lit.scene._fn("scene_append_blocks_device")(lit.scene.handle, arr, len(descs), flags, None)
    idx = np.ascontiguousarray(indices, np.uint16)
    return lit.scene._fn("scene_update_blocks_device")(lit.scene.handle, idx.ctypes.data, arr, len(descs), flags, None)


def _descs(blocks, derive=False):
    out, keep = [], {}
    for b in blocks:   # (a block listed many times goes to the device once)
        if id(b) not in keep:
            keep[id(b)] = on_device(b, derive)
        d = abi.BlockDesc()
        keep[id(b)].fill_desc(d)
        out.append(d)
    return out, keep


def _host_descs(blocks):
    arr = aicb200._block_descs(blocks)
    return [arr[i] for i in range(len(blocks))]


def rejections(n_blocks):
    """(label, indices or None for an append, blocks, how to spoil the descriptors) of every host-side check."""
    good = scenes.make_voxel_block(3, resolution=4)
    bad_idx = scenes.make_voxel_block(4, resolution=4)
    bad_idx.indices = bad_idx.indices.copy()
    bad_idx.indices.flat[5] = bad_idx.palette.shape[0]
    big = Block(resolution=4, indices=np.zeros((4, 4, 4), np.uint16), palette=np.zeros((65537, 8), np.float32))

    def field(name, value, at=0):
        def spoil(ds):
            setattr(ds[at], name, value)
        return spoil

    def bounds(ds):
        ds[0].voxel_bounds.lower[0] = 2
    return [
        ("resolution", [1], [good], field("resolution", 3)),
        ("n_indices", [1], [good], field("n_indices", 7)),
        ("bounds", [1], [good], bounds),
        ("index past the table", [n_blocks], [good], None),
        ("bad voxel index in block 2", [1, 2, 3], [good, good, bad_idx], None),
        ("bad voxel index, then a bad resolution", [1, 2], [bad_idx, good], field("resolution", 3, 1)),
        ("palette over 65536", [1], [big], None),
        ("a bad voxel index before a palette over 65536", [1, 2], [bad_idx, big], None),
        ("append past 65536 ids", None, [good] * (65537 - n_blocks), None),
    ]


def test_every_rejection_matches_the_host_twin():
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    t = Twin(None, mixed)
    before = t.state(t.dev)
    for label, indices, blocks, spoil in rejections(len(mixed.blocks)):
        hd = _host_descs(blocks)
        dd, keep = _descs(blocks)
        if spoil:
            spoil(hd)
            spoil(dd)
        lib = aicb200.load_library()
        st_host = _raw_host(t.host, indices, hd)
        msg_host = lib.aicb_last_error().decode()
        st_dev = _raw_call(t.dev, indices, dd)
        msg_dev = lib.aicb_last_error().decode()
        assert st_host != abi.OK, label
        assert (st_dev, msg_dev) == (st_host, msg_host), label
        assert_same(t.state(t.dev), before, label)
    t.close()


def _raw_host(lit, indices, descs):
    arr = (abi.BlockDesc * len(descs))(*descs)
    if indices is None:
        return lit.scene._fn("scene_append_blocks")(lit.scene.handle, arr, len(descs))
    idx = np.ascontiguousarray(indices, np.uint16)
    return lit.scene._fn("scene_update_blocks")(lit.scene.handle, idx.ctypes.data, arr, len(descs))


def test_pointer_and_derive_rejections_change_nothing():
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    t = Twin(None, mixed)
    before = t.state(t.dev)
    lib = aicb200.load_library()
    good = scenes.make_voxel_block(3, resolution=4)
    host_block = _host_descs([good])   # host memory where device memory goes
    assert _raw_call(t.dev, [1], host_block) == abi.ERR_INVALID
    assert "not device memory" in lib.aicb_last_error().decode()
    dd, keep = _descs([good])
    dd[0].indices += 1   # misaligned
    assert _raw_call(t.dev, [1], dd) == abi.ERR_INVALID
    assert "aligned" in lib.aicb_last_error().decode()
    if torch.cuda.device_count() > 1:
        other = torch.zeros(64, dtype=torch.int16, device=torch.device("cuda", 1))
        dd, keep = _descs([good])
        dd[0].indices = other.data_ptr()
        assert _raw_call(t.dev, [1], dd) == abi.ERR_INVALID
        assert "another device" in lib.aicb_last_error().decode()
    # a NaN colour sum: derive's status and message, naming the block
    pal = np.zeros((3, 8), dtype=np.float32)   # +inf and -inf emission: a NaN sum
    pal[1, :4] = pal[2, :4] = (1.0, 1.0, 1.0, 0.5)
    pal[1, 4], pal[2, 4] = np.inf, -np.inf
    idx = np.ones((4, 4, 4), dtype=np.uint16)
    idx[:, :, 2:] = 2
    blocks = [good, Block(resolution=4, indices=idx, palette=pal)]
    with pytest.raises(AicbError) as want:
        aicb200.Context.default().derive_block_light(blocks)
    dd, keep = _descs(blocks, derive=True)
    assert _raw_call(t.dev, [1, 2], dd, abi.BLOCKS_DERIVE_LIGHT) == want.value.status
    assert "block 1: its colour or emission sum is NaN" in lib.aicb_last_error().decode()
    assert lib.aicb_last_error().decode() in str(want.value)
    assert_same(t.state(t.dev), before, "rejected")
    with pytest.raises(ValueError):
        t.dev.update_blocks([1, 2], [on_device(good), good])
    t.close()


def test_inputs_written_on_a_side_stream():
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    t = Twin(None, mixed)
    b = scenes.make_voxel_block(17, resolution=32, palette_size=20)
    side = torch.cuda.Stream(DEV)
    with torch.cuda.stream(side):
        idx = torch.zeros(b.indices.shape, dtype=torch.int32, device=DEV)
        torch.cuda._sleep(20_000_000)   # the producer is still running when the call is issued
        idx += torch.from_numpy(b.indices.astype(np.int32)).to(DEV)
        pal = torch.from_numpy(b.palette).to(DEV) * 1.0
        db = DeviceBlock(b.resolution, b.voxel_lower, idx.to(torch.uint16), pal, light=light_of(b))
        t.dev.update_blocks([12], [db])
    side.synchronize()
    t.host.update_blocks([12], [b])
    t.check("side stream")
    t.close()
