"""The set of changed cubes (aicb_light_changes_count / aicb_light_take_changes and their group forms): the cubes whose
light texel the light calls wrote, SpaceChange::CubeLight in the reference (space.rs:1079-1083), taken by the host in
increasing index order with their texels as they are at the take.  Every check runs on one context and on groups of 1,
2 and 3 contexts of one device; a group's set is device 0's, and its replicas stay identical."""
import ctypes as C

import numpy as np
import pytest

import aicb200
from aicb200 import AicbError, Block, GraphicsOptions, Space, SpaceRaytracer, abi, scenes
from test_gpu_group_light import assert_replicas_identical, c4_slice, group_scene
from test_gpu_light import NO_RAYS, OPAQUE, VISIBLE, WHITE, all_cubes, empty_space, light_scene

pytestmark = pytest.mark.gpu

TARGETS = (None, [0], [0, 0], [0, 0, 0])   # None: one context
TARGET_IDS = ("ctx", "group1", "group2", "group3")


class Lit:
    """A scene on one context or on a group, with the light calls both have and the group's own downloads."""

    def __init__(self, devices, space):
        self.devices = devices
        self.space = space
        if devices is None:
            self.group = None
            self.scene = SpaceRaytracer(space, GraphicsOptions())
        else:
            self.group, self.scene = group_scene(devices, space)

    def __getattr__(self, name):
        return getattr(self.scene, name)

    def field(self):
        """The light volume; on a group every replica's, checked identical."""
        if self.group is None:
            return self.scene.light_download()
        return assert_replicas_identical(self.scene, len(self.devices))

    def frame(self, cam, opts):
        if self.group is None:
            return aicb200.render_layers((self.scene, cam, opts)).data
        return self.group.render_layers((self.scene, cam, opts)).data

    def abi_calls(self):
        return self.scene._fn("light_changes_count"), self.scene._fn("light_take_changes"), self.scene.handle

    def close(self):
        (self.scene if self.group is None else self.group).close()


def opaque_for_light(block):
    """EvaluatedBlock::opaque_for_light_computation: opaque on every face and not emitting light."""
    return block.light_opaque_faces == 0x3F and not any(v != 0.0 for v in block.light_emission)


def cubes_set_opaque(space, cubes, ids):
    """Linear indices of the edited cubes whose block changed to one opaque for light, the edits applied in order."""
    cur = space.block_ids.copy()
    out = set()
    for c, i in zip(cubes, ids):
        at = tuple(np.asarray(c) - np.array(space.lower))
        if cur[at] == i:
            continue
        cur[at] = i
        if opaque_for_light(space.blocks[i]):
            out.add(int(np.ravel_multi_index(at, space.size)))
    return out


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_set_cube_opaque_notification(devices):
    """light/tests.rs:176-202: setting the only cube of a 1^3 space to an opaque block announces that cube."""
    s = Lit(devices, empty_space((1, 1, 1), [Block(color=WHITE)]))
    assert s.light_changes_count() == 0   # no light call yet
    s.light_edit_and_propagate([(0, 0, 0)], [1], 0)
    assert s.light_changes_count() == 1
    idx, tx = s.light_take_changes()
    assert idx.dtype == np.uint32 and tx.dtype == np.uint8 and tx.shape == (1, 4)
    assert idx.tolist() == [0] and tuple(tx[0]) == (0, 0, 0, OPAQUE)
    assert s.light_changes_count() == 0
    s.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_step_announces_the_cubes_it_lit(devices):
    """light/tests.rs:108-156: in 3x1x1 under a red sky, setting (0,0,0) to white stores OPAQUE there and lights
    (1,0,0); (2,0,0) sees no surface and is not written."""
    s = Lit(devices, empty_space((3, 1, 1), [Block(color=WHITE)], sky=[(1.0, 0.0, 0.0)]))
    s.light_edit_and_propagate([(0, 0, 0)], [1], 0)
    idx, tx = s.light_take_changes()
    assert idx.tolist() == [0, 1]
    assert tuple(tx[0]) == (0, 0, 0, OPAQUE) and tuple(tx[1]) == (144, 0, 0, VISIBLE)
    assert tuple(s.field()[2, 0, 0]) == (0, 0, 0, NO_RAYS)
    s.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_fast_evaluate_announces_exactly_the_texels_it_changed(devices):
    space = light_scene()
    before = space.light.reshape(-1, 4).copy()
    s = Lit(devices, space)
    s.light_fast_evaluate()
    after = s.field().reshape(-1, 4)
    changed = np.flatnonzero((before != after).any(axis=1))
    assert 0 < len(changed) < len(before)
    idx, tx = s.light_take_changes()
    assert np.array_equal(idx, changed)
    assert np.array_equal(tx, after[idx])
    s.close()


@pytest.mark.parametrize("make,n_edits", [(lambda: light_scene(seed=9), 60), (c4_slice, 300)],
                         ids=["light_scene", "c4_slice"])
@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_propagation_announces_every_texel_it_changed(devices, make, n_edits):
    space = make()
    s = Lit(devices, space)
    s.light_fast_evaluate()
    s.light_evaluate(0)
    s.light_take_changes()
    assert s.light_changes_count() == 0
    before = s.field().reshape(-1, 4)
    rng = np.random.default_rng(4)
    cubes = np.stack([rng.integers(0, space.size[a], n_edits) + space.lower[a] for a in range(3)], axis=1).astype(np.int32)
    ids = rng.integers(0, len(space.blocks), n_edits).astype(np.uint16)
    updates, _ = s.light_edit_and_propagate(cubes, ids, 0)
    assert updates > 0
    after = s.field().reshape(-1, 4)
    assert s.light_changes_count() > 0
    idx, tx = s.light_take_changes()
    assert (np.diff(idx.astype(np.int64)) > 0).all(), "indices not strictly increasing"
    assert np.array_equal(tx, after[idx]), "texels differ from the downloaded field"
    taken = set(idx.tolist())
    changed = np.flatnonzero((before != after).any(axis=1))
    missing = [int(i) for i in changed if int(i) not in taken]
    assert not missing, f"{len(missing)} changed texels not announced, e.g. {missing[:5]}"
    opaque = cubes_set_opaque(space, cubes, ids)
    assert opaque and opaque <= taken, sorted(opaque - taken)[:5]
    # every cube update stores at most its own texel and guesses into its six neighbours
    assert len(idx) <= 7 * updates + n_edits, (len(idx), updates)
    again_idx, again_tx = s.light_take_changes()
    assert len(again_idx) == 0 and again_tx.shape == (0, 4)
    s.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_calls_that_write_no_light_add_nothing(devices):
    space = light_scene(seed=9)
    s = Lit(devices, space)
    s.light_fast_evaluate()
    s.light_evaluate(0)
    s.light_take_changes(discard=True)
    assert s.light_changes_count() == 0
    field = s.field()
    cubes = all_cubes(space)
    s.light_compute(cubes[:64])
    assert s.light_changes_count() == 0, "light_compute"
    lit = np.array([(7, 9, 11, VISIBLE), (1, 2, 3, VISIBLE)], dtype=np.uint8)
    s.update_cubes(cubes[100:102], space.block_ids.reshape(-1)[100:102], lit)
    assert s.light_changes_count() == 0, "update_cubes"
    s.upload_light(field)
    assert s.light_changes_count() == 0, "upload_light"
    opts = GraphicsOptions(lighting_display=aicb200.LIGHT_LINEAR)
    s.frame(scenes.standard_camera(space, opts, 64, 48), opts)
    assert s.light_changes_count() == 0, "a frame"
    inside = [space.lower[0] + 2, space.lower[1] + 3, space.lower[2] + 4]
    outside = [space.lower[0] + space.size[0], space.lower[1], space.lower[2]]
    for edit_cubes, edit_ids in (([inside, outside], [1, 1]), ([inside, inside], [1, len(space.blocks)])):
        with pytest.raises(AicbError) as e:
            s.light_edit_and_propagate(np.array(edit_cubes, dtype=np.int32), np.array(edit_ids, dtype=np.uint16), 0)
        assert e.value.status == abi.ERR_INVALID
        assert s.light_changes_count() == 0, "a rejected edit"
    s.close()
    # evaluate_light with nothing queued (light/tests.rs:162-174): 0 updates, nothing announced
    s = Lit(devices, empty_space((3, 1, 1), [Block(color=WHITE)]))
    assert s.light_evaluate(0)[0] == 0
    assert s.light_changes_count() == 0
    s.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_take_rules_of_the_c_abi(devices):
    space = light_scene(seed=9)
    s = Lit(devices, space)
    s.light_fast_evaluate()
    count_fn, take_fn, handle = s.abi_calls()
    n = s.light_changes_count()
    assert n > 1
    idx = np.zeros(n, dtype=np.uint32)
    tx = np.zeros((n, 4), dtype=np.uint8)
    got = C.c_size_t(12345)
    assert take_fn(handle, idx.ctypes.data, tx.ctypes.data, n - 1, C.byref(got)) == abi.ERR_INVALID
    assert got.value == n and s.light_changes_count() == n
    assert take_fn(handle, idx.ctypes.data, None, n, C.byref(got)) == abi.ERR_INVALID
    assert take_fn(handle, None, tx.ctypes.data, n, C.byref(got)) == abi.ERR_INVALID
    assert s.light_changes_count() == n
    got = C.c_size_t(0)
    assert take_fn(handle, idx.ctypes.data, tx.ctypes.data, n, C.byref(got)) == abi.OK
    assert got.value == n
    first = idx.copy()
    # the same writes again, then discarded without a copy
    s.upload_light(space.light)
    s.light_fast_evaluate()
    assert s.light_changes_count() == n
    got = C.c_size_t(0)
    assert take_fn(handle, None, None, 0, C.byref(got)) == abi.OK
    assert got.value == n and s.light_changes_count() == 0
    assert take_fn(handle, idx.ctypes.data, tx.ctypes.data, n, C.byref(got)) == abi.OK and got.value == 0
    assert (np.diff(first.astype(np.int64)) > 0).all()
    s.close()
    unlit = Space(space.lower, space.block_ids, space.blocks, sky_colors=space.sky_colors, light_max_distance=0)
    s = Lit(devices, unlit)
    count_fn, take_fn, handle = s.abi_calls()
    got = C.c_size_t(0)
    assert count_fn(handle, C.byref(got)) == abi.ERR_INVALID
    assert take_fn(handle, idx.ctypes.data, tx.ctypes.data, n, C.byref(got)) == abi.ERR_INVALID
    assert take_fn(handle, None, None, 0, C.byref(got)) == abi.ERR_INVALID
    with pytest.raises(AicbError) as e:
        s.light_changes_count()
    assert e.value.status == abi.ERR_INVALID
    s.close()
