"""The light side of a block redefinition (aicb_light_relight_blocks / aicb_group_light_relight_blocks): after
update_blocks gives an index a new definition, every cube holding it takes Mutation::set's light rule
(modified_cube_needs_update, space/light/updater.rs:135-173) with that definition, found by a scan of the cells on the
device, and the light relaxes.  Converged fields must meet the light contract of tests/test_gpu_light.py against the
oracle doing the same (oracle_light/), and the edit path that places a copy of the new definition in those cubes.
Every check runs on one context and on groups of 1, 2 and 3 contexts of one device; a group's replicas stay
identical."""
import numpy as np
import pytest

import aicb200
from aicb200 import AicbError, Block, GraphicsOptions, Space, SpaceRaytracer, abi, scenes
from lightorc import LightOracle
from test_gpu_light import OPAQUE, VISIBLE, compare_fields, light_scene
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit

pytestmark = pytest.mark.gpu

# light_scene's block 2 (opaque green), as it is and as a lamp
LAMP_OFF = Block(color=(0.2, 0.9, 0.3, 1.0))
LAMP_ON = Block(color=(0.2, 0.9, 0.3, 1.0), emission=(3.0, 2.0, 1.0))
# light_scene's block 3 (translucent red) made opaque
RED_WALL = Block(color=(0.9, 0.2, 0.1, 1.0))


def converged(devices, space):
    """The scene on `devices` and the oracle, both converged to epsilon 0, the set of changed cubes emptied."""
    lit = Lit(devices, space)
    lit.light_fast_evaluate()
    lit.light_evaluate(0)
    lit.light_take_changes(discard=True)
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    return lit, ol


def redefine(lit, ol, index, block):
    """update_blocks + light_relight_blocks on the scene, the same on the oracle; the scene's (updates, max_diff)."""
    lit.update_blocks([index], [block])
    got = lit.light_relight_blocks([index], 0)
    ol.update_blocks([index], [block])
    ol.relight_blocks([index])
    ol.evaluate(0)
    return got


def holders(space, index):
    """The cubes holding `index` and their linear indices, in increasing order."""
    at = np.argwhere(space.block_ids == index)
    return (at + np.array(space.lower)).astype(np.int32), np.ravel_multi_index(at.T, space.size)


def with_blocks(space, changes, field):
    blocks = list(space.blocks)
    for i, b in changes.items():
        blocks[i] = b
    return Space(space.lower, space.block_ids, blocks, light=field, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_lamp_on_and_off(devices):
    space = light_scene(seed=9)
    lit, ol = converged(devices, space)
    _, lamps = holders(space, 2)
    assert len(lamps) > 0
    updates, _ = redefine(lit, ol, 2, LAMP_ON)
    assert updates > 0
    on = lit.field()
    compare_fields(on, ol.field())
    assert (on.reshape(-1, 4)[lamps, 3] == VISIBLE).all()   # an opaque emitter takes its emission as its light
    updates, _ = redefine(lit, ol, 2, LAMP_OFF)
    assert updates > 0
    off = lit.field()
    compare_fields(off, ol.field())
    assert (off.reshape(-1, 4)[lamps, 3] == OPAQUE).all()
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_block_becomes_opaque(devices):
    space = light_scene(seed=9)
    lit, ol = converged(devices, space)
    _, walls = holders(space, 3)
    assert len(walls) > 0
    before = lit.field()
    assert not (before.reshape(-1, 4)[walls, 3] == OPAQUE).any()
    redefine(lit, ol, 3, RED_WALL)
    field = lit.field()
    assert (field.reshape(-1, 4)[walls, 3] == OPAQUE).all()
    taken, texels = lit.light_take_changes()
    assert set(walls.tolist()) <= set(taken.tolist())
    assert np.array_equal(texels, field.reshape(-1, 4)[taken])
    compare_fields(field, ol.field())
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_relight_equals_the_edit_path(devices):
    """Relighting L after redefining it, and placing a copy L' of the new definition in every cube holding L with a
    propagating edit, queue the same cubes: the fields meet the contract against each other."""
    space = light_scene(seed=9)
    for index, block in ((3, RED_WALL), (4, Block(color=(0.3, 0.3, 0.9, 0.5), emission=(0.5, 1.0, 2.0))),
                         (1, Block(color=(0.1, 0.3, 0.9, 1.0)))):
        relit, _ = converged(devices, space)
        edited, _ = converged(devices, space)
        relit.update_blocks([index], [block])
        n_relit, _ = relit.light_relight_blocks([index], 0)
        edited.append_blocks([block])
        cubes, _ = holders(space, index)
        n_edited, _ = edited.light_edit_and_propagate(cubes, np.full(len(cubes), len(space.blocks), dtype=np.uint16), 0)
        assert n_relit > 0 and n_edited > 0
        compare_fields(relit.field(), edited.field())
        relit.close()
        edited.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_relit_field_is_quiescent(devices):
    space = light_scene(seed=9)
    lit, ol = converged(devices, space)
    redefine(lit, ol, 3, RED_WALL)
    assert lit.light_evaluate(0)[0] == 0
    stats = lit.light_stats()
    assert stats["cube_updates"] == 0
    # an index that no cube holds, and an empty list, add nothing
    lit.append_blocks([Block(color=(1.0, 1.0, 1.0, 1.0), emission=(5.0, 5.0, 5.0))])
    lit.light_take_changes(discard=True)
    field = lit.field()
    assert lit.light_relight_blocks([len(space.blocks)], 0) == (0, 0)
    assert lit.light_relight_blocks([], 0) == (0, 0)
    assert lit.light_changes_count() == 0
    assert np.array_equal(lit.field(), field)
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_frames_follow_the_relit_light(devices):
    space = light_scene(seed=9)
    lit, ol = converged(devices, space)
    redefine(lit, ol, 2, LAMP_ON)
    redefine(lit, ol, 3, RED_WALL)
    field = lit.field()
    opts = GraphicsOptions(lighting_display=aicb200.LIGHT_LINEAR)
    cam = scenes.standard_camera(space, opts, 64, 48)
    fresh = SpaceRaytracer(with_blocks(space, {2: LAMP_ON, 3: RED_WALL}, field), opts)
    assert np.array_equal(lit.frame(cam, opts), aicb200.render_layers((fresh, cam, opts)).data)
    fresh.close()
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_wide_cells(devices):
    """A table grown past 16384 blocks holds u32 cells: a cube holding a high index is found by the u32 scan."""
    space = light_scene(seed=9)
    lit, ol = converged(devices, space)
    high = 16400
    filler = [Block(color=(0.5, 0.5, 0.5, 1.0))] * (high - len(space.blocks))
    new = filler + [Block(color=(0.8, 0.3, 0.3, 0.5))]
    lit.append_blocks(new)
    ol.append_blocks(new)
    cubes, _ = holders(space, 3)
    ids = np.full(len(cubes), high, dtype=np.uint16)
    lit.light_edit_and_propagate(cubes, ids, 0)
    ol.set_cubes(cubes, ids)
    ol.evaluate(0)
    compare_fields(lit.field(), ol.field())
    updates, _ = redefine(lit, ol, high, Block(color=(0.8, 0.3, 0.3, 1.0), emission=(2.0, 1.0, 0.5)))
    assert updates > 0
    compare_fields(lit.field(), ol.field())
    updates, _ = redefine(lit, ol, high, Block(color=(0.8, 0.3, 0.3, 1.0)))
    assert updates > 0
    field = lit.field()
    _, walls = holders(space, 3)
    assert (field.reshape(-1, 4)[walls, 3] == OPAQUE).all()
    compare_fields(field, ol.field())
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_rejected_relights_change_nothing(devices):
    space = light_scene(seed=9)
    lit, _ = converged(devices, space)
    lit.update_blocks([3], [RED_WALL])   # a relight would now change the field
    opts = GraphicsOptions(lighting_display=aicb200.LIGHT_LINEAR)
    cam = scenes.standard_camera(space, opts, 64, 48)
    field, frame = lit.field(), lit.frame(cam, opts)
    fn = lit.scene._fn("light_relight_blocks")
    calls = [lambda: aicb200._check(fn(lit.scene.handle, None, 2, 0, None, None)),
             lambda: lit.light_relight_blocks([3, len(space.blocks)], 0),
             lambda: lit.light_relight_blocks([65535], 0)]
    for call in calls:
        with pytest.raises(AicbError) as e:
            call()
        assert e.value.status == abi.ERR_INVALID
        assert np.array_equal(lit.field(), field)   # (on a group: every replica, checked identical)
        assert lit.light_changes_count() == 0
        assert np.array_equal(lit.frame(cam, opts), frame)
    assert lit.light_relight_blocks([3], 0)[0] > 0
    lit.close()
    unlit = Lit(devices, Space(space.lower, space.block_ids, space.blocks, sky_colors=space.sky_colors,
                               light_max_distance=0))
    with pytest.raises(AicbError) as e:
        unlit.light_relight_blocks([3], 0)
    assert e.value.status == abi.ERR_INVALID
    unlit.close()
