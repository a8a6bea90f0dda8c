"""aicb_light_edit_cubes and its group form: Mutation::set x n in list order without propagation, the light rule on the
device against the final cells (DESIGN.md §4b).  Before any propagation its queue, texels, set of changed cubes and
count must equal the oracle's entry-by-entry result byte for byte, and its frames those of a scene created from the
edited Space; after propagation its light must meet the contract of tests/test_gpu_light.py against the oracle and
against aicb_light_edit_and_propagate.  Every check runs on one context and on groups of 1, 2 and 3 contexts of one
device; a group's replicas stay identical."""
import ctypes as C

import numpy as np
import pytest

from aicb200 import AicbError, Block, Space, SpaceRaytracer, abi, scenes
from editlists import edit_cubes_rule, edit_list, kinds
from resumeorc import LightOracle
from test_gpu_append_blocks import OPTIONS, assert_same, every_output, narrow_space, wide_blocks
from test_gpu_light import compare_fields, light_scene
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit
from test_gpu_region import assert_frames_equal, frames, fresh_frames, with_light

pytestmark = pytest.mark.gpu

QUEUED = ((0, 2, 5), (6, 8, 6), 230)   # cubes queued before the edits, so that cancellations show


def converge(space):
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    return with_light(space, ol.field())


@pytest.fixture(scope="module")
def converged_space():
    """light_scene with the oracle's converged light: a scene and an oracle created from it hold the same texels."""
    return converge(light_scene(seed=9))


def wide_light_space():
    """narrow_space with its table grown past 16384 blocks (a scene created from it has 32-bit cells), lit."""
    space = narrow_space()
    return Space(space.lower, space.block_ids, space.blocks + wide_blocks(), light=space.light,
                 sky_colors=space.sky_colors, light_max_distance=12)


def scattered(space, n, batch):
    """scenes.c4_edits' random draws on `space`: cubes from the lower quarter upwards, any block of the table."""
    cubes, ids = scenes.c4_edits(space, n, batch)
    cubes = np.minimum(cubes, np.array(space.size) - 1) + np.array(space.lower)
    return cubes.astype(np.int32), ids


def lists(space, form):
    """Three consecutive lists of the form."""
    rng = np.random.default_rng({"mixed": 1, "scattered": 2, "opaque": 3, "air": 4, "lamp": 5, "wide": 6}[form])
    for k in range(3):
        if form == "mixed":
            yield edit_list(space, seed=40 + k)
        elif form == "scattered":
            yield scattered(space, 200, k)
        elif form == "wide":
            cubes, _ = scattered(space, 150, k)
            n0 = len(space.blocks) - len(wide_blocks())
            pick = [0, 3, 16300, 16383, n0, n0 + 1, n0 + 5, n0 + 9, n0 + 39]
            ids = rng.choice(np.asarray(pick, dtype=np.uint16), len(cubes)).astype(np.uint16)
            dup = rng.integers(0, len(cubes), len(cubes) // 3)   # cubes named again later in the list
            again = rng.choice(np.asarray(pick, dtype=np.uint16), len(dup)).astype(np.uint16)
            yield np.concatenate([cubes, cubes[dup]]), np.concatenate([ids, again])
        else:
            cubes = np.stack([rng.integers(0, space.size[a], 120) + space.lower[a] for a in range(3)], axis=1)
            block = {"opaque": 1, "air": 0, "lamp": 5}[form]
            yield cubes.astype(np.int32), np.full(len(cubes), block, dtype=np.uint16)


def edited_space(space, final, light):
    return Space(space.lower, final, space.blocks, light=light, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


@pytest.mark.parametrize("form", ["mixed", "scattered", "opaque", "air", "lamp", "wide"])
@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_edit_cubes_equals_sets_in_order_before_any_propagation(converged_space, devices, form):
    space = converge(wide_light_space()) if form == "wide" else converged_space
    lit, ol = Lit(devices, space), LightOracle(space)
    lit.light_queue_region(*QUEUED)
    ol.queue_region(*QUEUED)
    for cubes, ids in lists(space, form):
        n, final, queue, field, changed = edit_cubes_rule(space, ol.queue(), ol.field(), cubes, ids)
        assert lit.light_edit_cubes(cubes, ids) == n
        ol.set_cubes(cubes, ids)
        assert np.array_equal(queue, ol.queue()) and np.array_equal(field, ol.field())   # the rule is the oracle's
        got_queue, got_field = lit.light_download_queue(), lit.field()
        assert np.array_equal(got_queue, queue), np.argwhere(got_queue != queue)[:4]
        assert np.array_equal(got_field, field), np.argwhere((got_field != field).any(axis=-1))[:4]
        idx, tx = lit.light_take_changes()
        assert idx.tolist() == changed
        assert np.array_equal(tx, field.reshape(-1, 4)[idx])
        space = edited_space(space, final, field)
        assert_frames_equal(frames(lit, space), fresh_frames(space), f"{form}")
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_edit_cubes_then_evaluate_converges_like_the_oracle_and_the_propagating_call(converged_space, devices):
    space = converged_space
    ol = LightOracle(space)
    edits, propagating = Lit(devices, space), Lit(devices, space)
    for cubes, ids in list(lists(space, "mixed")) + list(lists(space, "scattered")):
        edits.light_edit_cubes(cubes, ids)
        assert edits.light_evaluate(0)[0] > 0
        assert propagating.light_edit_and_propagate(cubes, ids, 0)[0] > 0
        ol.set_cubes(cubes, ids)
        ol.evaluate(0)
        field = edits.field()
        compare_fields(field, ol.field())
        compare_fields(field, propagating.field())
        assert edits.light_evaluate(0)[0] == 0   # quiescent
        assert not edits.light_download_queue().any()
    edits.close()
    propagating.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_tick_loop_converges(converged_space, devices):
    """update_light_system's tick: this tick's CubeBlock batch, then one budgeted step; after the last batch the ticks
    go on until the queue is empty."""
    space = converged_space
    lit, ol = Lit(devices, space), LightOracle(space)
    batches = list(lists(space, "scattered")) + list(lists(space, "mixed"))
    for cubes, ids in batches:
        lit.light_edit_cubes(cubes, ids)
        info = lit.light_update_from_queue(300)
        assert 0 < info["update_count"] <= 300
        ol.set_cubes(cubes, ids)
    for _ in range(10000):
        if lit.light_update_from_queue(300)["queue_count"] == 0:
            break
    assert not lit.light_download_queue().any()
    ol.evaluate(0)
    compare_fields(lit.field(), ol.field())
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_host_mirror_follows_the_edits(converged_space, devices):
    """aicb_scene_update_blocks re-encodes the cells of a redefined block from the host mirror: a block edited in by the
    list turns from a single voxel into a brick and back, and the frames (on one context every output) equal those of a
    scene created from the edited Space."""
    space = converged_space
    lit = Lit(devices, space)
    cubes, ids = edit_list(space, seed=7)
    glass = kinds(space)["glass"][0]
    ids[::5] = glass
    n, final, _, _, _ = edit_cubes_rule(space, np.zeros(space.size, np.uint8), space.light, cubes, ids)
    assert lit.light_edit_cubes(cubes, ids) == n and (final == glass).any()
    blocks = list(space.blocks)
    for b in (scenes.make_voxel_block(3, resolution=8, alpha=0.5), Block(color=(0.3, 0.8, 0.2, 0.5))):
        lit.update_blocks([glass], [b])
        blocks[glass] = b
        edited = Space(space.lower, final, blocks, light=lit.field(), sky_colors=space.sky_colors,
                       light_max_distance=space.light_max_distance)
        assert_frames_equal(frames(lit, edited), fresh_frames(edited), f"block {glass} as {type(b).__name__}")
        if devices is None:
            fresh = SpaceRaytracer(edited, OPTIONS[0], lit.scene.ctx)
            for opts in OPTIONS[:2]:
                cam = scenes.standard_camera(space, opts, 64, 48)
                assert_same(every_output(lit.scene, opts, cam), every_output(fresh, opts, cam), f"block {glass}")
            fresh.close()
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_rejected_calls_change_nothing(converged_space, devices):
    space = converged_space
    lit = Lit(devices, space)
    lit.light_queue_region(*QUEUED)
    field, queue, changed, frame = lit.field(), lit.light_download_queue(), lit.light_changes_count(), frames(lit, space)
    cubes, ids = edit_list(space, seed=5)
    outside = cubes.copy()
    outside[-1] = (space.lower[0], space.lower[1] + space.size[1], space.lower[2])
    past = ids.copy()
    past[-1] = len(space.blocks)
    for c, i in ((outside, ids), (cubes, past)):
        with pytest.raises(AicbError) as e:
            lit.light_edit_cubes(c, i)
        assert e.value.status == abi.ERR_INVALID
    with pytest.raises(ValueError):
        lit.light_edit_cubes(cubes, ids[:-1])
    fn = lit._fn("light_edit_cubes")
    n = C.c_size_t(5)
    assert fn(lit.handle, None, ids.ctypes.data, 3, C.byref(n)) == abi.ERR_INVALID
    assert fn(lit.handle, cubes.ctypes.data, None, 3, C.byref(n)) == abi.ERR_INVALID
    assert fn(None, cubes.ctypes.data, ids.ctypes.data, 3, None) == abi.ERR_INVALID
    assert fn(lit.handle, cubes.ctypes.data, ids.ctypes.data, 1 << 32, None) == abi.ERR_INVALID
    # n == 0 changes nothing and reports 0, NULL arrays included
    assert fn(lit.handle, None, None, 0, C.byref(n)) == abi.OK and n.value == 0
    assert lit.light_edit_cubes(np.zeros((0, 3), np.int32), np.zeros(0, np.uint16)) == 0
    assert np.array_equal(lit.field(), field) and np.array_equal(lit.light_download_queue(), queue)
    assert lit.light_changes_count() == changed
    assert_frames_equal(frames(lit, space), frame, "after the rejected calls")
    lit.close()
    unlit = Lit(devices, Space(space.lower, space.block_ids, space.blocks, sky_colors=space.sky_colors, light_max_distance=0))
    before = frames(unlit, space)
    with pytest.raises(AicbError) as e:
        unlit.light_edit_cubes(cubes, ids)
    assert e.value.status == abi.ERR_INVALID
    assert_frames_equal(frames(unlit, space), before, "LightPhysics::None")
    unlit.close()
