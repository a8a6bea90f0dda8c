"""The box calls (aicb_scene_update_region / aicb_light_edit_region and their group forms): Space::fill and
fill_uniform over a region as one call per box.  aicb_light_edit_region is Mutation::set for every cube of the box in
interior_iter order (space.rs:1392-1412): its queue, texels and set of changed cubes must equal the oracle's byte for
byte before any propagation, and its converged light must meet the contract of tests/test_gpu_light.py against the
oracle and against aicb_light_edit_and_propagate with the cubes listed.  aicb_scene_update_region must equal
aicb_scene_update_cubes with the cubes listed, on 16-bit and 32-bit cells.  Every check runs on one context and on
groups of 1, 2 and 3 contexts of one device; a group's replicas stay identical."""
import ctypes as C

import numpy as np
import pytest

import aicb200
from aicb200 import AicbError, Block, GraphicsOptions, Space, SpaceRaytracer, abi, scenes
from regionfill import BOXES, box_cubes, box_slices, filled, mixed_fill
from resumeorc import LightOracle
from test_gpu_append_blocks import OPTIONS, assert_same, every_output, narrow_space, wide_blocks
from test_gpu_light import OPAQUE, compare_fields, light_scene
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit, cubes_set_opaque

pytestmark = pytest.mark.gpu

OPTS = GraphicsOptions(view_distance=60.0, lighting_display=aicb200.LIGHT_LINEAR)
QUEUED = ((0, 2, 5), (6, 8, 6), 230)   # cubes queued before the fills, across both BOXES


def with_light(space, field):
    return Space(space.lower, space.block_ids, space.blocks, light=field, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


@pytest.fixture(scope="module")
def converged_space():
    """light_scene with the oracle's converged light: a scene and an oracle created from it hold the same texels."""
    space = light_scene(seed=9)
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    return with_light(space, ol.field())


def fills(space, form):
    """Per box of BOXES: what is passed as block_ids, and the same as one id per cube."""
    for k, (lower, size) in enumerate(BOXES):
        ids = mixed_fill(space, lower, size, seed=11 + k) if form == "array" else {"opaque": 1, "air": 0, "lamp": 5}[form]
        yield lower, size, ids, np.broadcast_to(np.asarray(ids, dtype=np.uint16), size).reshape(-1)


def frames(lit, space):
    cam = scenes.standard_camera(space, OPTS, 64, 48)
    text = (aicb200 if lit.group is None else lit.group).render_layers_terminal((lit.scene, cam, OPTS))
    return {"srgb8": lit.frame(cam, OPTS), "text": text["text"], "rgba": text["rgba"]}


def assert_frames_equal(got, want, label):
    for k in got:
        assert got[k].tobytes() == want[k].tobytes(), f"{label}: {k} differs"


def fresh_frames(space):
    fresh = Lit(None, space)
    out = frames(fresh, space)
    fresh.close()
    return out


@pytest.mark.parametrize("form", ["array", "opaque", "air", "lamp"])
@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_edit_region_equals_sets_in_order_before_any_propagation(converged_space, devices, form):
    space = converged_space
    lit, ol = Lit(devices, space), LightOracle(space)
    lit.light_queue_region(*QUEUED)
    ol.queue_region(*QUEUED)
    for lower, size, ids, flat in fills(space, form):
        cubes = box_cubes(lower, size)
        differing = int((space.block_ids[box_slices(space, lower, size)].reshape(-1) != flat).sum())
        assert 0 < differing < len(flat) or form != "array"
        assert lit.light_edit_region(lower, size, ids) == differing
        ol.set_cubes(cubes, flat)
        queue, field = lit.light_download_queue(), lit.field()
        assert np.array_equal(queue, ol.queue()), np.argwhere(queue != ol.queue())[:4]
        assert np.array_equal(field, ol.field()), np.argwhere((field != ol.field()).any(axis=-1))[:4]
        opaque = sorted(cubes_set_opaque(space, cubes, flat))
        assert lit.light_changes_count() == len(opaque)
        idx, tx = lit.light_take_changes()
        assert idx.tolist() == opaque
        assert (tx == np.array([0, 0, 0, OPAQUE], dtype=np.uint8)).all()
        space = filled(space, lower, size, ids, light=field)
        assert_frames_equal(frames(lit, space), fresh_frames(space), f"{form} {lower}")
    if form == "array":
        assert (queue == 250).any() and (queue == 230).any() and (queue == 0).any()
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_edit_region_then_evaluate_equals_the_list_path(devices):
    space = light_scene(seed=9)
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    boxed, listed = Lit(devices, space), Lit(devices, space)
    for s in (boxed, listed):
        s.light_fast_evaluate()
        s.light_evaluate(0)
    for lower, size, ids, flat in fills(space, "array"):
        boxed.light_edit_region(lower, size, ids)
        assert boxed.light_evaluate(0)[0] > 0
        assert listed.light_edit_and_propagate(box_cubes(lower, size), flat, 0)[0] > 0
        ol.set_cubes(box_cubes(lower, size), flat)
        ol.evaluate(0)
        field = boxed.field()
        compare_fields(field, listed.field())
        compare_fields(field, ol.field())
        assert boxed.light_evaluate(0)[0] == 0   # quiescent
        assert not boxed.light_download_queue().any()
    boxed.close()
    listed.close()


def wide_space():
    """narrow_space with its table grown past 16384 blocks: a scene created from it has 32-bit cells."""
    space = narrow_space()
    return Space(space.lower, space.block_ids, space.blocks + wide_blocks(), light=space.light, sky_colors=space.sky_colors)


@pytest.mark.parametrize("cells", ["u16", "u32"])
@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_update_region_equals_update_cubes(devices, cells):
    space = scenes.small_mixed_scene(n=12, seed=7) if cells == "u16" else wide_space()
    n_blocks = len(space.blocks)
    if cells == "u32":
        assert n_blocks > 16384
    rng = np.random.default_rng(3)
    boxed, listed = Lit(devices, space), Lit(devices, space)
    lo = space.lower
    boxes = (((lo[0], lo[1] + 1, lo[2] + 1), (4, 5, 9)), ((lo[0] + 3, lo[1], lo[2] + 3), (space.size[0] - 3, 3, space.size[2] - 3)),
             ((lo[0] + 1, lo[1] + 2, lo[2]), (3, 2, space.size[2])), ((lo[0] + 5, lo[1] + 5, lo[2] + 2), (1, 1, 1)))
    for k, (lower, size) in enumerate(boxes):
        uniform, lit = k % 2 == 1, k < 2
        ids = int(rng.integers(1, n_blocks)) if uniform else rng.integers(max(0, n_blocks - 50), n_blocks, size).astype(np.uint16)
        light = rng.integers(0, 256, tuple(size) + (4,)).astype(np.uint8) if lit else None
        boxed.update_region(lower, size, ids, light)
        flat = np.broadcast_to(np.asarray(ids, dtype=np.uint16), size).reshape(-1)
        listed.update_cubes(box_cubes(lower, size), flat, None if light is None else light.reshape(-1, 4))
        space = filled(space, lower, size, ids)
        assert np.array_equal(boxed.field(), listed.field()), f"box {k}: texels"
        assert_frames_equal(frames(boxed, space), frames(listed, space), f"box {k}")
    if devices is None:   # every output of one context, against a scene created from the final Space
        fresh = SpaceRaytracer(with_light(space, boxed.field()), OPTIONS[0], boxed.scene.ctx)
        for opts in OPTIONS[:2]:
            cam = scenes.standard_camera(space, opts, 64, 48)
            assert_same(every_output(boxed.scene, opts, cam), every_output(fresh, opts, cam), "fresh scene")
        fresh.close()
    boxed.close()
    listed.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_update_region_leaves_the_queue_and_the_changed_cubes(converged_space, devices):
    space = converged_space
    lit = Lit(devices, space)
    lit.light_queue_region(*QUEUED)
    queue, changed = lit.light_download_queue(), lit.light_changes_count()
    lower, size = BOXES[0]
    texels = np.full(tuple(size) + (4,), 77, dtype=np.uint8)
    lit.update_region(lower, size, mixed_fill(space, lower, size, seed=4), texels)
    assert np.array_equal(lit.light_download_queue(), queue) and lit.light_changes_count() == changed
    assert (lit.field()[box_slices(space, lower, size)] == 77).all()
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_whole_bounds_box_writes_the_cells_of_fill_uniform(converged_space, devices):
    """Mutation::fill_uniform takes one of two branches (space.rs:1455-1479).  Over the whole bounds it replaces the
    palette and queues every cube at 210 (fill_uniform + light_queue_region here); over a smaller region it is
    Mutation::fill.  A box call over the whole bounds is the second branch: the same cells, but a queue that holds 250
    for the changed cubes and their neighbours only, by the reference's own difference between the branches."""
    space = converged_space
    boxed, every = Lit(devices, space), Lit(devices, space)
    n = boxed.light_edit_region(space.lower, space.size, 0)
    assert n == int((space.block_ids != 0).sum())
    every.fill_uniform(Block.air())
    every.light_queue_region(space.lower, space.size, 210)
    cam = scenes.standard_camera(space, OPTS, 64, 48)
    flat = GraphicsOptions(view_distance=60.0, lighting_display=aicb200.LIGHT_NONE)   # the texels differ: OPAQUE stays
    assert np.array_equal(boxed.frame(cam, flat), every.frame(cam, flat))
    queue = boxed.light_download_queue()
    assert set(np.unique(queue).tolist()) == {0, 250} and (every.light_download_queue() == 210).all()
    ol = LightOracle(space)
    ol.set_cubes(box_cubes(space.lower, space.size), np.zeros(space.block_ids.size, dtype=np.uint16))
    assert np.array_equal(queue, ol.queue()) and np.array_equal(boxed.field(), ol.field())
    boxed.close()
    every.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_rejected_box_calls_change_nothing(converged_space, devices):
    space = converged_space
    lit = Lit(devices, space)
    lit.light_queue_region(*QUEUED)
    field, queue, changed, frame = lit.field(), lit.light_download_queue(), lit.light_changes_count(), frames(lit, space)
    lower, size = BOXES[0]
    ids = mixed_fill(space, lower, size, seed=2)
    past = ids.copy()
    past[-1, -1, -1] = len(space.blocks)
    outside = (lower[0] - 1, lower[1], lower[2])
    beyond = (size[0], size[1], space.size[2] + 1)
    for call in (lit.light_edit_region, lit.update_region):
        for args in ((outside, size, ids), (lower, beyond, 1), (lower, size, past), (lower, size, len(space.blocks))):
            with pytest.raises(AicbError) as e:
                call(*args)
            assert e.value.status == abi.ERR_INVALID
        with pytest.raises(ValueError):
            call(lower, size, ids[:-1])
        with pytest.raises(ValueError):
            call(lower, size, ids.reshape(-1))
    with pytest.raises(ValueError):
        lit.update_region(lower, size, ids, np.zeros(tuple(size) + (3,), dtype=np.uint8))
    n = C.c_size_t(5)
    assert lit._fn("light_edit_region")(lit.handle, None, None, 1, C.byref(n)) == abi.ERR_INVALID
    assert lit._fn("scene_update_region")(lit.handle, None, None, 1, None) == abi.ERR_INVALID
    assert lit._fn("light_edit_region")(None, None, None, 1, None) == abi.ERR_INVALID
    # a region of volume 0 is accepted and does nothing
    assert lit.light_edit_region(lower, (size[0], 0, size[2]), 1) == 0
    lit.update_region(lower, (0, size[1], size[2]), 1)
    assert np.array_equal(lit.field(), field) and np.array_equal(lit.light_download_queue(), queue)
    assert lit.light_changes_count() == changed
    assert_frames_equal(frames(lit, space), frame, "after the rejected calls")
    lit.close()
    unlit = Lit(devices, Space(space.lower, space.block_ids, space.blocks, sky_colors=space.sky_colors, light_max_distance=0))
    before = frames(unlit, space)
    with pytest.raises(AicbError) as e:
        unlit.light_edit_region(lower, size, ids)
    assert e.value.status == abi.ERR_INVALID
    assert_frames_equal(frames(unlit, space), before, "LightPhysics::None")
    unlit.close()
