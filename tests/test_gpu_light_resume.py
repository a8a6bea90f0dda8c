"""The light update queue across save and load on the GPU (aicb_light_queue_uninitialized, aicb_light_queue_region,
aicb_light_download_queue and their group forms): the load rule of Space::new_from_builder (space.rs:290-313),
light_needs_update_in_region (space/light/updater.rs:122-133) and the save form of Serialize for space::Read
(save/conversion.rs:773-785).  The queue equals the oracle's (oracle_light/, tests/resumeorc.py) bit for bit in every
state reached without a relaxation round; a Space saved with its queue and loaded again resumes the saved work and
meets the light contract (tests/test_gpu_light.py: compare_fields) against the oracle resumed from the same save.
Every check runs on one context and on groups of 1, 2 and 3 contexts of one device."""
import ctypes as C

import numpy as np
import pytest

import aicb200
from aicb200 import AicbError, GraphicsOptions, Space, abi, ingest, scenes
from resumeorc import LightOracle
from test_gpu_light import compare_fields
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit
from test_ingest import space_success_json
from test_oracle_light_resume import OPAQUE, NO_RAYS, VISIBLE, fill_uniform_space, row_3x1x1, space_success

pytestmark = pytest.mark.gpu

OPTS = GraphicsOptions(lighting_display=aicb200.LIGHT_LINEAR, fog=aicb200.FOG_ABRUPT)


def abi_queue_calls(lit):
    return (lit.scene._fn("light_queue_uninitialized"), lit.scene._fn("light_queue_region"),
            lit.scene._fn("light_download_queue"))


def download_queue_counted(lit):
    """The queue through the C ABI, with its n_queued output."""
    _, _, download = abi_queue_calls(lit)
    out = np.zeros(lit.space.size, dtype=np.uint8)
    n = C.c_size_t(12345)
    assert download(lit.scene.handle, out.ctypes.data, out.size, C.byref(n)) == abi.OK
    assert n.value == int((out > 0).sum())
    return out


def with_light(space, light, block_ids=None):
    return Space(space.lower, space.block_ids if block_ids is None else block_ids, space.blocks, light=light,
                 sky_colors=space.sky_colors, light_max_distance=space.light_max_distance)


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_light_queue_remembered(devices):
    """save/tests.rs:819-854: the saved statuses [Opaque, Uninitialized, NoRays] step to [Opaque, Visible, NoRays]."""
    saved = np.zeros((3, 1, 1, 4), dtype=np.uint8)
    saved[0, 0, 0, 3], saved[2, 0, 0, 3] = OPAQUE, NO_RAYS
    lit = Lit(devices, row_3x1x1(saved))
    assert lit.light_queue_uninitialized() == 1
    assert list(download_queue_counted(lit)[:, 0, 0]) == [0, 210, 0]
    assert np.array_equal(lit.field(), saved)            # no texel written
    assert lit.light_changes_count() == 0
    assert lit.light_evaluate(0)[0] == 1
    assert list(lit.field()[:, 0, 0, 3]) == [OPAQUE, VISIBLE, NO_RAYS]
    assert not lit.light_download_queue().any()
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_queue_region_known_answers(devices):
    """fill_uniform_entire_space (space/tests.rs:411-434): every cube queued at UNINIT; clipped, raise-only, as the
    oracle."""
    space = fill_uniform_space()
    lit, ol = Lit(devices, space), LightOracle(space)
    for lower, size, prio in (((-5, 0, 1), (10, 10, 10), 230), ((0, 3, 0), (400, 16, 2), 210),
                              ((390, 3, 0), (100, 100, 100), 7), ((1000, 0, 0), (5, 5, 5), 250),
                              ((17, 9, 0), (1, 1, 1), 255)):
        lit.light_queue_region(lower, size, prio)
        ol.queue_region(lower, size, prio)
        assert np.array_equal(download_queue_counted(lit), ol.queue()), (lower, size, prio)
    q = lit.light_download_queue()
    assert (q > 0).all() and (q == 210).sum() == 400 * 16 * 2 - 5 * 7 * 1 - 1
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_space_success_saves_the_reference_bytes(devices):
    """save/tests.rs:653-746: m.set([1, 2, 5], block); evaluate_light(0); the saved light is the reference's."""
    lit = Lit(devices, space_success())
    lit.light_edit_and_propagate([(1, 2, 5)], [1], 0)
    queue = download_queue_counted(lit)
    assert not queue.any()
    value = ingest.light_to_value(lit.field(), queue)
    assert ingest.gz_decode(value) == ingest.gz_decode(space_success_json()["light"])
    lit.close()


def c4_with_uninitialized(n=32, frac=0.15, seed=3):
    """C4 at n^3 after fast_evaluate_light, then a random subset of the texels marked Uninitialized (r, g, b kept)."""
    space = scenes.config_c4(n=n)
    ol = LightOracle(space)
    ol.fast_evaluate()
    field = ol.field()
    rng = np.random.default_rng(seed)
    field[rng.random(space.size) < frac, 3] = 0
    return with_light(space, field)


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_queue_equals_the_oracle_bit_for_bit(devices):
    space = c4_with_uninitialized()
    n_uninit = int((space.light[..., 3] == 0).sum())
    lit, ol = Lit(devices, space), LightOracle(space)
    assert not download_queue_counted(lit).any()         # aicb_scene_create leaves the queue empty
    steps = [
        ("region 230", lambda o: o.light_queue_region((3, 5, 7), (9, 20, 4), 230) if o is lit
         else o.queue_region((3, 5, 7), (9, 20, 4), 230)),
        ("region 200", lambda o: o.light_queue_region((-4, 10, 0), (12, 3, 40), 200) if o is lit
         else o.queue_region((-4, 10, 0), (12, 3, 40), 200)),
        ("uninitialized", None),
        ("uninitialized again", None),
        ("region 250 inside", lambda o: o.light_queue_region((20, 20, 20), (2, 2, 2), 250) if o is lit
         else o.queue_region((20, 20, 20), (2, 2, 2), 250)),
    ]
    for name, step in steps:
        if step is None:
            assert lit.light_queue_uninitialized() == n_uninit == ol.queue_uninitialized(), name
        else:
            step(lit)
            step(ol)
        assert np.array_equal(download_queue_counted(lit), ol.queue()), name
        assert np.array_equal(lit.field(), space.light), name
    # fast_evaluate_light replaces the queue (and the field)
    lit.light_fast_evaluate()
    ol.fast_evaluate()
    assert np.array_equal(download_queue_counted(lit), ol.queue())
    assert np.array_equal(lit.field(), ol.field())
    lit.close()


def apply_edits(space, cubes, ids):
    block_ids = space.block_ids.copy()
    for c, i in zip(cubes, ids):
        block_ids[tuple(np.asarray(c) - np.asarray(space.lower))] = i
    return block_ids


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_saved_and_loaded_space_resumes_its_queue(devices):
    space = scenes.config_c4(n=32)
    a = Lit(devices, space)
    a.light_fast_evaluate()
    a.light_evaluate(1)
    cubes, ids = scenes.c4_edits(space, 40, 0)
    a.light_edit_and_propagate(cubes, ids, 32)
    field, queue = a.field(), download_queue_counted(a)
    assert queue.any()                                   # work left for the load to resume
    a.close()
    saved = ingest.light_from_value(ingest.light_to_value(field, queue), space.size)
    loaded = with_light(space, saved, apply_edits(space, cubes, ids))
    want = (queue > 0) | (field[..., 3] == 0)
    b = Lit(devices, loaded)
    assert b.light_queue_uninitialized() == int(want.sum())
    assert np.array_equal(download_queue_counted(b), np.where(want, 210, 0).astype(np.uint8))
    resumed, _, _ = b.light_evaluate(0)
    ol = LightOracle(loaded)
    assert ol.queue_uninitialized() == int(want.sum())
    ol.evaluate(0)
    compare_fields(b.field(), ol.field())
    assert not b.light_download_queue().any()
    b.close()
    # today's load: fast_evaluate + evaluate(0) throws the saved field away and does more work
    c = Lit(devices, loaded)
    c.light_fast_evaluate()
    again, _, _ = c.light_evaluate(0)
    assert 0 < resumed < again
    c.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_queue_calls_have_no_side_effects(devices):
    space = c4_with_uninitialized(n=24)
    lit = Lit(devices, space)
    assert lit.light_evaluate(0)[0] == 0                 # (the queue is empty) the light state exists from here on
    cam = scenes.standard_camera(space, OPTS, 64, 48)
    field, frame = lit.field(), lit.frame(cam, OPTS)
    bytes_before = lit.device_bytes if devices is None else None
    lit.light_queue_region((0, 0, 0), (5, 5, 5), 240)
    lit.light_queue_uninitialized()
    download_queue_counted(lit)
    assert np.array_equal(lit.field(), field)
    assert lit.light_changes_count() == 0
    assert np.array_equal(lit.frame(cam, OPTS), frame)
    if devices is None:
        assert lit.device_bytes == bytes_before
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_scene_without_a_light_volume_queues_nothing(devices):
    space = c4_with_uninitialized(n=16)
    lit = Lit(devices, with_light(space, None))
    assert lit.light_queue_uninitialized() == 0
    assert not download_queue_counted(lit).any()
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_rejected_calls_change_nothing(devices):
    space = c4_with_uninitialized(n=16)
    lit = Lit(devices, space)
    lit.light_queue_region((0, 0, 0), (4, 4, 4), 220)
    queue, field = lit.light_download_queue(), lit.field()
    uninit, region, download = abi_queue_calls(lit)
    h = lit.scene.handle
    box = abi.Aab()
    box.lower[:] = [0, 0, 0]
    box.size[:] = [16, 16, 16]
    out = np.zeros(space.size, dtype=np.uint8)
    assert region(h, None, 210) == abi.ERR_INVALID
    assert region(h, C.byref(box), 0) == abi.ERR_INVALID
    assert download(h, None, out.size, None) == abi.ERR_INVALID
    assert download(h, out.ctypes.data, out.size - 1, None) == abi.ERR_INVALID
    assert download(h, out.ctypes.data, out.size + 1, None) == abi.ERR_INVALID
    assert uninit(None, None) == region(None, C.byref(box), 210) == download(None, out.ctypes.data, out.size, None) \
        == abi.ERR_INVALID
    assert np.array_equal(lit.light_download_queue(), queue)
    assert np.array_equal(lit.field(), field)
    assert lit.light_changes_count() == 0
    lit.close()
    # LightPhysics::None
    unlit = Lit(devices, Space(space.lower, space.block_ids, space.blocks, sky_colors=space.sky_colors,
                               light_max_distance=0))
    for call in (unlit.light_queue_uninitialized, lambda: unlit.light_queue_region((0, 0, 0), (16, 16, 16), 210),
                 unlit.light_download_queue):
        with pytest.raises(AicbError) as e:
            call()
        assert e.value.status == abi.ERR_INVALID
    unlit.close()
