"""The light update queue across save and load, on the CPU: the light oracle's restatement of Space::new_from_builder's
load rule (space.rs:290-313) and of light_needs_update_in_region (space/light/updater.rs:122-133), and
ingest.light_to_value, the save form of Serialize for space::Read (save/conversion.rs:773-785).  Pinned on the
reference's own tests: space_light_queue_remembered (save/tests.rs:819-854), fill_uniform_entire_space
(space/tests.rs:411-434) and space_success (save/tests.rs:653-746)."""
import numpy as np
import pytest

from aicb200 import Block, Space, ingest
from resumeorc import LightOracle
from test_ingest import space_success_json

OPAQUE, NO_RAYS, UNINIT, VISIBLE = 128, 1, 0, 255
GREY = Block(color=(0.5, 0.5, 0.5, 1.0))


def row_3x1x1(light):
    """save/tests.rs:822-828: a 3x1x1 Space, block0 (opaque) at [0, 0, 0], LightPhysics::DEFAULT (Rays, 30)."""
    ids = np.array([1, 0, 0], dtype=np.uint16).reshape(3, 1, 1)
    return Space((0, 0, 0), ids, [Block.air(), GREY], light=light, light_max_distance=30)


def space_success(light=None):
    """save/tests.rs:657-672: bounds [1, 2, 3] .. [4, 5, 6], Sky::Uniform(Rgb::ONE), Rays { 123 }, all AIR."""
    ids = np.zeros((3, 3, 3), dtype=np.uint16)
    return Space((1, 2, 3), ids, [Block.air(), GREY], light=light, sky_colors=[(1.0, 1.0, 1.0)], light_max_distance=123)


def test_light_queue_remembered():
    # Before saving: m.set([0, 0, 0], block0) leaves [1, 0, 0] queued and [0, 0, 0] updated (save/tests.rs:829-836)
    ol = LightOracle(Space((0, 0, 0), np.zeros((3, 1, 1), np.uint16), [Block.air(), GREY], light_max_distance=30))
    ol.set_cubes([(0, 0, 0)], [1])
    assert list(ol.field()[:, 0, 0, 3]) == [OPAQUE, NO_RAYS, NO_RAYS]
    assert list(ol.queue()[:, 0, 0]) == [0, 250, 0]
    # Saving marks the queued cubes Uninitialized (LightSerV1 status 0; Opaque 2, NoRays 1)
    value = ingest.light_to_value(ol.field(), ol.queue())
    assert list(np.frombuffer(ingest.gz_decode(value), np.uint8).reshape(3, 4)[:, 3]) == [2, 0, 1]
    saved = ingest.light_from_value(value, (3, 1, 1))
    assert list(saved[:, 0, 0, 3]) == [OPAQUE, UNINIT, NO_RAYS]
    # Loading queues them at Priority::UNINIT, and one step updates them (save/tests.rs:846-853)
    loaded = LightOracle(row_3x1x1(saved))
    assert loaded.queue_len() == 0
    assert loaded.queue_uninitialized() == 1
    assert list(loaded.queue()[:, 0, 0]) == [0, 210, 0]
    loaded.evaluate(0)
    assert list(loaded.field()[:, 0, 0, 3]) == [OPAQUE, VISIBLE, NO_RAYS]
    assert loaded.queue_len() == 0


def test_queue_uninitialized_raises_and_never_lowers():
    light = np.zeros((3, 1, 1, 4), dtype=np.uint8)            # all Uninitialized
    ol = LightOracle(row_3x1x1(light))
    ol.queue_region((0, 0, 0), (1, 1, 1), 250)
    ol.queue_region((1, 0, 0), (1, 1, 1), 200)
    assert ol.queue_uninitialized() == 3
    assert list(ol.queue()[:, 0, 0]) == [250, 210, 210]


def test_no_light_physics_queues_nothing():
    space = row_3x1x1(np.zeros((3, 1, 1, 4), dtype=np.uint8))
    space.light_max_distance = 0
    ol = LightOracle(space)
    assert ol.queue_uninitialized() == 0
    ol.queue_region((0, 0, 0), (3, 1, 1), 210)
    assert ol.queue_len() == 0


def fill_uniform_space():
    """space/tests.rs:413-423: fill_uniform(bounds, block) over [0, 3, 0] + [400, 16, 2]."""
    ids = np.ones((400, 16, 2), dtype=np.uint16)
    return Space((0, 3, 0), ids, [Block.air(), GREY], light_max_distance=30)


def test_queue_region_of_the_whole_space():
    """fill_uniform_entire_space: every cube ends in the queue (light_needs_update_in_region(bounds, UNINIT))."""
    ol = LightOracle(fill_uniform_space())
    ol.queue_region((0, 3, 0), (400, 16, 2), 210)
    q = ol.queue()
    assert q.shape == (400, 16, 2) and (q == 210).all()
    assert ol.queue_len() == 400 * 16 * 2


def test_queue_region_is_clipped_and_raise_only():
    ol = LightOracle(fill_uniform_space())
    ol.queue_region((-5, 0, 1), (10, 10, 10), 230)            # x 0..5, y 3..10, z 1..2 of the Space
    want = np.zeros((400, 16, 2), dtype=np.uint8)
    want[0:5, 0:7, 1:2] = 230
    assert np.array_equal(ol.queue(), want)
    ol.queue_region((0, 3, 0), (400, 16, 2), 210)             # raises the rest, keeps the 230s
    want[want == 0] = 210
    assert np.array_equal(ol.queue(), want)
    ol.queue_region((390, 3, 0), (100, 100, 100), 7)          # never lowers
    assert np.array_equal(ol.queue(), want)
    ol.queue_region((1000, 0, 0), (5, 5, 5), 250)             # an empty intersection does nothing
    assert np.array_equal(ol.queue(), want)
    with pytest.raises(ValueError):
        ol.queue_region((0, 3, 0), (1, 1, 1), 0)              # Priority::MIN never enters the queue
    assert np.array_equal(ol.queue(), want)


def space_success_field():
    """save/tests.rs:667-671: m.set([1, 2, 5], block); m.evaluate_light(0)."""
    ol = LightOracle(space_success())
    ol.set_cubes([(1, 2, 5)], [1])
    ol.evaluate(0)
    assert ol.queue_len() == 0
    return ol.field()


def test_light_to_value_gives_the_reference_bytes():
    want = ingest.gz_decode(space_success_json()["light"])    # save/tests.rs:735-739
    field = space_success_field()
    assert ingest.gz_decode(ingest.light_to_value(field)) == want
    assert ingest.gz_decode(ingest.light_to_value(field, np.zeros((3, 3, 3), np.uint8))) == want


def test_light_to_value_marks_queued_cubes_and_round_trips():
    field = space_success_field()
    queue = np.zeros((3, 3, 3), dtype=np.uint8)
    queue[0, 0, 1] = 250                                      # a Visible cube
    queue[0, 0, 2] = 1                                        # the Opaque one
    queue[2, 2, 2] = 210                                      # a NoRays cube
    value = ingest.light_to_value(field, queue)
    raw = np.frombuffer(ingest.gz_decode(value), np.uint8).reshape(3, 3, 3, 4)
    assert (raw[queue > 0, 3] == 0).all()
    assert np.array_equal(raw[..., :3], field[..., :3])      # r, g, b are kept
    v = space_success_json()
    v["light"] = value
    loaded = ingest.space_from_value(v)
    want = field.copy()
    want[queue > 0, 3] = UNINIT
    assert np.array_equal(loaded.light, want)
    assert np.array_equal(ingest.light_from_value(value, (3, 3, 3)), want)
    # and the loaded Space resumes exactly the three queued cubes
    ol = LightOracle(loaded)
    assert ol.queue_uninitialized() == 3
    assert np.array_equal(ol.queue() > 0, queue > 0)


def test_light_to_value_rejects_what_lightserv1_cannot_hold():
    field = space_success_field()
    field[0, 0, 0, 3] = 7
    with pytest.raises(ValueError):
        ingest.light_to_value(field)
    with pytest.raises(ValueError):
        ingest.light_to_value(space_success_field(), np.zeros(5, np.uint8))
