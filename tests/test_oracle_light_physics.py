"""The light oracle's side of SpaceChange::Physics (oracle_light/: orc_light_set_physics), on the CPU: a restatement of
LightStorage::maybe_reinitialize_for_physics_change (space/light/updater.rs:80-113).  A new LightPhysics reinitialises
the light, so it must give exactly what a fresh oracle over the Space with the new physics gives after fast_evaluate;
a new sky alone, or an unchanged physics, leaves the field and the queue as they were."""
import numpy as np
import pytest

from aicb200 import Space, scenes
from physicsorc import LightOracle
from test_gpu_light import light_scene

UNIFORM_SKY = [(0.4, 0.5, 0.9)]
OCTANT_SKY = scenes.OCTANT_SKY


def with_physics(space, sky_colors, light_max_distance):
    return Space(space.lower, space.block_ids, space.blocks, light=space.light, sky_colors=sky_colors,
                 light_max_distance=light_max_distance)


def partly_converged(space):
    """An oracle with light in flight: fast_evaluate, then a few hundred updates, the queue not yet empty."""
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0, max_updates=300)
    assert ol.queue_len() > 0
    return ol


# (sky of the Space, new sky, new distance); light_scene's distance is 12
CHANGES = {
    "distance": (OCTANT_SKY, OCTANT_SKY, 6),
    "octants_to_uniform_and_distance": (OCTANT_SKY, UNIFORM_SKY, 6),
    "uniform_to_octants_and_distance": (UNIFORM_SKY, OCTANT_SKY, 20),
    "none_to_rays": (OCTANT_SKY, UNIFORM_SKY, 12),
}


@pytest.mark.parametrize("name", sorted(CHANGES))
def test_new_light_physics_equals_a_fresh_fast_evaluate(name):
    old_sky, new_sky, distance = CHANGES[name]
    space = with_physics(light_scene(seed=9), old_sky, 0 if name == "none_to_rays" else 12)
    ol = LightOracle(space)
    if space.light_max_distance:
        ol = partly_converged(space)
    ol.set_physics(new_sky, distance)
    fresh = LightOracle(with_physics(space, new_sky, distance))
    fresh.fast_evaluate()
    assert np.array_equal(ol.field(), fresh.field())
    assert ol.queue_len() == fresh.queue_len() > 0
    # and the two go on alike
    assert ol.evaluate(0) == fresh.evaluate(0)
    assert np.array_equal(ol.field(), fresh.field())


def test_unchanged_physics_is_a_no_op():
    space = light_scene(seed=9)
    ol = partly_converged(space)
    field, queued = ol.field(), ol.queue_len()
    ol.set_physics(space.sky_colors, space.light_max_distance)
    assert np.array_equal(ol.field(), field)
    assert ol.queue_len() == queued


@pytest.mark.parametrize("new_sky", [UNIFORM_SKY, [(c[2], c[0], c[1]) for c in OCTANT_SKY]], ids=["uniform", "octants"])
def test_new_sky_alone_leaves_the_light_and_the_queue(new_sky):
    space = light_scene(seed=9)
    ol = partly_converged(space)
    field, queued = ol.field(), ol.queue_len()
    ol.set_physics(new_sky, space.light_max_distance)
    assert np.array_equal(ol.field(), field)
    assert ol.queue_len() == queued
    # the new BlockSky is the one light reads from then on
    ol.fast_evaluate()
    fresh = LightOracle(with_physics(space, new_sky, space.light_max_distance))
    fresh.fast_evaluate()
    assert np.array_equal(ol.field(), fresh.field())


def test_none_empties_the_light_and_rays_come_back():
    space = light_scene(seed=9)
    ol = partly_converged(space)
    ol.set_physics(space.sky_colors, 0)
    assert ol.queue_len() == 0
    assert ol.evaluate(0) == (0, 0)
    ol.set_physics(space.sky_colors, 12)
    fresh = LightOracle(space)
    fresh.fast_evaluate()
    assert np.array_equal(ol.field(), fresh.field())
    assert ol.queue_len() == fresh.queue_len()
