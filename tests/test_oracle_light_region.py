"""Mutation::fill over a box leaves the same light queue and texels in whatever order its cubes are set: the oracle's
Mutation::set (modified_cube_needs_update, space/light/updater.rs:135-173) over a box in interior_iter order, in reverse
and shuffled.  aicb_light_edit_region relies on this to apply the rule to every cube of the box at once."""
import numpy as np
import pytest

from aicb200 import Space
from regionfill import BOXES, box_cubes, mixed_fill
from resumeorc import LightOracle
from test_gpu_light import light_scene


@pytest.fixture(scope="module")
def converged():
    """light_scene with its converged light."""
    space = light_scene(seed=9)
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    return Space(space.lower, space.block_ids, space.blocks, light=ol.field(), sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


def after_sets(space, cubes, ids, order):
    ol = LightOracle(space)
    ol.queue_region((0, 2, 5), (6, 8, 6), 230)
    ol.set_cubes(cubes[order], ids[order])
    return ol.queue(), ol.field()


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("box", BOXES + (((-2, 1, 3), (14, 14, 14)),), ids=["low_x", "high_xz", "bounds"])
def test_the_order_of_a_box_of_sets_does_not_matter(converged, box, seed):
    lower, size = box
    cubes = box_cubes(lower, size)
    ids = mixed_fill(converged, lower, size, seed).reshape(-1)
    n = len(cubes)
    queue, field = after_sets(converged, cubes, ids, np.arange(n))
    assert (queue == 250).any() and (queue == 230).any() and (field[..., 3] == 128).any()
    for name, order in (("reverse", np.arange(n)[::-1]), ("shuffled", np.random.default_rng(seed).permutation(n))):
        q, f = after_sets(converged, cubes, ids, order)
        assert np.array_equal(q, queue), f"{name}: the queue differs at {np.argwhere(q != queue)[:4]}"
        assert np.array_equal(f, field), f"{name}: the field differs"


@pytest.mark.parametrize("uniform", [0, 1, 5], ids=["air", "opaque", "lamp"])
def test_the_order_of_a_uniform_fill_does_not_matter(converged, uniform):
    lower, size = BOXES[1]
    cubes = box_cubes(lower, size)
    ids = np.full(len(cubes), uniform, dtype=np.uint16)
    queue, field = after_sets(converged, cubes, ids, np.arange(len(cubes)))
    q, f = after_sets(converged, cubes, ids, np.random.default_rng(7).permutation(len(cubes)))
    assert np.array_equal(q, queue) and np.array_equal(f, field)
