"""aicb_light_edit_cubes' rule, restated in numpy (editlists.edit_cubes_rule), leaves byte for byte the queue, texels and
set of changed cubes of the oracle's Mutation::set applied entry by entry (orc_light_set_cubes): on lists with heavy
duplication, A -> B -> A and B -> A -> B chains, neighbouring cubes, cubes on the bounds and every kind of block, over
a queue seeded beforehand so that cancellations show."""
import numpy as np
import pytest

from aicb200 import Space
from editlists import NEWLY_VISIBLE, edit_cubes_rule, edit_list
from resumeorc import LightOracle
from test_gpu_light import light_scene
from test_gpu_light_changes import cubes_set_opaque, opaque_for_light

QUEUED = 230


@pytest.fixture(scope="module")
def converged():
    """An 8^3 light_scene with its converged light."""
    space = light_scene(n=8, seed=4, lower=(-3, 2, 1))
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    return Space(space.lower, space.block_ids, space.blocks, light=ol.field(), sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


def seeded_oracle(space):
    ol = LightOracle(space)
    ol.queue_region(space.lower, space.size, QUEUED)
    return ol


@pytest.mark.parametrize("seed", range(24))
def test_rule_equals_sets_in_order(converged, seed):
    space = converged
    cubes, ids = edit_list(space, seed)
    ol = seeded_oracle(space)
    n, final, queue, field, changed = edit_cubes_rule(space, ol.queue(), ol.field(), cubes, ids)
    ol.set_cubes(cubes, ids)
    assert np.array_equal(queue, ol.queue()), np.argwhere(queue != ol.queue())[:4]
    assert np.array_equal(field, ol.field()), np.argwhere((field != ol.field()).any(axis=-1))[:4]
    assert changed == sorted(cubes_set_opaque(space, cubes, ids))
    assert 0 < n < len(ids)   # the lists hold both changing and same-block entries
    assert (queue == NEWLY_VISIBLE).any() and (queue == QUEUED).any() and (queue == 0).any()


def test_a_cube_set_opaque_and_back_keeps_its_opaque_texel(converged):
    """After air -> opaque -> air the cube holds air with an OPAQUE texel, queued at NEWLY_VISIBLE, and is in the set:
    the texels are not a function of the final cells."""
    space = converged
    at = tuple(int(v) for v in np.argwhere(space.block_ids == 0)[0])
    opaque = next(i for i, b in enumerate(space.blocks) if opaque_for_light(b))
    cube = np.array(space.lower) + at
    cubes, ids = np.array([cube, cube], dtype=np.int32), np.array([opaque, 0], dtype=np.uint16)
    ol = seeded_oracle(space)
    n, final, queue, field, changed = edit_cubes_rule(space, ol.queue(), ol.field(), cubes, ids)
    ol.set_cubes(cubes, ids)
    assert n == 2 and final[at] == 0
    assert tuple(field[at]) == (0, 0, 0, 128) and queue[at] == NEWLY_VISIBLE
    assert changed == [int(np.ravel_multi_index(at, space.size))]
    assert np.array_equal(queue, ol.queue()) and np.array_equal(field, ol.field())


def test_same_block_entries_change_nothing(converged):
    space = converged
    ol = seeded_oracle(space)
    queue, field = ol.queue(), ol.field()
    cubes, _ = edit_list(space, 3)
    ids = np.array([space.block_ids[tuple(c - np.array(space.lower))] for c in cubes], dtype=np.uint16)
    n, final, q, f, changed = edit_cubes_rule(space, queue, field, cubes, ids)
    ol.set_cubes(cubes, ids)
    assert n == 0 and not changed and np.array_equal(final, space.block_ids)
    assert np.array_equal(q, queue) and np.array_equal(q, ol.queue()) and np.array_equal(f, ol.field())
