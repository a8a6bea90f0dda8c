"""A light step with a count budget on the oracle behaves as LightStorage::update_light_from_queue
(space/light/updater.rs:180-290): it makes min(budget, what the queue offers) updates, reports the queue it leaves, does
nothing with a zero budget, and steps repeated until the queue is done reach evaluate_light's field.  The GPU's
aicb_light_update_from_queue is held to the same contract (tests/test_gpu_light_step.py)."""
import numpy as np
import pytest

from aicb200 import Space, scenes
from regionfill import BOXES, box_cubes, mixed_fill
from steporc import LightOracle
from test_gpu_light import light_scene


def with_light(space, light):
    return Space(space.lower, space.block_ids, space.blocks, light=light, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


def fast_evaluated():
    """light_scene after fast_evaluate_light: its queue holds every visible cube at Priority::ESTIMATED."""
    ol = LightOracle(light_scene(seed=9))
    ol.fast_evaluate()
    return ol


def converged_then_filled():
    """light_scene converged, then a box filled with a mix of blocks: a queue of several priorities."""
    space = light_scene(seed=9)
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    lower, size = BOXES[0]
    ol = LightOracle(with_light(space, ol.field()))
    ol.set_cubes(box_cubes(lower, size), mixed_fill(space, lower, size, 2).reshape(-1))
    return ol


def resumed():
    """C4 at 24^3 after fast_evaluate_light with 15 % of its texels saved Uninitialized, its queue resumed."""
    space = scenes.config_c4(n=24)
    ol = LightOracle(space)
    ol.fast_evaluate()
    field = ol.field()
    field[np.random.default_rng(3).random(space.size) < 0.15, 3] = 0
    ol = LightOracle(with_light(space, field))
    assert ol.queue_uninitialized() > 0
    return ol


MAKERS = {"fast_evaluated": fast_evaluated, "filled": converged_then_filled, "resumed": resumed}


def assert_info_matches_queue(info, ol):
    q = ol.queue()
    assert info["queue_count"] == int((q > 0).sum())
    assert info["max_queue_priority"] == int(q.max())
    assert not (q == 1).any(), "a priority-1 entry: evaluate(0) would leave it, a step would not"


@pytest.mark.parametrize("make", MAKERS.values(), ids=MAKERS.keys())
def test_update_count_is_the_budget_or_what_the_queue_offered(make):
    available = make().evaluate(0)[0]
    assert available > 0
    for budget in (1, 37, available - 1, available, available + 1, 2**62):
        ol = make()
        info = ol.step(budget)
        assert info["update_count"] == min(budget, available), budget
        assert_info_matches_queue(info, ol)
        if budget >= available:
            assert info["queue_count"] == 0 and info["max_queue_priority"] == 0


@pytest.mark.parametrize("make", MAKERS.values(), ids=MAKERS.keys())
def test_zero_budget_changes_nothing(make):
    ol = make()
    field, queue = ol.field(), ol.queue()
    info = ol.step(0)
    assert info["update_count"] == 0 and info["max_update_difference"] == 0
    assert info["queue_count"] > 0 and info["max_queue_priority"] == int(queue.max())
    assert_info_matches_queue(info, ol)
    assert np.array_equal(ol.field(), field) and np.array_equal(ol.queue(), queue)


@pytest.mark.parametrize("budget", [50, 613])
@pytest.mark.parametrize("make", MAKERS.values(), ids=MAKERS.keys())
def test_repeated_steps_reach_evaluates_field(make, budget):
    """The oracle pops one cube at a time, so steps split its evaluate_light at the budget: the same updates in the same
    order, and the same field."""
    whole = make()
    total = whole.evaluate(0)[0]
    ol = make()
    done, steps = 0, 0
    while True:
        info = ol.step(budget)
        done += info["update_count"]
        steps += 1
        assert_info_matches_queue(info, ol)
        if info["max_queue_priority"] <= 1:
            break
        assert info["update_count"] == budget
    assert done == total and steps == -(-total // budget)
    assert np.array_equal(ol.field(), whole.field())
    assert ol.queue_len() == 0
