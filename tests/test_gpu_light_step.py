"""The light step of a tick (aicb_light_update_from_queue and its group form): LightStorage::update_light_from_queue
(space/light/updater.rs:180-290) with a budget of cube updates, reporting LightUpdatesInfo (updater.rs:970-984).  A
round that does not fit in the budget takes the top of the queue by (priority, then lowest index); a round that fits is
aicb_light_evaluate's.  Every check runs on one context and on groups of 1, 2 and 3 contexts of one device."""
import ctypes as C

import numpy as np
import pytest

from aicb200 import AicbError, Space, abi
from regionfill import BOXES, mixed_fill
from steporc import LightOracle
from test_gpu_light import compare_fields, light_scene
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit
from test_gpu_light_resume import c4_with_uninitialized

pytestmark = pytest.mark.gpu

# a second queued region, away from the filled box, at a priority below NEWLY_VISIBLE (250)
EXTRA_REGION = ((5, 1, 3), (6, 8, 6), 240)


def with_light(space, light):
    return Space(space.lower, space.block_ids, space.blocks, light=light, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


@pytest.fixture(scope="module")
def converged():
    """light_scene with the light the GPU converges it to: no Uninitialized texel and an empty queue."""
    space = light_scene(seed=9)
    lit = Lit(None, space)
    lit.light_fast_evaluate()
    lit.light_evaluate(0)
    field = lit.field()
    assert not lit.light_download_queue().any()
    lit.close()
    assert (field[..., 3] != 0).all()
    return with_light(space, field)


def edited(devices, space):
    """The converged scene with a box filled (queued at 250 with its neighbours) and EXTRA_REGION queued at 240: no
    Uninitialized texel and no priority-1 entry, so a round's result does not depend on the order of its cubes."""
    lit = Lit(devices, space)
    lower, size = BOXES[0]
    assert lit.light_edit_region(lower, size, mixed_fill(space, lower, size, 2)) > 0
    lit.light_queue_region(*EXTRA_REGION)
    return lit


def difference_priority(a, b):
    """PackedLight::difference_priority (space/light/data.rs:193-211) of two texels (r, g, b, status)."""
    d = int(np.abs(a[:3].astype(int) - b[:3].astype(int)).max())
    if a[3] != b[3]:
        d = min(255, d + 63)
    return d


def assert_info_matches_queue(info, lit):
    q = lit.light_download_queue()
    assert info["queue_count"] == int((q > 0).sum())
    assert info["max_queue_priority"] == int(q.max())
    assert lit.light_stats()["cube_updates"] == info["update_count"]


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_info_equals_the_downloaded_queue(devices):
    lit = Lit(devices, light_scene(seed=9))
    lit.light_fast_evaluate()
    queue, field = lit.light_download_queue(), lit.field()
    info = lit.light_update_from_queue(0)
    assert info["update_count"] == 0 and info["max_update_difference"] == 0 and info["queue_count"] > 100
    assert_info_matches_queue(info, lit)
    assert np.array_equal(lit.light_download_queue(), queue) and np.array_equal(lit.field(), field)
    info = lit.light_update_from_queue(100)   # inside the first band: a cut round
    assert info["update_count"] == 100 and info["max_update_difference"] > 0
    assert_info_matches_queue(info, lit)
    info = lit.light_update_from_queue()
    assert info["update_count"] > 0
    assert_info_matches_queue(info, lit)
    assert info["queue_count"] == 0 and info["max_queue_priority"] == 0
    lit.close()


@pytest.mark.parametrize("cut_level", [250, 240])
@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_one_cut_round_updates_exactly_the_top_of_the_queue(converged, devices, cut_level):
    lit = edited(devices, converged)
    f0 = lit.field().reshape(-1, 4)
    q0 = lit.light_download_queue().reshape(-1).astype(np.int64)
    n250, n240 = int((q0 == 250).sum()), int((q0 == 240).sum())
    assert n250 > 1 and n240 > 1 and int(((q0 > 0) & (q0 < 234)).sum()) == 0   # one band: 250 and 240
    budget = n250 // 2 if cut_level == 250 else n250 + n240 // 2
    queued = np.flatnonzero(q0)
    top = queued[np.lexsort((queued, -q0[queued]))][:budget]   # priority descending, then index ascending
    cubes = (np.stack(np.unravel_index(top, converged.size), axis=1) + np.array(converged.lower)).astype(np.int32)
    computed = lit.light_compute(cubes)                        # on F0; stores nothing
    info = lit.light_update_from_queue(budget)
    assert info["update_count"] == budget
    want = f0.copy()
    diffs = [difference_priority(computed[i], f0[c]) for i, c in enumerate(top)]
    for i, c in enumerate(top):
        if diffs[i] > 0:
            want[c] = computed[i]
    got = lit.field().reshape(-1, 4)
    assert np.array_equal(got, want), f"{int((got != want).any(axis=1).sum())} texels differ"
    assert info["max_update_difference"] == max(diffs)
    q1 = lit.light_download_queue().reshape(-1)
    rest = np.ones(len(q0), dtype=bool)
    rest[top] = False
    assert (q1[rest] >= q0[rest]).all(), "a cube outside the step lost its queued priority"
    assert_info_matches_queue(info, lit)
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_unbounded_step_equals_evaluate(converged, devices):
    results = {}
    for form in ("step", "evaluate"):
        lit = edited(devices, converged)
        n = lit.light_update_from_queue()["update_count"] if form == "step" else lit.light_evaluate(0)[0]
        results[form] = (n, lit.field(), lit.light_download_queue(), *lit.light_take_changes())
        lit.close()
    step, evaluate = results["step"], results["evaluate"]
    assert step[0] == evaluate[0] > 0
    for name, a, b in zip(("field", "queue", "changed cubes", "changed texels"), step[1:], evaluate[1:]):
        assert np.array_equal(a, b), name


BUDGETS = (1, 57, 0, 400, 3000, None)


def run_budgets(devices, space):
    lit = edited(devices, space)
    out = []
    for b in BUDGETS:
        info = lit.light_update_from_queue(b)
        out.append((info, lit.field(), lit.light_download_queue()))
    out.append(lit.light_take_changes())
    lit.close()
    return out


def assert_same_runs(a, b, label):
    for i, (x, y) in enumerate(zip(a[:-1], b[:-1])):
        assert x[0] == y[0], (label, BUDGETS[i])
        assert np.array_equal(x[1], y[1]) and np.array_equal(x[2], y[2]), (label, BUDGETS[i])
    assert all(np.array_equal(x, y) for x, y in zip(a[-1], b[-1])), (label, "changed cubes")


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_steps_are_deterministic(converged, devices):
    first = run_budgets(devices, converged)
    assert first[0][0]["update_count"] == 1 and first[2][0]["update_count"] == 0
    assert_same_runs(first, run_budgets(devices, converged), "again")
    if devices is not None:
        assert_same_runs(first, run_budgets(None, converged), "one context")


def step_until_done(lit, budget, max_steps=5000):
    for _ in range(max_steps):
        info = lit.light_update_from_queue(budget)
        if info["max_queue_priority"] <= 1:
            return info
        assert info["update_count"] == budget
    raise AssertionError("the queue did not drain")


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_small_steps_converge_to_the_oracle(devices):
    space = light_scene(seed=9)
    lit, ol = Lit(devices, space), LightOracle(space)
    lit.light_fast_evaluate()
    ol.fast_evaluate()
    step_until_done(lit, 150)
    ol.evaluate(0)
    compare_fields(lit.field(), ol.field())
    lit.close()
    # a saved Space's queue resumed (Uninitialized texels)
    space = c4_with_uninitialized(n=24)
    lit, ol = Lit(devices, space), LightOracle(space)
    assert lit.light_queue_uninitialized() == ol.queue_uninitialized() > 0
    info = step_until_done(lit, 2000)
    assert info["queue_count"] == 0
    ol.evaluate(0)
    compare_fields(lit.field(), ol.field())
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_rejected_calls_change_nothing(devices):
    space = light_scene(seed=9)
    unlit = Space(space.lower, space.block_ids, space.blocks, sky_colors=space.sky_colors, light_max_distance=0)
    lit = Lit(devices, unlit)
    fn = lit.scene._fn("light_update_from_queue")
    info = abi.LightUpdatesInfo()
    info.update_count = 77
    assert fn(lit.scene.handle, 10, C.byref(info)) == abi.ERR_INVALID   # LightPhysics::None
    assert info.update_count == 77
    with pytest.raises(AicbError) as e:
        lit.light_update_from_queue(10)
    assert e.value.status == abi.ERR_INVALID
    lit.close()
    lit = Lit(devices, space)
    lit.light_fast_evaluate()
    queue, field, changed = lit.light_download_queue(), lit.field(), lit.light_changes_count()
    assert fn(None, 10, C.byref(info)) == abi.ERR_INVALID and info.update_count == 77
    assert np.array_equal(lit.light_download_queue(), queue) and np.array_equal(lit.field(), field)
    assert lit.light_changes_count() == changed
    assert fn(lit.scene.handle, 64, None) == abi.OK                     # info may be NULL
    stats = lit.light_stats()
    assert stats["cube_updates"] == 64 and stats["rounds"] > 0
    lit.close()
