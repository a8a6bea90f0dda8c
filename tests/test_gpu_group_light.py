"""Light propagation on a device group (aicb_group_light_*): every device walks a share of each round against its own
replica, device 0 applies and pushes what it wrote, and every replica stays current.  The group must meet the
single-context contract (tests/test_gpu_light.py) and leave identical replicas.  One H100 is enough: the same device
is named several times, each name its own context."""
import numpy as np
import pytest

import aicb200
import orc
from aicb200 import AicbError, Block, GraphicsOptions, Space, SpaceRaytracer, abi, scenes
from test_gpu_light import NO_RAYS, OPAQUE, VISIBLE, WHITE, all_cubes, compare_fields, empty_space, light_scene

pytestmark = pytest.mark.gpu

DEVICES = ([0], [0, 0], [0, 0, 0])


def group_scene(devices, space):
    g = aicb200.DeviceGroup(devices)
    return g, g.add_scene(space)


def assert_replicas_identical(gs, n):
    first = gs.light_download(0)
    for i in range(1, n):
        assert np.array_equal(gs.light_download(i), first), f"replica {i} differs from replica 0"
    return first


def slab_space():
    """The translucent-slab scene of test_gpu_light: rays that cross more than four translucent blocks take the
    lockstep walk."""
    n = 14
    ids = np.zeros((n, n, n), dtype=np.uint16)
    ids[:, 0, :] = 1
    ids[3:11, 2:9, 6] = 2
    ids[3:11, 2:9, 7] = 3
    ids[3:11, 2:9, 8] = 2
    ids[5:9, 9:13, 3:12] = 3
    ids[6, 4, 2] = 4
    blocks = [Block.air(), Block(color=(0.7, 0.7, 0.7, 1.0)), Block(color=(0.3, 0.6, 0.9, 0.125)),
              Block(color=(0.9, 0.5, 0.2, 0.0625), emission=(0.05, 0.02, 0.0)),
              Block(color=(0.1, 0.1, 0.1, 1.0), emission=(6.0, 5.0, 3.0))]
    light = np.zeros((n, n, n, 4), dtype=np.uint8)
    light[..., 3] = NO_RAYS
    return Space((0, 0, 0), ids, blocks, light=light, sky_colors=scenes.OCTANT_SKY, light_max_distance=20)


def c4_slice():
    """The 32^3 slice of BASELINE configs[4]'s shape that test_light_bench_shape_flood uses."""
    n = 32
    h = scenes.grid_hash(21, (n, n, n))
    blocks = [Block.air()] + [Block(color=(0.3 + 0.1 * i, 0.8 - 0.1 * i, 0.5, 1.0)) for i in range(4)] + \
             [Block(color=(0.1, 0.1, 0.1, 1.0), emission=(3.0, 3.0, 2.0))]
    ids = np.where((h & np.uint64(15)) == 0, 1 + ((h >> np.uint64(8)) % np.uint64(5)).astype(np.int64), 0).astype(np.uint16)
    ids[:, : n // 4, :] = 1
    light = np.zeros((n, n, n, 4), dtype=np.uint8)
    light[..., 3] = NO_RAYS
    return Space((0, 0, 0), ids, blocks, light=light, sky_colors=scenes.OCTANT_SKY, light_max_distance=30)


def with_field(space, field):
    return Space(space.lower, space.block_ids, space.blocks, light=field, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


@pytest.mark.parametrize("make,max_updates", [(light_scene, 800), (slab_space, 1500)])
def test_group_compute_light_is_bit_exact(make, max_updates):
    space = make()
    ol = orc.OracleLight(space)
    ol.fast_evaluate()
    ol.evaluate(0, max_updates=max_updates)
    field = ol.field()
    cubes = all_cubes(space)
    ref = ol.compute(cubes)
    rt = SpaceRaytracer(with_field(space, field), GraphicsOptions())
    alone = rt.light_compute(cubes)
    alone_overflow = rt.light_stats()["rounds"]
    assert np.array_equal(alone, ref)
    if make is slab_space:
        assert alone_overflow > 0
    for devices in DEVICES:
        g, gs = group_scene(devices, with_field(space, field))
        got = gs.light_compute(cubes)
        assert np.array_equal(got, ref), f"{devices}: {np.argwhere((got != ref).any(axis=1))[:5]}"
        stats = gs.light_stats()
        assert stats["cube_updates"] == len(cubes)
        assert stats["rounds"] == alone_overflow, (devices, stats["rounds"], alone_overflow)
        assert np.array_equal(assert_replicas_identical(gs, len(devices)), field)   # compute stores nothing
        g.close()
    rt.close()


@pytest.mark.parametrize("devices", DEVICES)
def test_reference_light_kats_on_groups(devices):
    """light/tests.rs:233-261 exact neighbour values around an opaque emitter; :111-160; :162-174."""
    sp = empty_space((3, 3, 3), [Block(color=WHITE, emission=(0.5, 1.0, 2.0))], sky=[(0.0, 0.0, 0.0)])
    g, gs = group_scene(devices, sp)
    gs.light_edit_and_propagate([(1, 1, 1)], [1], 0)
    f = assert_replicas_identical(gs, len(devices))
    L = orc.lib()
    val = lambda t: tuple(np.float32(L.orc_packed_light_lut(int(v))) for v in t[:3])
    f32 = np.float32
    assert val(f[0, 1, 1]) == val(f[2, 1, 1]) == (f32(0.13397168), f32(0.26794338), f32(0.53588676))
    assert val(f[1, 0, 1]) == val(f[1, 2, 1]) == (f32(0.1649385), f32(0.32987696), f32(0.6597539))
    assert val(f[1, 1, 0]) == val(f[1, 1, 2]) == (f32(0.21763763), f32(0.43527526), f32(0.8705506))
    g.close()
    # `evaluate_light`: 0, then 2 updates, then 0
    g, gs = group_scene(devices, empty_space((3, 1, 1), [Block(color=WHITE)]))
    assert gs.light_evaluate(0)[0] == 0
    assert gs.light_edit_and_propagate([(1, 0, 0)], [1], 0)[0] == 2
    assert gs.light_evaluate(0)[0] == 0
    g.close()
    # `step`: the cube next to a new opaque block takes the sky colour
    g, gs = group_scene(devices, empty_space((3, 1, 1), [Block(color=WHITE)], sky=[(1.0, 0.0, 0.0)]))
    n, md = gs.light_edit_and_propagate([(0, 0, 0)], [1], 0)
    f = assert_replicas_identical(gs, len(devices))
    assert n == 1 and tuple(f[0, 0, 0]) == (0, 0, 0, OPAQUE) and tuple(f[2, 0, 0]) == (0, 0, 0, NO_RAYS)
    assert tuple(f[1, 0, 0]) == (144, 0, 0, VISIBLE)
    g.close()


@pytest.mark.parametrize("devices", DEVICES)
def test_group_converged_field_matches_oracle(devices):
    space = light_scene()
    ol = orc.OracleLight(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    g, gs = group_scene(devices, space)
    gs.light_fast_evaluate()
    n, md, nv = gs.light_evaluate(0)
    assert n > 0 and nv > 0
    stats = gs.light_stats()
    assert stats["cube_updates"] == n and stats["chart_node_visits"] == nv and stats["rounds"] > 0
    assert stats["device_seconds"] > 0
    compare_fields(assert_replicas_identical(gs, len(devices)), ol.field())
    g.close()


def edited_ids(space, cubes, ids):
    out = space.block_ids.copy()
    for c, i in zip(cubes, ids):
        out[tuple(c - np.array(space.lower))] = i
    return out


@pytest.mark.parametrize("make", [lambda: light_scene(seed=9), c4_slice], ids=["light_scene", "c4_slice"])
@pytest.mark.parametrize("devices", DEVICES)
def test_group_edits_then_propagate(devices, make):
    space = make()
    ol = orc.OracleLight(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    g, gs = group_scene(devices, space)
    gs.light_fast_evaluate()
    gs.light_evaluate(0)
    rng = np.random.default_rng(4)
    cubes = np.stack([rng.integers(0, space.size[a], 60) + space.lower[a] for a in range(3)], axis=1).astype(np.int32)
    ids = rng.integers(0, len(space.blocks), 60).astype(np.uint16)
    ol.set_cubes(cubes, ids)
    ol.evaluate(0)
    n, md = gs.light_edit_and_propagate(cubes, ids, 0)
    assert n > 0
    field = assert_replicas_identical(gs, len(devices))
    compare_fields(field, ol.field())
    # every strip of a group frame reads its own replica's cells and light: the frame equals one context's frame of a
    # fresh scene made of the edited ids and replica 0's field
    opts = GraphicsOptions(lighting_display=aicb200.LIGHT_LINEAR)
    cam = scenes.standard_camera(space, opts, 64, 48)
    fresh = SpaceRaytracer(Space(space.lower, edited_ids(space, cubes, ids), space.blocks, light=field,
                                 sky_colors=space.sky_colors, light_max_distance=space.light_max_distance), opts)
    got = g.render_layers((gs, cam, opts))
    ref = aicb200.render_layers((fresh, cam, opts))
    assert np.array_equal(got.data, ref.data), devices
    fresh.close()
    g.close()


@pytest.mark.parametrize("devices", DEVICES)
def test_rejected_group_light_calls_change_no_replica(devices):
    space = light_scene(seed=9)
    g, gs = group_scene(devices, space)
    gs.light_fast_evaluate()
    gs.light_evaluate(0)
    opts = GraphicsOptions(lighting_display=aicb200.LIGHT_LINEAR)
    cam = scenes.standard_camera(space, opts, 64, 48)
    before = [gs.light_download(i) for i in range(len(devices))]
    frame = g.render_layers((gs, cam, opts)).data
    inside = [space.lower[0] + 2, space.lower[1] + 3, space.lower[2] + 4]
    outside = [space.lower[0] + space.size[0], space.lower[1], space.lower[2]]
    for cubes, ids in (([inside, outside], [1, 1]), ([inside, inside], [1, len(space.blocks)])):
        with pytest.raises(AicbError) as e:
            gs.light_edit_and_propagate(np.array(cubes, dtype=np.int32), np.array(ids, dtype=np.uint16), 0)
        assert e.value.status == abi.ERR_INVALID
        for i in range(len(devices)):
            assert np.array_equal(gs.light_download(i), before[i]), f"replica {i} changed"
        assert np.array_equal(g.render_layers((gs, cam, opts)).data, frame)
    with pytest.raises(AicbError) as e:
        gs.light_download(len(devices))
    assert e.value.status == abi.ERR_INVALID
    g.close()
    unlit = Space(space.lower, space.block_ids, space.blocks, sky_colors=space.sky_colors, light_max_distance=0)
    g, gs = group_scene(devices, unlit)
    for call in (gs.light_fast_evaluate, lambda: gs.light_evaluate(0), lambda: gs.light_compute(all_cubes(space)[:4]),
                 lambda: gs.light_edit_and_propagate(np.array([inside], dtype=np.int32), np.array([1], dtype=np.uint16))):
        with pytest.raises(AicbError) as e:
            call()
        assert e.value.status == abi.ERR_INVALID
    g.close()
