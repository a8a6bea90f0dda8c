"""SpaceChange::Physics on the GPU (aicb_scene_set_physics / aicb_group_scene_set_physics): Space::set_physics
(space.rs:609-630) and LightStorage::maybe_reinitialize_for_physics_change (space/light/updater.rs:80-113).  A new
LightPhysics reinitialises the light exactly as the oracle does (oracle_light/: orc_light_set_physics); a new sky alone
leaves the light and reaches frames and later light calls; None frees the light.  After every change, every output
equals that of a scene created fresh with the new physics and the light the scene holds.  Every check runs on one
context and on groups of 1, 2 and 3 contexts of one device; a group's replicas stay identical."""
import ctypes as C

import numpy as np
import pytest

import aicb200
import orc
from aicb200 import AicbError, GraphicsOptions, RtRenderer, Space, SpaceRaytracer, abi, scenes
from physicsorc import LightOracle
from test_gpu_light import all_cubes, compare_fields, light_scene
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit

pytestmark = pytest.mark.gpu

OCTANT_SKY = scenes.OCTANT_SKY
UNIFORM_SKY = [(0.4, 0.5, 0.9)]
OPTS = GraphicsOptions(lighting_display=aicb200.LIGHT_LINEAR, fog=aicb200.FOG_ABRUPT)


def with_physics(space, light, sky_colors, light_max_distance):
    return Space(space.lower, space.block_ids, space.blocks, light=light, sky_colors=sky_colors,
                 light_max_distance=light_max_distance)


def converged(devices, space):
    """The scene on `devices` and the light oracle, both converged to epsilon 0, the set of changed cubes emptied."""
    lit = Lit(devices, space)
    lit.light_fast_evaluate()
    lit.light_evaluate(0)
    lit.light_take_changes(discard=True)
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    return lit, ol


def outputs(lit, cam):
    """The layered sRGB8 frame, the texture's colour and depth, and the terminal frame's text, layer and colour of a
    Lit (or of a SpaceRaytracer)."""
    scene, group = (lit, None) if isinstance(lit, SpaceRaytracer) else (lit.scene, lit.group)
    world = (scene, cam, OPTS)
    host = aicb200 if group is None else group
    srgb = host.render_layers(world).data
    rgba, depth, _ = host.render_layers_texture(world, depth_transform=cam.depth_transform())
    term = host.render_layers_terminal(world)
    return {"srgb8": srgb, "texture_rgba": rgba, "texture_depth": depth, "terminal_text": term["text"],
            "terminal_layer": term["layer"], "terminal_rgba": term["rgba"]}


def fresh_outputs(space, cam):
    rt = SpaceRaytracer(space, OPTS)
    try:
        return outputs(rt, cam)
    finally:
        rt.close()


def assert_same_outputs(got, want, what):
    for k in want:
        assert np.array_equal(got[k], want[k]), f"{what}: {k} differs"


def light_calls(lit, space):
    cube = np.array([space.lower], dtype=np.int32)
    return {
        "fast_evaluate": lambda: lit.light_fast_evaluate(),
        "compute": lambda: lit.light_compute(cube),
        "evaluate": lambda: lit.light_evaluate(0),
        "edit_and_propagate": lambda: lit.light_edit_and_propagate(cube, [1], 0),
        "relight_blocks": lambda: lit.light_relight_blocks([1], 0),
        "download": lambda: lit.field(),
        "changes_count": lambda: lit.light_changes_count(),
        "take_changes": lambda: lit.light_take_changes(discard=True),
    }


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_new_distance_reinitialises_the_light(devices):
    space = light_scene(seed=9)
    lit, ol = converged(devices, space)
    lit.set_physics(space.sky_colors, 6)
    ol.set_physics(space.sky_colors, 6)
    assert np.array_equal(lit.field(), ol.field())   # fast_evaluate_light's field, before any evaluation
    assert lit.light_changes_count() == int(np.prod(space.size))
    updates, _, _ = lit.light_evaluate(0)
    assert updates > 0
    ol.evaluate(0)
    compare_fields(lit.field(), ol.field())
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_new_sky_alone_keeps_the_light_and_reaches_light_calls(devices):
    space = light_scene(seed=9)
    lit, _ = converged(devices, space)
    field = lit.field()
    lit.set_physics(UNIFORM_SKY, space.light_max_distance)
    assert np.array_equal(lit.field(), field)
    assert lit.light_changes_count() == 0
    assert lit.light_evaluate(0)[0] == 0
    # compute_light reads the new sky's sky_term
    cubes = all_cubes(space)
    now = with_physics(space, field, UNIFORM_SKY, space.light_max_distance)
    assert np.array_equal(lit.light_compute(cubes), orc.OracleLight(now).compute(cubes))
    # and so does propagation after an edit
    rng = np.random.default_rng(4)
    edits = np.stack([rng.integers(0, space.size[a], 60) + space.lower[a] for a in range(3)], axis=1).astype(np.int32)
    ids = rng.integers(0, len(space.blocks), 60).astype(np.uint16)
    updates, _ = lit.light_edit_and_propagate(edits, ids, 0)
    assert updates > 0
    ol = LightOracle(now)
    ol.set_cubes(edits, ids)
    ol.evaluate(0)
    compare_fields(lit.field(), ol.field())
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_rays_none_rays(devices):
    space = light_scene(seed=9)
    lit, _ = converged(devices, space)
    cam = scenes.standard_camera(space, OPTS, 64, 48)
    bytes_before = lit.device_bytes if devices is None else None
    lit.set_physics(space.sky_colors, 0)
    if devices is None:
        assert bytes_before - lit.device_bytes >= 4 * int(np.prod(space.size))
    assert_same_outputs(outputs(lit, cam), fresh_outputs(with_physics(space, None, space.sky_colors, 0), cam), "None")
    for name, call in light_calls(lit, space).items():
        with pytest.raises(AicbError) as e:
            call()
        assert e.value.status == abi.ERR_INVALID, name
    lit.set_physics(space.sky_colors, 12)
    ol = LightOracle(space)
    ol.fast_evaluate()
    assert np.array_equal(lit.field(), ol.field())
    assert lit.light_changes_count() == int(np.prod(space.size))
    lit.close()
    # a scene created without light and with LightPhysics::None
    unlit = Lit(devices, with_physics(space, None, UNIFORM_SKY, 0))
    with pytest.raises(AicbError):
        unlit.light_fast_evaluate()
    unlit.set_physics(UNIFORM_SKY, 12)
    ol = LightOracle(with_physics(space, None, UNIFORM_SKY, 12))
    ol.fast_evaluate()
    assert np.array_equal(unlit.field(), ol.field())
    assert unlit.light_changes_count() == int(np.prod(space.size))
    unlit.light_evaluate(0)
    ol.evaluate(0)
    compare_fields(unlit.field(), ol.field())
    unlit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_frames_follow_physics(devices):
    space = light_scene(seed=9)
    lit, _ = converged(devices, space)
    cam = scenes.standard_camera(space, OPTS, 64, 48)
    # (sky, distance): a new sky alone (Octants -> Uniform), a new sky and distance (-> Octants, 6), None, Rays again
    for sky, distance in ((UNIFORM_SKY, 12), (OCTANT_SKY, 6), (UNIFORM_SKY, 0), (OCTANT_SKY, 12)):
        lit.set_physics(sky, distance)
        light = lit.field() if distance else None
        want = fresh_outputs(with_physics(space, light, sky, distance), cam)
        assert_same_outputs(outputs(lit, cam), want, f"sky {len(sky)}, distance {distance}")
        if distance:
            lit.light_evaluate(0)   # frames of a field the new physics has moved on
            want = fresh_outputs(with_physics(space, lit.field(), sky, distance), cam)
            assert_same_outputs(outputs(lit, cam), want, f"sky {len(sky)}, distance {distance}, evaluated")
    lit.close()


def test_set_physics_while_a_frame_is_in_flight():
    """A frame issued before a change to None, which frees the light volume it reads, is the frame of the old physics."""
    import torch

    space = light_scene(seed=9)
    lit, _ = converged(None, space)
    rt = lit.scene
    cam = scenes.standard_camera(space, OPTS, 320, 240)
    r = RtRenderer(cam, rt.ctx)
    r.rt = rt
    before = r.draw().data.reshape(-1, 4)
    lib = aicb200.load_library()
    n = cam.data.fb_width * cam.data.fb_height
    d_out = torch.zeros((n, 4), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    o = OPTS.to_abi(True)
    assert lib.aicb_render_srgb8_device(rt.handle, C.byref(cam.data), C.byref(o), None, d_out.data_ptr(), n,
                                        C.c_void_p(stream.cuda_stream)) == abi.OK
    rt.set_physics(UNIFORM_SKY, 0)
    info = abi.RenderInfo()
    assert lib.aicb_render_finish(rt.handle, C.byref(info)) == abi.OK
    torch.cuda.synchronize()
    assert np.array_equal(d_out.cpu().numpy(), before)
    after = r.draw().data.reshape(-1, 4)
    assert not np.array_equal(after, before)
    lit.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_rejected_calls_change_nothing(devices):
    space = light_scene(seed=9)
    lit, _ = converged(devices, space)
    cam = scenes.standard_camera(space, OPTS, 64, 48)
    field, frames = lit.field(), outputs(lit, cam)
    bytes_before = lit.device_bytes if devices is None else None
    fn = lit.scene._fn("scene_set_physics")
    sky = aicb200._sky(UNIFORM_SKY)
    for handle, sky_arg in ((lit.scene.handle, None), (None, C.byref(sky))):
        for distance in (0, 6, 12):
            assert fn(handle, sky_arg, distance) == abi.ERR_INVALID
            assert np.array_equal(lit.field(), field)   # (on a group: every replica, checked identical)
            assert lit.light_changes_count() == 0
            if devices is None:
                assert lit.device_bytes == bytes_before
            assert_same_outputs(outputs(lit, cam), frames, "after a rejected call")
    # an unchanged physics is accepted and does nothing
    lit.set_physics(space.sky_colors, space.light_max_distance)
    assert np.array_equal(lit.field(), field)
    assert lit.light_changes_count() == 0
    lit.close()
