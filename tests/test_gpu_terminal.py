"""aicb_render_layers_terminal / aicb_group_render_layers_terminal — the desktop terminal's frame (terminal.rs:114-142):
ColorCharacterBuf through every layer — against the CPU restatement (oracle_terminal/) bit for bit, against the
library's other calls on the same layers, and on device groups."""
import ctypes as C

import numpy as np
import pytest

import aicb200
import orc
import termorc
from aicb200 import (FOG_NONE, LIGHT_BOUNCE, LIGHT_FLAT, LIGHT_LINEAR, LIGHT_NONE, TRANSPARENCY_VOLUMETRIC, AicbError,
                     Block, Camera, Context, GraphicsOptions, RtRenderer, Space, SpaceRaytracer, Viewport, abi, scenes)
from test_gpu_resolve import faint_slab

pytestmark = pytest.mark.gpu

NO_WORLD = aicb200.srgb8_to_linear((0xBC, 0xBC, 0xBC)) + (1.0,)
CASES = [
    dict(world=True, ui=True, backdrop=(0.1, 0.3, 0.6, 0.5)),
    dict(world=True, ui=True, backdrop=None),
    dict(world=True, ui=False, backdrop=(0.9, 0.2, 0.1, 0.25)),
    dict(world=False, ui=True, backdrop=(0.0, 0.5, 0.0, 0.3)),   # NO_WORLD_TO_SHOW
    dict(world=False, ui=True, backdrop=None),                   # NO_WORLD_TO_SHOW
]


@pytest.fixture(autouse=True, scope="module")
def _oracle_rounds_once():
    prev = orc.get_libm()
    orc.set_libm(orc.LIBM_CR)
    termorc.set_libm(termorc.LIBM_CR)
    yield
    orc.set_libm(prev)


def layer_setup(mixed_space, ui_space, aa, debug=False, w=64, h=48):
    wopts = GraphicsOptions(view_distance=40.0, antialiasing_always=aa, exposure=1.75, debug_pixel_cost=debug)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT, exposure=0.625,
                            antialiasing_always=aa)
    wcam = scenes.standard_camera(mixed_space, wopts, w, h)
    ucam = scenes.standard_camera(ui_space, uopts, w, h, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    return wopts, uopts, wcam, ucam


def pick(c, world, ui):
    return (world if c["world"] else None), (ui if c["ui"] else None)


def same_frame(a, b):
    """rgba as f32 bits, text and layer equal."""
    return (np.array_equal(a["rgba"].view(np.uint32), b["rgba"].view(np.uint32)) and
            np.array_equal(a["text"], b["text"]) and np.array_equal(a["layer"], b["layer"]))


@pytest.mark.parametrize("aa,debug", [(False, False), (True, False), (False, True), (True, True)])
def test_frame_equals_the_oracle_and_the_other_calls(aa, debug):
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    wopts, uopts, wcam, ucam = layer_setup(mixed, ui_space, aa, debug)
    wrt = SpaceRaytracer(mixed, wopts)
    urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
    wo, uo = termorc.Scene(mixed), termorc.Scene(ui_space)
    for c in CASES:
        label = f"aa={aa} debug={debug} {c}"
        got = aicb200.render_layers_terminal(*pick(c, (wrt, wcam, wopts), (urt, ucam, uopts)), c["backdrop"], NO_WORLD)
        ref = termorc.render_layers_terminal(*pick(c, (wo, wcam, wopts), (uo, ucam, uopts)), c["backdrop"], NO_WORLD)
        assert same_frame(got, ref), label
        assert got["info"].cubes_traced == ref["cubes_traced"], label
        # the same rays as draw_rgba through the layers: its bytes are the colour's sRGB8 encoding, its info the same
        img = aicb200.render_layers(*pick(c, (wrt, wcam, wopts), (urt, ucam, uopts)), c["backdrop"], NO_WORLD)
        assert np.array_equal(termorc.to_srgb8(got["rgba"]), img.data.reshape(-1, 4)), label
        assert got["info"].cubes_traced == img.info.cubes_traced and got["info"].counters == img.info.counters, label
        assert got["info"].rays == img.info.rays
        if c["ui"] and not debug:
            assert (got["layer"] == abi.LAYER_UI).any()
        if c["backdrop"] is not None or not c["world"]:   # the backdrop's or the paint's " "
            assert (got["text"] == abi.TEXT_BLANK).any()
    if not debug:   # world only, no backdrop: the text of print_space's entry point (the first hit either way)
        got = aicb200.render_layers_terminal((wrt, wcam, wopts), None, None, None)
        text = np.zeros(64 * 48, dtype=np.int32)
        o = wopts.to_abi(True)
        lib = aicb200.load_library()
        assert lib.aicb_render_text(wrt.handle, C.byref(wcam.data), C.byref(o), text.ctypes.data, text.size,
                                    None) == abi.OK
        assert np.array_equal(got["text"].reshape(-1), text)
        assert (got["layer"][got["text"] >= 0] == abi.LAYER_WORLD).all()
    urt.close()
    wrt.close()


def corridor():
    """16 x 16 x 1500 cubes of air, one block at the far end: the rays down its length reach the 1000-step cap."""
    ids = np.zeros((16, 16, 1500), dtype=np.uint16)
    ids[:, :, -1] = 1
    return Space((0, 0, 0), ids, [Block.air(), Block(color=(0.5, 0.5, 0.5, 1.0))])


def test_step_cap_is_x():
    space = corridor()
    opts = GraphicsOptions(fog=FOG_NONE, lighting_display=LIGHT_NONE, view_distance=3000.0, fov_y=20.0)
    cam = Camera(opts, Viewport.with_scale(1.0, (25, 17)))   # the centre pixel looks straight down the corridor
    cam.look_at_y_up((8.0, 8.0, -2.0), (8.0, 8.0, 1500.0))
    rt = SpaceRaytracer(space, opts)
    got = aicb200.render_layers_terminal((rt, cam, opts), None, None, NO_WORLD)
    ref = termorc.render_layers_terminal((termorc.Scene(space), cam, opts), None, None, NO_WORLD)
    assert (got["text"] == abi.TEXT_INCOMPLETE).any() and (got["text"] == abi.TEXT_ENTERED_SPACE).any()
    assert same_frame(got, ref)
    assert got["info"].cubes_traced == ref["cubes_traced"]
    rt.close()


@pytest.mark.parametrize("lighting", [LIGHT_NONE, LIGHT_FLAT, LIGHT_LINEAR])
def test_deep_frame_overflows_then_matches_through_both_compositing_paths(lighting):
    """19-65 surfaces per ray in the world layer behind a UI layer: the world pass of a fresh context overflows the 8
    hit slots per ray and is re-issued from the UI pass's accumulator and text.  Then the world alone matches the
    oracle through resolve_kernel (None / Flat) and through shade_kernel + encode_kernel."""
    world = faint_slab()
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    wopts = GraphicsOptions(lighting_display=lighting, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0,
                            exposure=1.5)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT)
    wcam = scenes.standard_camera(world, wopts, 64, 32, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    ucam = scenes.standard_camera(ui_space, uopts, 64, 32, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    tw = termorc.Scene(world)
    ref = termorc.render_layers_terminal((tw, wcam, wopts), (termorc.Scene(ui_space), ucam, uopts), None, NO_WORLD)
    ref_world = termorc.render_layers_terminal((tw, wcam, wopts), None, None, NO_WORLD)
    ctx = Context()
    try:
        wrt = SpaceRaytracer(world, wopts, ctx)
        urt = SpaceRaytracer(ui_space, uopts, ctx)
        got = aicb200.render_layers_terminal((wrt, wcam, wopts), (urt, ucam, uopts), None, NO_WORLD)
        assert got["info"].counters[2] > 8 * 64 * 32   # more surface hits than 8 per world ray
        assert (got["layer"] == abi.LAYER_UI).any() and (got["layer"] == abi.LAYER_WORLD).any()
        assert same_frame(got, ref)
        assert got["info"].cubes_traced == ref["cubes_traced"]
        for fused in ((True, False) if lighting != LIGHT_LINEAR else (False,)):
            if fused:
                empty = RtRenderer(wcam, ctx)
                empty.update(Space((0, 0, 0), np.zeros((4, 4, 4), dtype=np.uint16), [Block.air()]))
                empty.draw_colorbuf()   # no surfaces: the next frame is fused
                empty.rt.close()
            got = aicb200.render_layers_terminal((wrt, wcam, wopts), None, None, NO_WORLD)
            assert (got["info"].stage_ms[3] == 0.0) == fused
            assert same_frame(got, ref_world), f"fused={fused}"
            assert got["info"].cubes_traced == ref_world["cubes_traced"]
        urt.close()
        wrt.close()
    finally:
        ctx.close()


DEVICES = ([0], [0, 0], [0, 0, 0])


@pytest.mark.parametrize("aa,debug,bounce", [(False, False, False), (True, False, False), (False, True, False),
                                             (False, False, True)],
                         ids=["False-False", "True-False", "False-True", "bounce"])
def test_group_frames_equal_the_single_context_frame(aa, debug, bounce):
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    wopts, uopts, wcam, ucam = layer_setup(mixed, ui_space, aa, debug, h=45)   # 45 rows: not a multiple of 16 x n
    if bounce:   # the world layer with LightingOption::Bounce, whose frames run a secondary pass per sample
        wopts = GraphicsOptions(view_distance=40.0, exposure=1.75, lighting_display=LIGHT_BOUNCE, bounce_samples=2)
    wrt = SpaceRaytracer(mixed, wopts)
    urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
    alone = [aicb200.render_layers_terminal(*pick(c, (wrt, wcam, wopts), (urt, ucam, uopts)), c["backdrop"], NO_WORLD)
             for c in CASES]
    for devices in DEVICES:
        g = aicb200.DeviceGroup(devices)
        gw, gu = g.add_scene(mixed), g.add_scene(ui_space)
        for c, ref in zip(CASES, alone):
            got = g.render_layers_terminal(*pick(c, (gw, wcam, wopts), (gu, ucam, uopts)), c["backdrop"], NO_WORLD)
            assert same_frame(got, ref), f"{devices} aa={aa} debug={debug} bounce={bounce} {c}"
            assert got["info"].cubes_traced == ref["info"].cubes_traced and got["info"].rays == ref["info"].rays
        g.close()
    urt.close()
    wrt.close()


def test_group_world_pass_overflow_on_every_device():
    world = faint_slab()
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    wopts = GraphicsOptions(lighting_display=LIGHT_FLAT, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT)
    w, h = 128, 96   # every device's share has more hits than its first stream (>= 65536 slots) holds
    wcam = scenes.standard_camera(world, wopts, w, h, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    ucam = scenes.standard_camera(ui_space, uopts, w, h, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    bd = (0.1, 0.3, 0.6, 0.5)
    ctx = Context()
    wrt = SpaceRaytracer(world, wopts, ctx)
    urt = SpaceRaytracer(ui_space, uopts, ctx)
    ref = aicb200.render_layers_terminal((wrt, wcam, wopts), (urt, ucam, uopts), bd, NO_WORLD)
    assert ref["info"].counters[2] > 8 * ref["info"].rays
    for devices in DEVICES:
        g = aicb200.DeviceGroup(devices)   # fresh contexts: every device's first world pass overflows
        gw, gu = g.add_scene(world), g.add_scene(ui_space)
        got = g.render_layers_terminal((gw, wcam, wopts), (gu, ucam, uopts), bd, NO_WORLD)
        assert same_frame(got, ref), f"{devices}"
        assert got["info"].cubes_traced == ref["info"].cubes_traced
        g.close()
    urt.close()
    wrt.close()
    ctx.close()


def test_rejected_input():
    space = scenes.small_mixed_scene(n=8, seed=7)
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(space, opts, 16, 8)
    lib = aicb200.load_library()
    rt = SpaceRaytracer(space, opts)
    o = opts.to_abi(True)
    layer = abi.Layer(rt.handle, C.pointer(cam.data), C.pointer(o))
    out = (abi.TerminalPixel * 200)()
    assert lib.aicb_render_layers_terminal(C.byref(layer), None, None, None, out, 127, None) == abi.ERR_INVALID
    assert lib.aicb_render_layers_terminal(C.byref(layer), None, None, None, None, 16 * 8, None) == abi.ERR_INVALID
    assert lib.aicb_render_layers_terminal(C.byref(layer), None, None, None, out, 16 * 8, None) == abi.OK
    other = Context()
    rt2 = SpaceRaytracer(space, opts, other)
    with pytest.raises(AicbError) as e:   # the layers on two contexts
        aicb200.render_layers_terminal((rt, cam, opts), (rt2, cam, opts))
    assert e.value.status == abi.ERR_INVALID
    g1, g2 = aicb200.DeviceGroup([0]), aicb200.DeviceGroup([0])
    s1, s2 = g1.add_scene(space), g2.add_scene(space)
    with pytest.raises(AicbError) as e:   # the layers in two groups
        g1.render_layers_terminal((s1, cam, opts), (s2, cam, opts))
    assert e.value.status == abi.ERR_INVALID
    gl = abi.GroupLayer(s1.handle, C.pointer(cam.data), C.pointer(o))
    assert lib.aicb_group_render_layers_terminal(C.byref(gl), None, None, None, out, 127, None) == abi.ERR_INVALID
    assert lib.aicb_group_render_layers_terminal(C.byref(gl), None, None, None, None, 16 * 8, None) == abi.ERR_INVALID
    g1.close()
    g2.close()
    rt2.close()
    other.close()
    rt.close()
