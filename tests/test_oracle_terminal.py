"""The CPU restatement of the desktop terminal's ColorCharacterBuf (oracle_terminal/aic_terminal.cpp): CharacterBuf's
rules on hand-built hits and traced rays, CharacterBuf::mean, the reference's print_space images (text.rs:196-341)
from world-only terminal text, and the colour against the layers oracle that aicb_render_layers_srgb8 is checked
against."""
import json
import os

import numpy as np
import pytest

import aicb200
import orc
import termorc
from aicb200 import FOG_NONE, LIGHT_NONE, Block, Camera, GraphicsOptions, Space, Viewport, abi, scenes
from termorc import BACKDROP, DEBUG_RG, ENTER_SPACE, INCOMPLETE, PAINT, SKY, SURFACE
from test_camera import color_for_make_blocks

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EMPTY, ENTERED, X, BLANK = abi.TEXT_EMPTY, abi.TEXT_ENTERED_SPACE, abi.TEXT_INCOMPLETE, abi.TEXT_BLANK
NONE, WORLD, UI = abi.LAYER_NONE, abi.LAYER_WORLD, abi.LAYER_UI
OPTS = GraphicsOptions(fog=FOG_NONE, lighting_display=LIGHT_NONE, view_distance=50.0)
HIT = (0.5, 0.5, -5.0, 0.0, 0.0, 1.0)    # meets cube (0, 0, 0) at t = 5
MISS = (5.5, 5.5, -5.0, 0.0, 0.0, 1.0)   # passes beside it, outside the Space
NO_WORLD = aicb200.srgb8_to_linear((0xBC, 0xBC, 0xBC)) + (1.0,)


def one_cube(color, index=1):
    """One cube of block `index` (the blocks before it are air), so that the two layers name different indices."""
    blocks = [Block.air()] * index + [Block(color=color)]
    return Space((0, 0, 0), np.full((1, 1, 1), index, dtype=np.uint16), blocks)


@pytest.fixture(scope="module")
def layers():
    termorc.set_libm(termorc.LIBM_CR)
    ui_partial = termorc.Scene(one_cube((0.2, 0.9, 0.3, 0.5), index=2))
    world = termorc.Scene(one_cube((0.8, 0.1, 0.1, 1.0)))
    return ui_partial, world


def trace(world_scene, ui_scene, backdrop=None, no_world=None, world_ray=HIT, ui_ray=HIT, opts=OPTS):
    w = (world_scene, opts) if world_scene else None
    u = (ui_scene, opts) if ui_scene else None
    r = termorc.trace_samples(w, u, backdrop, no_world, [world_ray] if w else None, [ui_ray] if u else None)
    return int(r["text"][0]), int(r["layer"][0]), r["colorbuf"][0]


# ---- CharacterBuf::add (text.rs:86-94) on hand-built hits ---------------------------------------------------------
def test_enter_space_and_sky():
    assert termorc.character_add((EMPTY, NONE), [(ENTER_SPACE, -1, NONE)]) == (ENTERED, NONE)
    assert termorc.character_add((ENTERED, NONE), [(ENTER_SPACE, -1, NONE)]) == (ENTERED, NONE)
    assert termorc.character_add((EMPTY, NONE), [(SKY, -1, NONE)]) == (EMPTY, NONE)        # the sky is ignored
    assert termorc.character_add((ENTERED, NONE), [(SKY, -1, NONE)]) == (ENTERED, NONE)
    assert termorc.character_add((7, WORLD), [(ENTER_SPACE, -1, NONE)]) == (7, WORLD)       # a Hit stays


def test_first_surface_names_its_block():
    hits = [(ENTER_SPACE, -1, NONE), (SURFACE, 3, UI), (SURFACE, 5, UI), (SKY, -1, NONE)]
    assert termorc.character_add((EMPTY, NONE), hits) == (3, UI)
    assert termorc.character_add((ENTERED, NONE), [(SURFACE, 4, WORLD)]) == (4, WORLD)


def test_incomplete_is_x_without_an_earlier_hit():
    assert termorc.character_add((ENTERED, NONE), [(INCOMPLETE, -1, NONE)]) == (X, NONE)
    assert termorc.character_add((2, WORLD), [(INCOMPLETE, -1, NONE)]) == (2, WORLD)
    assert termorc.character_add((X, NONE), [(SURFACE, 2, WORLD)]) == (X, NONE)   # "X" is a Hit too


@pytest.mark.parametrize("exception", [BACKDROP, DEBUG_RG, PAINT])
def test_backdrop_debug_and_paint_are_blank(exception):
    assert termorc.character_add((EMPTY, NONE), [(exception, -1, NONE)]) == (BLANK, NONE)
    assert termorc.character_add((ENTERED, NONE), [(exception, -1, NONE)]) == (BLANK, NONE)
    assert termorc.character_add((6, UI), [(exception, -1, NONE)]) == (6, UI)
    assert termorc.character_add((BLANK, NONE), [(SURFACE, 1, WORLD)]) == (BLANK, NONE)


# ---- CharacterBuf::mean (text.rs:96-108) ---------------------------------------------------------------------------
def test_mean():
    assert termorc.character_mean([(ENTERED, NONE), (EMPTY, NONE)]) == (EMPTY, NONE)
    assert termorc.character_mean([(EMPTY, NONE), (ENTERED, NONE), (ENTERED, NONE), (ENTERED, NONE)]) == (EMPTY, NONE)
    assert termorc.character_mean([(ENTERED, NONE)] * 4) == (ENTERED, NONE)
    assert termorc.character_mean([(ENTERED, NONE), (EMPTY, NONE), (5, WORLD), (7, UI)]) == (5, WORLD)
    assert termorc.character_mean([(BLANK, NONE), (5, WORLD), (EMPTY, NONE), (EMPTY, NONE)]) == (BLANK, NONE)
    assert termorc.character_mean([(EMPTY, NONE), (EMPTY, NONE), (EMPTY, NONE), (X, NONE)]) == (X, NONE)
    assert termorc.character_mean([(9, UI)]) == (9, UI)


# ---- the layer walk on traced rays -------------------------------------------------------------------------------
def test_world_surface_and_miss(layers):
    _, world = layers
    assert trace(world, None)[:2] == (1, WORLD)
    assert trace(world, None, world_ray=MISS)[:2] == (EMPTY, NONE)   # never entered the one-cube Space


def test_ui_name_survives_the_world_pass(layers):
    ui, world = layers
    text, layer, cb = trace(world, ui)
    assert (text, layer) == (2, UI)
    assert cb[3] == 0.0   # the world's opaque cube behind the half-transparent UI cube
    assert trace(world, ui, ui_ray=MISS)[:2] == (1, WORLD)


def test_backdrop_is_blank_before_the_world(layers):
    ui, world = layers
    bd = (0.1, 0.2, 0.3, 0.5)
    assert trace(world, None, backdrop=bd)[:2] == (BLANK, NONE)               # riding in front of the world
    assert trace(world, ui, backdrop=bd, ui_ray=MISS)[:2] == (BLANK, NONE)
    assert trace(world, ui, backdrop=bd)[:2] == (2, UI)                       # the UI hit came first
    assert trace(None, ui, backdrop=bd, ui_ray=MISS)[:2] == (BLANK, NONE)


def test_debug_pixel_cost_is_blank_without_a_hit(layers):
    _, world = layers
    dbg = GraphicsOptions(fog=FOG_NONE, lighting_display=LIGHT_NONE, view_distance=50.0, debug_pixel_cost=True)
    assert trace(world, None, world_ray=MISS, opts=dbg)[:2] == (BLANK, NONE)
    assert trace(world, None, opts=dbg)[:2] == (1, WORLD)


def test_paint_replaces_a_ui_named_block(layers):
    ui, _ = layers
    text, layer, cb = trace(None, ui, no_world=NO_WORLD)
    assert (text, layer) == (BLANK, NONE)   # P::paint starts a fresh accumulator
    assert cb[3] == np.float32(1.0) - np.float32(NO_WORLD[3])
    assert trace(None, ui, no_world=NO_WORLD, ui_ray=MISS)[:2] == (BLANK, NONE)
    assert trace(None, ui, ui_ray=MISS)[:2] == (EMPTY, NONE)   # without the paint colour: nothing


def corridor():
    """16 x 16 x 1500 cubes of air, one block at the far end: a ray down its length counts more than 1000 steps."""
    ids = np.zeros((16, 16, 1500), dtype=np.uint16)
    ids[:, :, -1] = 1
    return Space((0, 0, 0), ids, [Block.air(), Block(color=(0.5, 0.5, 0.5, 1.0))])


def test_step_cap_is_x():
    termorc.set_libm(termorc.LIBM_CR)
    sc = termorc.Scene(corridor())
    opts = GraphicsOptions(fog=FOG_NONE, lighting_display=LIGHT_NONE, view_distance=3000.0)
    r = termorc.trace_samples((sc, opts), None, None, None, [(8.5, 8.5, -1.0, 0.0, 0.0, 1.0),
                                                              (8.5, 8.5, 0.5, 1.0, 0.0, 0.1)])
    assert list(r["text"]) == [X, ENTERED]   # the second ray leaves through the side after a few steps


# ---- the reference's known answers: print_space (text.rs:196-258, 265-341) ----------------------------------------
def print_space_rows(space, chars):
    """PrintSpace::fmt's 80 x 40 rays (as tests/test_camera.py builds them), traced as a world-only terminal frame."""
    opts = GraphicsOptions()
    cam = Camera(opts, Viewport((40.0, 40.0), (80, 40)))
    center = [space.lower[a] + space.size[a] / 2.0 for a in range(3)]
    cam.look_at_y_up(aicb200.eye_for_look_at(space.lower, space.size, (1.0, 1.0, 1.0)), center)
    rays = [cam.project_ndc_into_world((x + 0.5) / 80.0 * 2.0 - 1.0, -((y + 0.5) / 40.0 * 2.0 - 1.0))
            for y in range(40) for x in range(80)]
    text = termorc.trace_samples((termorc.Scene(space), opts), None, None, None, np.array(rays))["text"]
    special = {EMPTY: ".", ENTERED: " ", BLANK: " ", X: "X"}
    return ["".join(special[int(t)] if t < 0 else chars[int(t)] for t in text[r * 80:(r + 1) * 80]) for r in range(40)]


def test_world_only_text_reproduces_print_space_images():
    termorc.set_libm(termorc.LIBM_CR)
    golden = json.load(open(os.path.join(GOLDEN, "text_images.json")))
    ids = np.array([1, 2, 3], dtype=np.uint16).reshape(3, 1, 1)
    space = Space((0, 0, 0), ids, [Block.air()] + [Block(color=color_for_make_blocks(i, 3)) for i in range(3)])
    assert print_space_rows(space, {1: "0", 2: "1", 3: "2"}) == golden["print_space_test"]
    idx = np.zeros((4, 2, 4), dtype=np.uint16)
    pal = np.zeros((1, 8), dtype=np.float32)
    pal[0, :4] = (1.0, 1.0, 1.0, 1.0)
    partial = Block(resolution=4, voxel_lower=(0, 0, 0), indices=idx, palette=pal)
    space = Space((0, 0, 0), np.array([1, 2], dtype=np.uint16).reshape(2, 1, 1),
                  [Block.air(), Block(color=color_for_make_blocks(0, 1)), partial])
    assert print_space_rows(space, {1: "0", 2: "P"}) == golden["partial_voxels"]


# ---- whole frames against the layers oracle -------------------------------------------------------------------------
CASES = [
    dict(world=True, ui=True, backdrop=(0.1, 0.3, 0.6, 0.5)),
    dict(world=True, ui=True, backdrop=None),
    dict(world=True, ui=False, backdrop=(0.9, 0.2, 0.1, 0.25)),
    dict(world=False, ui=True, backdrop=(0.0, 0.5, 0.0, 0.3)),
    dict(world=False, ui=True, backdrop=None),
]


@pytest.mark.parametrize("aa", [False, True])
def test_frame_colour_and_cubes_traced_equal_the_layers_oracle(aa):
    """to_srgb8 of the terminal's colour is draw_rgba's pixel, and the rays stop where draw_rgba's do; a world-only
    frame's text is print_space's CharacterBuf (the first hit under either stop rule)."""
    orc.set_libm(orc.LIBM_CR)
    termorc.set_libm(termorc.LIBM_CR)
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    wopts = GraphicsOptions(view_distance=40.0, antialiasing_always=aa, exposure=1.75)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, exposure=0.625, antialiasing_always=aa)
    wcam = scenes.standard_camera(mixed, wopts, 24, 18)
    ucam = scenes.standard_camera(ui_space, uopts, 24, 18, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    tw, tu = termorc.Scene(mixed), termorc.Scene(ui_space)
    ow, ou = orc.OracleScene(mixed), orc.OracleScene(ui_space)
    for c in CASES:
        t = termorc.render_layers_terminal((tw, wcam, wopts) if c["world"] else None,
                                           (tu, ucam, uopts) if c["ui"] else None, c["backdrop"], NO_WORLD)
        ref = orc.render_layers((ow, wcam, wopts) if c["world"] else None, (ou, ucam, uopts) if c["ui"] else None,
                                c["backdrop"], NO_WORLD)
        assert np.array_equal(termorc.to_srgb8(t["rgba"]), ref["srgb8"]), f"aa={aa} {c}"
        assert t["cubes_traced"] == ref["cubes_traced"], f"aa={aa} {c}"
        named = t["text"] >= 0
        assert (t["layer"][named] != NONE).all() and (t["layer"][~named] == NONE).all()
        if c["ui"]:
            assert (t["layer"] == UI).any()
        if c["backdrop"] is not None and not c["ui"]:   # the backdrop comes before every world hit
            assert (t["text"] == BLANK).all()
    t = termorc.render_layers_terminal((tw, wcam, wopts), None, None, None)
    want = ow.render(wcam, wopts, accum_mode=1)["text"]
    assert np.array_equal(t["text"].reshape(-1), want)
