"""GPU parity tests (run with `-m gpu` on an H100): the CUDA path, called through the C ABI,
against the oracle on identical Space / Camera / options.

Bar (BASELINE.json north_star: +-1 ULP per f32 channel, hit indices bit-exact).  What is asserted here is
stronger and leaves no slack for an ordering bug to hide in: hit indices, step counts, depths, **every ColorBuf
channel and every sRGB8 byte are bit-identical (0 ULP)** to the oracle evaluating f32::powf / f32::exp the way
the device does (correctly rounded: `orc.LIBM_CR`).  The only other difference between that oracle and the
reference on this host is glibc's powf / expf, which tests/test_oracle_libm.py bounds per call (<= 1 ULP, the
two modes agree on ~99 % of calls) and per image."""
import itertools
import json
import os

import numpy as np
import pytest

import aicb200
import orc
from aicb200 import (FOG_ABRUPT, FOG_COMPROMISE, FOG_NONE, FOG_PHYSICAL, LIGHT_COARSE, LIGHT_FLAT, LIGHT_LINEAR,
                     LIGHT_NONE, LIGHT_SMOOTHSTEP, TRANSPARENCY_SURFACE, TRANSPARENCY_THRESHOLD,
                     TRANSPARENCY_VOLUMETRIC, Block, Camera, GraphicsOptions, RtRenderer, Space, SpaceRaytracer,
                     Viewport, scenes)

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")



@pytest.fixture(autouse=True, scope="module")
def _oracle_rounds_once():
    """The oracle of this module evaluates powf / expf in f64 and rounds once, like the device."""
    prev = orc.get_libm()
    orc.set_libm(orc.LIBM_CR)
    yield
    orc.set_libm(prev)


def compare(gpu, ref, label=""):
    assert np.array_equal(gpu["hit"], ref["hit"]), f"{label}: hit records differ"
    assert np.array_equal(gpu["steps"], ref["steps"]), f"{label}: step counts differ"
    assert np.array_equal(gpu["depth"], ref["depth"]), f"{label}: depths differ"
    ulp = orc.ulp_diff(gpu["colorbuf"], ref["colorbuf"])
    assert ulp.max() == 0, f"{label}: ColorBuf max ulp {ulp.max()} at {np.argwhere(ulp > 0)[:4]}"
    return 0


def same_srgb8(img, ref, label=""):
    got = img.data.reshape(-1, 4)
    assert np.array_equal(got, ref["srgb8"]), f"{label}: {(got != ref['srgb8']).any(axis=1).sum()} sRGB8 pixels differ"


def render_both(space, cam, opts, shard=None):
    r = RtRenderer(cam)
    r.update(space)
    gpu = r.draw_colorbuf(shard=shard)
    img = r.draw(shard=shard)
    ref = orc.OracleScene(space).render(cam, opts, shard=shard)
    return gpu, img, ref


@pytest.fixture(scope="module")
def mixed():
    return scenes.small_mixed_scene(n=12, seed=7)


@pytest.mark.parametrize("transparency", [TRANSPARENCY_SURFACE, TRANSPARENCY_VOLUMETRIC, TRANSPARENCY_THRESHOLD])
@pytest.mark.parametrize("lighting", [LIGHT_NONE, LIGHT_FLAT, LIGHT_COARSE, LIGHT_LINEAR, LIGHT_SMOOTHSTEP])
@pytest.mark.parametrize("fog", [FOG_NONE, FOG_ABRUPT, FOG_COMPROMISE, FOG_PHYSICAL])
def test_option_matrix(mixed, transparency, lighting, fog):
    opts = GraphicsOptions(fog=fog, lighting_display=lighting, transparency=transparency, view_distance=40.0,
                           transparency_threshold=0.3)
    cam = scenes.standard_camera(mixed, opts, 96, 64)
    gpu, img, ref = render_both(mixed, cam, opts)
    compare(gpu, ref, f"t{transparency} l{lighting} f{fog}")
    assert gpu["info"].cubes_traced == ref["cubes_traced"] == int(ref["steps"].sum())
    same_srgb8(img, ref)
    assert img.info.cubes_traced == ref["cubes_traced"]


@pytest.mark.parametrize("direction", [(1, 0.6, 1), (-1, -0.3, 0.2), (0, 1, 0), (0, 0, -1), (1, 0, 0), (0.3, -1, -0.7)])
def test_camera_directions_and_inside(mixed, direction):
    """Axis-aligned views (zero direction components, ties) and a camera inside the Space (Face7::Within)."""
    opts = GraphicsOptions(view_distance=60.0)
    for scale in (1.0, 0.2):
        cam = scenes.standard_camera(mixed, opts, 64, 48, direction=direction, distance_scale=scale)
        gpu, img, ref = render_both(mixed, cam, opts)
        compare(gpu, ref, f"dir {direction} scale {scale}")


def test_antialiasing_and_debug_pixel_cost(mixed):
    for kw in (dict(antialiasing_always=True), dict(debug_pixel_cost=True),
               dict(antialiasing_always=True, transparency=TRANSPARENCY_SURFACE, fog=FOG_NONE, lighting_display=LIGHT_FLAT)):
        opts = GraphicsOptions(view_distance=40.0, **kw)
        cam = scenes.standard_camera(mixed, opts, 48, 32)
        gpu, img, ref = render_both(mixed, cam, opts)
        compare(gpu, ref, str(kw))
        same_srgb8(img, ref)


def test_premultiplied_f16_output(mixed):
    """raytrace_to_texture.rs:645-661: [f16(r * exposure), f16(g * exposure), f16(b * exposure), f16(alpha)] of
    ColorBuf::into_premultiplied_rgba.  Exact against the same conversion of the GPU's own ColorBuf and of the
    oracle's ColorBuf."""
    for kw in (dict(), dict(exposure=2.5), dict(antialiasing_always=True)):
        opts = GraphicsOptions(view_distance=40.0, **kw)
        cam = scenes.standard_camera(mixed, opts, 64, 48)
        r = RtRenderer(cam)
        r.update(mixed)
        got = r.draw_rgba16f().reshape(-1, 4)
        exposure = np.float32(cam.data.exposure)

        def convert(cb):
            alpha = np.clip(np.float32(1.0) - cb[:, 3], np.float32(0.0), np.float32(1.0))
            with np.errstate(over="ignore"):
                return np.stack([(cb[:, 0] * exposure), (cb[:, 1] * exposure), (cb[:, 2] * exposure), alpha], axis=1).astype(np.float16)

        own = convert(r.draw_colorbuf(want_depth=False, want_hit=False, want_steps=False)["colorbuf"])
        assert np.array_equal(got.view(np.uint16), own.view(np.uint16))
        ref = convert(orc.OracleScene(mixed).render(cam, opts)["colorbuf"])
        assert np.array_equal(got.view(np.uint16), ref.view(np.uint16))


def test_tone_mapping_and_exposure(mixed):
    for kw in (dict(tone_mapping=aicb200.TONE_REINHARD, maximum_intensity=1.0, exposure=2.0),
               dict(tone_mapping=aicb200.TONE_CLAMP, maximum_intensity=0.5, exposure=0.5)):
        opts = GraphicsOptions(view_distance=40.0, **kw)
        cam = scenes.standard_camera(mixed, opts, 48, 32)
        gpu, img, ref = render_both(mixed, cam, opts)
        same_srgb8(img, ref)


def test_no_light_volume_and_uniform_sky():
    space = scenes.small_mixed_scene(n=10, seed=3, with_light=False, octant_sky=False)
    for lighting in (LIGHT_FLAT, LIGHT_LINEAR):
        opts = GraphicsOptions(lighting_display=lighting, view_distance=50.0)
        cam = scenes.standard_camera(space, opts, 64, 48)
        gpu, img, ref = render_both(space, cam, opts)
        compare(gpu, ref, f"nolight l{lighting}")


def test_row_strip_shards_reassemble_the_frame(mixed):
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(mixed, opts, 64, 50)
    r = RtRenderer(cam)
    r.update(mixed)
    full = r.draw().data
    for count in (2, 3):
        out = np.zeros_like(full)
        for index in range(count):
            part = r.draw(shard=(16, index, count)).data
            rows = [y for y in range(50) if (y // 16) % count == index]
            assert part.shape[0] == len(rows)
            out[rows] = part
            ref = orc.OracleScene(mixed).render(cam, opts, shard=(16, index, count))
            assert np.array_equal(part.reshape(-1, 4), ref["srgb8"])
        assert np.array_equal(out, full), "N-shard frame differs from the 1-shard frame"


def test_explicit_rays_including_degenerate(mixed):
    """SpaceRaytracer::trace_ray on hand-made rays: zero / NaN / huge directions, axis-aligned, grazing."""
    rng = np.random.default_rng(5)
    rays = []
    lo = np.array(mixed.lower, dtype=np.float64)
    size = np.array(mixed.size, dtype=np.float64)
    for _ in range(2000):
        o = lo + rng.uniform(-0.5, 1.5, 3) * size
        d = rng.normal(size=3) * 10.0 ** rng.uniform(-2, 2)
        rays.append(np.concatenate([o, d]))
    c = lo + size / 2
    rays += [np.concatenate([c, [0, 0, 0]]), np.concatenate([c, [np.nan, 1, 0]]), np.concatenate([c, [1e200, 0, 0]]),
             np.concatenate([c, [1, 0, 0]]), np.concatenate([c, [0, -1, 0]]), np.concatenate([c, [0, 0, 1e-30]]),
             np.concatenate([lo - 1.0, [1, 1, 1]]), np.concatenate([lo + [0.0, 0.0, -3.0], [0, 0, 2.0]]),
             np.concatenate([lo + size + 5.0, [-1, -1, -1]]), np.concatenate([[1e12, 0, 0], [-1, 0, 0]])]
    rays = np.array(rays)
    for opts in (GraphicsOptions(view_distance=50.0),
                 GraphicsOptions(transparency=TRANSPARENCY_SURFACE, fog=FOG_NONE, lighting_display=LIGHT_NONE)):
        for include_sky in (True, False):
            rt = SpaceRaytracer(mixed, opts)
            gpu = rt.trace_rays(rays, include_sky=include_sky, want_depth=True, want_hit=True, want_steps=True)
            ref = orc.OracleScene(mixed).trace_rays(rays, opts, include_sky=include_sky)
            compare(gpu, ref, f"explicit rays sky={include_sky}")


def test_reference_kat_scenes_on_gpu():
    """The surface.rs known-answer scenes (surface.rs:541-835) through the CUDA path: hit, depth, steps."""
    idx = np.ones((4, 4, 4), dtype=np.uint16)
    idx[1:, 2:, :] = 0
    pal = np.zeros((2, 8), dtype=np.float32)
    pal[1, :4] = (1, 1, 0, 1)
    slab = Block(resolution=4, indices=idx, palette=pal)
    ids = np.array([0, 1, 2], dtype=np.uint16).reshape(1, 3, 1)
    space = Space((0, 0, 0), ids, [Block.air(), Block(color=(1, 0, 0, 1)), slab])
    opts = GraphicsOptions.unaltered_colors()
    opts.transparency = TRANSPARENCY_SURFACE
    rt = SpaceRaytracer(space, opts)
    got = rt.trace_rays([[0.25, -0.5, 0.25, 0.0, 1.0, 0.0]], include_sky=False, want_depth=True, want_hit=True, want_steps=True)
    assert got["depth"][0] == 1.5
    assert list(got["hit"][0]) == [0, 1, 0, 0, 0, 0, 1, aicb200.abi.FACE_NY]
    assert list(got["colorbuf"][0]) == [1.0, 0.0, 0.0, 0.0]
    # Invisible{0.5}, EnterSurface (opaque) -> the next count sees opacity and stops: 3 steps
    assert got["steps"][0] == 3
    ref = orc.OracleScene(space).trace_rays([[0.25, -0.5, 0.25, 0.0, 1.0, 0.0]], opts, include_sky=False)
    assert ref["steps"][0] == 3


def _ascii_from_gpu(space, direction, chars):
    opts = GraphicsOptions()
    cam = Camera(opts, Viewport((40.0, 40.0), (80, 40)))
    center = [space.lower[a] + space.size[a] / 2.0 for a in range(3)]
    cam.look_at_y_up(aicb200.eye_for_look_at(space.lower, space.size, direction), center)
    rays = []
    for ych in range(40):
        y = -((ych + 0.5) / 40.0 * 2.0 - 1.0)
        for xch in range(80):
            rays.append(cam.project_ndc_into_world((xch + 0.5) / 80.0 * 2.0 - 1.0, y))
    got = SpaceRaytracer(space, opts).trace_rays(np.array(rays), want_hit=True, want_steps=True)
    rows = []
    for ych in range(40):
        row = ""
        for xch in range(80):
            i = ych * 80 + xch
            h = got["hit"][i]
            if h[7] >= 0:
                bid = int(space.block_ids[h[0] - space.lower[0], h[1] - space.lower[1], h[2] - space.lower[2]])
                row += chars[bid]
            else:
                row += " " if got["steps"][i] > 0 else "."
        rows.append(row)
    return rows


def test_text_golden_images_on_gpu():
    """raytracer/text.rs:196-258, 265-341: the reference's 80x40 ASCII hit-identity images from the GPU hit buffer."""
    golden = json.load(open(os.path.join(GOLDEN, "text_images.json")))
    ids = np.array([1, 2, 3], dtype=np.uint16).reshape(3, 1, 1)
    grey = lambda i, n: (i / (n - 1),) * 3 + (1.0,) if n > 1 else (0.5, 0.5, 0.5, 1.0)
    space = Space((0, 0, 0), ids, [Block.air()] + [Block(color=grey(i, 3)) for i in range(3)])
    assert _ascii_from_gpu(space, (1.0, 1.0, 1.0), {1: "0", 2: "1", 3: "2"}) == golden["print_space_test"]
    idx = np.zeros((4, 2, 4), dtype=np.uint16)
    pal = np.zeros((1, 8), dtype=np.float32)
    pal[0, :4] = (1, 1, 1, 1)
    partial = Block(resolution=4, indices=idx, palette=pal)
    space = Space((0, 0, 0), np.array([1, 2], dtype=np.uint16).reshape(2, 1, 1),
                  [Block.air(), Block(color=grey(0, 1)), partial])
    assert _ascii_from_gpu(space, (1.0, 1.0, 1.0), {1: "0", 2: "P"}) == golden["partial_voxels"]


def test_golden_png_emission_on_gpu():
    """test-renderers `emission` case (cases/src/lib.rs:297-348, threshold 1) rendered by the CUDA path."""
    from test_golden_images import check_threshold, common_camera, golden
    from aicb200 import srgb8_to_linear
    c200 = srgb8_to_linear((200, 0, 0))[0]
    pal = np.zeros((3, 8), dtype=np.float32)
    pal[0, :4] = (1, 1, 1, 1)
    pal[1, :4] = (c200, 0, 0, 1); pal[1, 4:7] = (0, c200, 0)
    pal[2, :4] = (0, 0, 0, 1); pal[2, 4:7] = (0, c200, 0)
    idx = np.zeros((4, 4, 4), dtype=np.uint16)
    idx[1, 2, :] = 1
    idx[2, 1, :] = 2
    space = Space((0, 0, 0), np.ones((1, 1, 1), dtype=np.uint16), [Block.air(), Block(resolution=4, indices=idx, palette=pal)],
                  sky_colors=[(0.5, 0.5, 0.5)])
    opts = GraphicsOptions.unaltered_colors()
    r = RtRenderer(common_camera(opts))
    r.update(space)
    check_threshold(r.draw().data, golden("emission-all"), [(1, 128 * 96)])


def test_config_c0_cpu_reference_case():
    """BASELINE configs[0]: 32^3 solid/empty res-1, 256x256 — full size."""
    space = scenes.config_c0()
    opts = GraphicsOptions.unaltered_colors()
    cam = scenes.standard_camera(space, opts, 256, 256)
    gpu, img, ref = render_both(space, cam, opts)
    compare(gpu, ref, "C0")
    assert np.array_equal(img.data.reshape(-1, 4), ref["srgb8"])


def test_config_c1_reduced_recursive_blocks():
    """BASELINE configs[1] shape at a size the oracle finishes in seconds: 32^3, res-16 blocks, 320x180."""
    space = scenes.config_c1(n=32, n_voxel_blocks=24, with_light=True)
    for opts in (GraphicsOptions.unaltered_colors(),
                 GraphicsOptions(lighting_display=LIGHT_FLAT, fog=FOG_NONE, view_distance=128.0),
                 GraphicsOptions(view_distance=128.0)):
        cam = scenes.standard_camera(space, opts, 320, 180)
        gpu, img, ref = render_both(space, cam, opts)
        compare(gpu, ref, "C1 reduced")
        same_srgb8(img, ref)


def test_config_c2_reduced_deep_transparency():
    """BASELINE configs[2] shape reduced: 48^3 mixed transparent, both Volumetric and Surface; many rays
    run into the 1000-step cap / the opacity cut-off."""
    space = scenes.config_c2(n=48, n_voxel_blocks=8, with_light=True)
    for transparency in (TRANSPARENCY_VOLUMETRIC, TRANSPARENCY_SURFACE):
        opts = GraphicsOptions.unaltered_colors()
        opts.transparency = transparency
        opts.view_distance = 192.0
        cam = scenes.standard_camera(space, opts, 240, 135)
        gpu, img, ref = render_both(space, cam, opts)
        compare(gpu, ref, f"C2 reduced t{transparency}")
    opts = GraphicsOptions(view_distance=192.0)
    cam = scenes.standard_camera(space, opts, 240, 135)
    gpu, img, ref = render_both(space, cam, opts)
    compare(gpu, ref, "C2 reduced default options")


def test_step_cap_is_reached_and_counted():
    """sr.rs:639-652: a long empty Space makes rays stop at exactly 1001 counted steps."""
    n = 400
    ids = np.zeros((n, 4, 4), dtype=np.uint16)
    space = Space((0, 0, 0), ids, [Block.air(), Block(color=(1, 1, 1, 1))])
    opts = GraphicsOptions.unaltered_colors()
    rays = np.array([[-0.5, 1.3, 2.2, 1.0, 0.004, 0.003], [0.5, 0.5, 0.5, 1.0, 0.9, 0.0]])
    gpu = SpaceRaytracer(space, opts).trace_rays(rays, want_steps=True, want_hit=True, want_depth=True)
    ref = orc.OracleScene(space).trace_rays(rays, opts)
    compare(gpu, ref, "step cap")
    # a res-16 filled space hits the cap: 16 voxel steps + events per cube
    blk = scenes.make_voxel_block(3, resolution=16, alpha=0.0005, fill_mask=1, partial_bounds=False)
    ids = np.ones((80, 2, 2), dtype=np.uint16)
    space = Space((0, 0, 0), ids, [Block.air(), blk])
    for transparency in (TRANSPARENCY_SURFACE, TRANSPARENCY_VOLUMETRIC):
        opts = GraphicsOptions.unaltered_colors()
        opts.transparency = transparency
        rays = np.array([[-0.5, 1.01, 0.99, 1.0, 0.001, 0.002]])
        gpu = SpaceRaytracer(space, opts).trace_rays(rays, want_steps=True, want_hit=True, want_depth=True)
        ref = orc.OracleScene(space).trace_rays(rays, opts)
        assert ref["steps"][0] == 1001
        compare(gpu, ref, "step cap res16")


def test_zero_and_prime_viewports(mixed):
    """cases viewport_zero / viewport_prime (cases/src/lib.rs:1167-1237): empty and odd-sized frames."""
    opts = GraphicsOptions(view_distance=40.0)
    for size in ((0, 0), (0, 5), (7, 0), (127, 61), (1, 1), (9, 5)):
        cam = scenes.standard_camera(mixed, opts, *size) if size[0] and size[1] else Camera(opts, Viewport((1.0, 1.0), size))
        r = RtRenderer(cam)
        r.update(mixed)
        img = r.draw()
        assert img.data.size == size[0] * size[1] * 4
        if size[0] and size[1]:
            ref = orc.OracleScene(mixed).render(cam, opts)
            same_srgb8(img, ref)


def test_buffer_length_mismatch_is_an_error(mixed):
    """renderer.rs:193-197 panics on a wrong output length; the C ABI returns AICB_ERR_INVALID."""
    import ctypes as C
    opts = GraphicsOptions()
    cam = scenes.standard_camera(mixed, opts, 16, 16)
    rt = SpaceRaytracer(mixed, opts)
    out = np.zeros((10, 4), dtype=np.uint8)
    o = opts.to_abi()
    st = aicb200.load_library().aicb_render_srgb8(rt.handle, C.byref(cam.data), C.byref(o), None, out.ctypes.data, 10, None)
    assert st == aicb200.abi.ERR_INVALID
    assert b"does not match" in aicb200.load_library().aicb_last_error()


def test_incremental_cube_update_equals_fresh_snapshot(mixed):
    """updating.rs:295-337: applying SpaceChange deltas == rebuilding the SpaceRaytracer."""
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(mixed, opts, 64, 48)
    r = RtRenderer(cam)
    r.update(mixed)
    rng = np.random.default_rng(2)
    cubes = np.stack([rng.integers(0, mixed.size[a], 50) + mixed.lower[a] for a in range(3)], axis=1)
    new_ids = rng.integers(0, len(mixed.blocks), 50).astype(np.uint16)
    new_light = rng.integers(0, 255, (50, 4)).astype(np.uint8)
    new_light[:, 3] = 255
    cubes[40:] = cubes[:10]   # cubes named twice in one batch keep their last value
    r.rt.update_cubes(cubes, new_ids, new_light)
    ids2 = mixed.block_ids.copy()
    light2 = mixed.light.copy()
    for c, i, l in zip(cubes, new_ids, new_light):
        p = tuple(c - np.array(mixed.lower))
        ids2[p] = i
        light2[p] = l
    fresh = Space(mixed.lower, ids2, mixed.blocks, light=light2, sky_colors=mixed.sky_colors)
    r2 = RtRenderer(cam)
    r2.update(fresh)
    assert np.array_equal(r.draw().data, r2.draw().data)


def test_block_definition_update_equals_fresh_snapshot(mixed):
    """updating.rs:128-150: replacing block definitions (SpaceChange::BlockEvaluation) == rebuilding the
    SpaceRaytracer.  Covers a colour change (kind unchanged), single voxel -> voxel brick (kind change: cells
    re-encoded), and a block that becomes invisible."""
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(mixed, opts, 64, 48)
    r = RtRenderer(cam)
    r.update(mixed)
    blocks = list(mixed.blocks)
    singles = [i for i, b in enumerate(blocks) if i and b.indices is None and not b.is_air]
    voxels = [i for i, b in enumerate(blocks) if b.indices is not None]
    assert len(singles) >= 2 and voxels
    new = {singles[0]: Block(color=(0.2, 0.9, 0.4, 1.0)),                          # recoloured
           singles[1]: scenes.make_voxel_block(11, resolution=8, alpha=0.5),      # single voxel -> brick
           voxels[0]: Block(color=(0.0, 0.0, 0.0, 0.0))}                          # brick -> invisible single voxel
    r.rt.update_blocks(list(new.keys()), list(new.values()))
    for i, b in new.items():
        blocks[i] = b
    fresh = Space(mixed.lower, mixed.block_ids, blocks, light=mixed.light, sky_colors=mixed.sky_colors)
    r2 = RtRenderer(cam)
    r2.update(fresh)
    assert np.array_equal(r.draw().data, r2.draw().data)
    a, b = r.draw_colorbuf(), r2.draw_colorbuf()
    assert np.array_equal(a["hit"], b["hit"]) and np.array_equal(a["steps"], b["steps"])


def test_full_size_1080p_properties():
    """BASELINE configs[1] at full size (128^3 res-16, 1920x1080): size-independent properties —
    determinism, cubes_traced == sum of per-pixel steps, shard union == frame — plus bit-level
    parity with the oracle on a band of rows."""
    space = scenes.config_c1(n=128)
    opts = GraphicsOptions.unaltered_colors()
    opts.view_distance = 512.0
    cam = scenes.standard_camera(space, opts, 1920, 1080)
    r = RtRenderer(cam)
    r.update(space)
    a = r.draw()
    b = r.draw()
    assert np.array_equal(a.data, b.data), "render is not deterministic"
    aux = r.draw_colorbuf(want_depth=False, want_hit=False)
    assert aux["info"].cubes_traced == int(aux["steps"].astype(np.int64).sum()) == a.info.cubes_traced
    out = np.zeros_like(a.data)
    for index in range(4):
        rows = [y for y in range(1080) if (y // 16) % 4 == index]
        out[rows] = r.draw(shard=(16, index, 4)).data
    assert np.array_equal(out, a.data)
    band = orc.OracleScene(space).render_rows(cam, opts, 536, 544, want_colorbuf=True)
    assert np.array_equal(a.data[536:544].reshape(-1, 4), band["srgb8"])
    assert orc.max_ulp_diff(aux["colorbuf"].reshape(1080, 1920, 4)[536:544].reshape(-1, 4), band["colorbuf"]) == 0


def test_full_size_bench_frame_c2():
    """The frame bench.py times (BASELINE configs[2]: 256^3 mixed transparent Space with a light volume, 1920x1080,
    GraphicsOptions::default() with view_distance 1024) at full size: determinism, cubes_traced == sum of the
    per-pixel steps, the union of 8 interleaved 16-row shards == the frame, and parity with the oracle on rows spread
    over the whole frame (sRGB8, ColorBuf and cubes_traced bit-identical)."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    import bench
    space, opts, w, h, _ = bench.make_workload("c2")
    cam = scenes.standard_camera(space, opts, w, h)
    r = RtRenderer(cam)
    r.update(space)
    a = r.draw()
    b = r.draw()
    assert np.array_equal(a.data, b.data), "render is not deterministic"
    aux = r.draw_colorbuf(want_depth=False, want_hit=False)
    assert aux["info"].cubes_traced == int(aux["steps"].astype(np.int64).sum()) == a.info.cubes_traced
    out = np.zeros_like(a.data)
    for index in range(8):
        rows = [y for y in range(h) if (y // 16) % 8 == index]
        out[rows] = r.draw(shard=(16, index, 8)).data
    assert np.array_equal(out, a.data)
    rows = [int((i + 0.5) * h / 24) for i in range(24)]
    ref = orc.render_rowlist(orc.OracleScene(space), cam, opts, rows, want_colorbuf=True)
    got = a.data[rows].reshape(-1, 4)
    assert np.array_equal(got, ref["srgb8"])
    cb = aux["colorbuf"].reshape(h, w, 4)[rows].reshape(-1, 4)
    ulp = orc.ulp_diff(cb, ref["colorbuf"])
    assert ulp.max() == 0, f"max ulp {ulp.max()}, {(ulp > 0).sum()} channels differ"
    assert int(aux["steps"].reshape(h, w)[rows].astype(np.int64).sum()) == ref["cubes_traced"]


def test_device_group_frame_equals_single_device_frame(mixed):
    """csrc/group.cu (aicb_group_*): several GPUs from one process — interleaved 16-row strips stored straight into
    device 0's frame.  Here the same device is named two and three times: the delivered frame and the summed
    RaytraceInfo must equal the one-device render's (renderer.rs:555: the info is a sum over the pixels)."""
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(mixed, opts, 96, 70)
    r = RtRenderer(cam)
    r.update(mixed)
    alone = r.draw()
    for devices in ([0, 0], [0, 0, 0]):
        g = aicb200.DeviceGroup(devices)
        g.update(mixed)
        img = g.draw(cam, opts)
        assert np.array_equal(img.data, alone.data)
        assert img.info.cubes_traced == alone.info.cubes_traced
        again = g.draw(cam, opts)
        assert np.array_equal(again.data, alone.data)
        g.close()


def test_print_space_through_the_text_entry():
    """raytracer/text.rs:196-258, 265-341 through aicb_render_text (CharacterBuf per pixel) — the reference's two
    80x40 golden images, character for character; and the same states as the oracle's CharacterBuf accumulator."""
    golden = json.load(open(os.path.join(GOLDEN, "text_images.json")))
    ids = np.array([1, 2, 3], dtype=np.uint16).reshape(3, 1, 1)
    grey = lambda i, n: (i / (n - 1),) * 3 + (1.0,) if n > 1 else (0.5, 0.5, 0.5, 1.0)
    space = Space((0, 0, 0), ids, [Block.air()] + [Block(color=grey(i, 3)) for i in range(3)])
    assert aicb200.print_space(space, (1.0, 1.0, 1.0), {1: "0", 2: "1", 3: "2"}) == golden["print_space_test"]
    idx = np.zeros((4, 2, 4), dtype=np.uint16)
    pal = np.zeros((1, 8), dtype=np.float32)
    pal[0, :4] = (1, 1, 1, 1)
    partial = Block(resolution=4, indices=idx, palette=pal)
    space = Space((0, 0, 0), np.array([1, 2], dtype=np.uint16).reshape(2, 1, 1),
                  [Block.air(), Block(color=grey(0, 1)), partial])
    assert aicb200.print_space(space, (1.0, 1.0, 1.0), {1: "0", 2: "P"}) == golden["partial_voxels"]


def test_text_output_equals_oracle_character_buf(mixed):
    import ctypes as C
    for kw in (dict(), dict(antialiasing_always=True), dict(transparency=TRANSPARENCY_SURFACE)):
        opts = GraphicsOptions(view_distance=40.0, **kw)
        cam = scenes.standard_camera(mixed, opts, 72, 40)
        rt = SpaceRaytracer(mixed, opts)
        out = np.zeros(72 * 40, dtype=np.int32)
        o = opts.to_abi(True)
        st = aicb200.load_library().aicb_render_text(rt.handle, C.byref(cam.data), C.byref(o), out.ctypes.data, out.size, None)
        assert st == 0
        ref = orc.OracleScene(mixed).render(cam, opts, accum_mode=1)["text"]
        ref = np.where(ref == -4, -3, ref)   # (no other exception hit reaches a CharacterBuf in these scenes)
        assert np.array_equal(out, ref), f"{kw}: {np.argwhere(out != ref)[:5]}"


def test_orthographic_render_equals_oracle_on_the_same_rays(mixed):
    """raytracer/ortho.rs:30-84: five axis-aligned pixel-perfect views.  The image must equal the oracle tracing the
    reference's rays (OrthoCamera::project_pixel_into_world, ortho.rs:209-297) one by one, and the layout must be
    MultiOrthoCamera's (:143-199)."""
    res = 4
    rt = SpaceRaytracer(mixed, GraphicsOptions.unaltered_colors())
    img = aicb200.render_orthographic(rt, res)
    sx, sy, sz = (mixed.size[a] * res for a in range(3))
    assert img.size == (sz + sx + sz + 2, sz + sy + sz + 2)
    lb = np.array(mixed.lower, dtype=np.float64)
    ub = lb + np.array(mixed.size, dtype=np.float64)
    views = [  # (image origin, size, corner, image right axis, image down axis, ray direction)
        ((sz + 1, 0), (sx, sz), (lb[0], ub[1], lb[2]), (1, 0, 0), (0, 0, 1), (0, -1, 0)),             # top
        ((0, sz + 1), (sz, sy), (lb[0], ub[1], lb[2]), (0, 0, 1), (0, -1, 0), (1, 0, 0)),             # left
        ((sz + 1, sz + 1), (sx, sy), (lb[0], ub[1], ub[2]), (1, 0, 0), (0, -1, 0), (0, 0, -1)),       # front
        ((sz + sx + 2, sz + 1), (sz, sy), (ub[0], ub[1], ub[2]), (0, 0, -1), (0, -1, 0), (-1, 0, 0)),  # right
        ((sz + 1, sz + sy + 2), (sx, sz), (lb[0], lb[1], ub[2]), (1, 0, 0), (0, 0, -1), (0, 1, 0)),   # bottom
    ]
    expect = np.zeros((img.size[1], img.size[0], 4), dtype=np.uint8)
    osc = orc.OracleScene(mixed)
    for (ox, oy), (w, h), corner, right, down, d in views:
        px, py = np.meshgrid(np.arange(w), np.arange(h))
        u = (px.ravel() + 0.5) / res
        v = (py.ravel() + 0.5) / res
        o = np.array(corner)[None, :] + u[:, None] * np.array(right, dtype=np.float64)[None, :] + v[:, None] * np.array(down, dtype=np.float64)[None, :]
        rays = np.concatenate([o, np.broadcast_to(np.array(d, dtype=np.float64), o.shape)], axis=1)
        ref = osc.trace_rays(rays, GraphicsOptions.unaltered_colors(), include_sky=True)
        expect[oy:oy + h, ox:ox + w] = orc.colorbuf_to_srgb8(ref["colorbuf"]).reshape(h, w, 4)
    assert np.array_equal(img.data, expect), f"{(img.data != expect).any(axis=2).sum()} pixels differ"
    assert (img.data[sz, :, 3] == 0).all() and (img.data[:, sz, 3] == 0).all()   # the gaps are transparent


def test_layers_ui_backdrop_world_and_no_world(mixed):
    """RtScene::trace_ray_through_layers (renderer.rs:454-478) against the oracle: a UI Space in front (own camera,
    no sky), a backdrop colour, the world continuing in the same accumulator; without a world, NO_WORLD_TO_SHOW."""
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    nw = aicb200.srgb8_to_linear((0xBC, 0xBC, 0xBC)) + (1.0,)
    for aa in (False, True):
        wopts = GraphicsOptions(view_distance=40.0, antialiasing_always=aa)
        uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT)
        wcam = scenes.standard_camera(mixed, wopts, 64, 48)
        ucam = scenes.standard_camera(ui_space, uopts, 64, 48, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
        wrt = SpaceRaytracer(mixed, wopts)
        urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
        wo, uo = orc.OracleScene(mixed), orc.OracleScene(ui_space)
        cases = [
            dict(world=True, ui=True, backdrop=(0.1, 0.3, 0.6, 0.5)),
            dict(world=True, ui=True, backdrop=None),
            dict(world=True, ui=False, backdrop=(0.9, 0.2, 0.1, 0.25)),
            dict(world=False, ui=True, backdrop=(0.0, 0.5, 0.0, 0.3)),
            dict(world=False, ui=True, backdrop=None),
        ]
        for c in cases:
            gw = (wrt, wcam, wopts) if c["world"] else None
            gu = (urt, ucam, uopts) if c["ui"] else None
            if not c["world"]:   # the lead layer's options choose the sample points
                uopts.antialiasing_always = aa
            got = aicb200.render_layers(gw, gu, c["backdrop"], nw)
            ref = orc.render_layers((wo, wcam, wopts) if c["world"] else None, (uo, ucam, uopts) if c["ui"] else None,
                                    c["backdrop"], nw)
            uopts.antialiasing_always = False
            assert np.array_equal(got.data.reshape(-1, 4), ref["srgb8"]), f"aa={aa} {c}: {(got.data.reshape(-1, 4) != ref['srgb8']).any(axis=1).sum()} pixels differ"
            assert got.info.cubes_traced == ref["cubes_traced"], f"aa={aa} {c}"


def test_full_size_c3_4k_properties():
    """BASELINE configs[3] at full size (256^3 res-16 blocks, 3840x2160): determinism, cubes_traced == sum of the
    per-pixel steps, the union of 8 interleaved 16-row shards == the frame (what 8 GPUs deliver), and bit-level parity
    with the oracle on rows spread over the frame."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    import bench
    space, opts, w, h, _ = bench.make_workload("c3")
    cam = scenes.standard_camera(space, opts, w, h)
    r = RtRenderer(cam)
    r.update(space)
    a = r.draw()
    b = r.draw()
    assert np.array_equal(a.data, b.data), "render is not deterministic"
    aux = r.draw_colorbuf(want_depth=False, want_hit=False)
    assert aux["info"].cubes_traced == int(aux["steps"].astype(np.int64).sum()) == a.info.cubes_traced
    out = np.zeros_like(a.data)
    for index in range(8):
        rows = [y for y in range(h) if (y // 16) % 8 == index]
        out[rows] = r.draw(shard=(16, index, 8)).data
    assert np.array_equal(out, a.data)
    rows = [int((i + 0.5) * h / 12) for i in range(12)]
    ref = orc.render_rowlist(orc.OracleScene(space), cam, opts, rows, want_colorbuf=True)
    assert np.array_equal(a.data[rows].reshape(-1, 4), ref["srgb8"])
    cb = aux["colorbuf"].reshape(h, w, 4)[rows].reshape(-1, 4)
    assert orc.max_ulp_diff(cb, ref["colorbuf"]) == 0
    assert int(aux["steps"].reshape(h, w)[rows].astype(np.int64).sum()) == ref["cubes_traced"]


def test_wide_cells_more_than_16384_blocks():
    """A Space whose palette has more than 16384 block indices (BlockIndex is u16, space.rs): the cells are stored as
    u32 (id | kind << 16) and the marching kernel runs its WIDE instantiation.  Parity on every output, incl. the
    CharacterBuf block indices and a cube delta."""
    import ctypes as C
    n = 20
    n_blocks = 17000
    rng = np.random.default_rng(17)
    cols = rng.uniform(0.05, 1.0, (n_blocks, 3))
    blocks = [Block.air()]
    for i in range(1, n_blocks):
        if i in (16500, 16600, 16700):
            blocks.append(scenes.make_voxel_block(i, resolution=8, alpha=(1.0, 0.5, 0.25)[(i // 100) % 3]))
        elif i % 7 == 0:
            blocks.append(Block(color=(cols[i, 0], cols[i, 1], cols[i, 2], 0.5)))
        else:
            blocks.append(Block(color=(cols[i, 0], cols[i, 1], cols[i, 2], 1.0)))
    h = scenes.grid_hash(23, (n, n, n))
    pick = (h >> np.uint64(8)) % np.uint64(n_blocks)
    special = np.array([16500, 16600, 16700], dtype=np.uint64)
    pick = np.where((h >> np.uint64(40)) % np.uint64(5) == 0, special[(h >> np.uint64(48)) % np.uint64(3)], pick)
    ids = np.where((h & np.uint64(7)) < 2, pick, 0).astype(np.uint16)
    assert ids.max() > 16384
    space = Space((-4, 0, 3), ids, blocks, light=scenes.noise_light(5, ids, blocks), sky_colors=scenes.OCTANT_SKY)
    for opts in (GraphicsOptions(view_distance=80.0),
                 GraphicsOptions(view_distance=80.0, transparency=TRANSPARENCY_SURFACE, lighting_display=LIGHT_FLAT)):
        cam = scenes.standard_camera(space, opts, 96, 64)
        gpu, img, ref = render_both(space, cam, opts)
        compare(gpu, ref, "wide cells")
        same_srgb8(img, ref)
        assert gpu["info"].cubes_traced == ref["cubes_traced"]
    opts = GraphicsOptions(view_distance=80.0)
    cam = scenes.standard_camera(space, opts, 72, 40)
    rt = SpaceRaytracer(space, opts)
    out = np.zeros(72 * 40, dtype=np.int32)
    o = opts.to_abi(True)
    assert aicb200.load_library().aicb_render_text(rt.handle, C.byref(cam.data), C.byref(o), out.ctypes.data, out.size, None) == 0
    ref = orc.OracleScene(space).render(cam, opts, accum_mode=1)["text"]
    assert np.array_equal(out, np.where(ref == -4, -3, ref))
    assert out.max() > 16384
    # SpaceChange::CubeBlock deltas on a wide scene == a fresh snapshot
    cubes = np.stack([rng.integers(0, n, 40) + space.lower[a] for a in range(3)], axis=1)
    new_ids = rng.integers(16380, 16990, 40).astype(np.uint16)
    r = RtRenderer(cam)
    r.update(space)
    r.rt.update_cubes(cubes, new_ids, None)
    ids2 = ids.copy()
    for c, i in zip(cubes, new_ids):
        ids2[tuple(c - np.array(space.lower))] = i
    r2 = RtRenderer(cam)
    r2.update(Space(space.lower, ids2, blocks, light=space.light, sky_colors=space.sky_colors))
    assert np.array_equal(r.draw().data, r2.draw().data)


# ---- LightingOption::Bounce (surface.rs:113-166) ------------------------------------------------------------------
@pytest.mark.parametrize("transparency", [TRANSPARENCY_SURFACE, TRANSPARENCY_VOLUMETRIC, TRANSPARENCY_THRESHOLD])
@pytest.mark.parametrize("samples,fog", [(1, FOG_NONE), (3, FOG_ABRUPT), (2, FOG_PHYSICAL)])
def test_bounce_lighting(mixed, transparency, samples, fog):
    """Secondary Lambertian rays from every fully opaque surface a ray ends on: ColorBuf, hits, per-pixel step counts
    (primary + secondary, sr.rs:689-692) and sRGB8 bit-identical to the oracle — same RNG stream per ray (xoshiro256++
    seeded from the direction's bits), same rejection sampling, same summation order."""
    opts = GraphicsOptions(fog=fog, lighting_display=aicb200.LIGHT_BOUNCE, bounce_samples=samples,
                           transparency=transparency, view_distance=40.0, transparency_threshold=0.3)
    cam = scenes.standard_camera(mixed, opts, 96, 64)
    gpu, img, ref = render_both(mixed, cam, opts)
    compare(gpu, ref, f"bounce t{transparency} s{samples} f{fog}")
    assert gpu["info"].cubes_traced == ref["cubes_traced"] == int(ref["steps"].sum())
    same_srgb8(img, ref)
    # it is not Flat lighting in disguise
    flat = orc.OracleScene(mixed).render(cam, GraphicsOptions(fog=fog, lighting_display=LIGHT_FLAT, transparency=transparency,
                                                              view_distance=40.0, transparency_threshold=0.3))
    assert not np.array_equal(flat["colorbuf"], ref["colorbuf"])
    assert ref["cubes_traced"] > flat["cubes_traced"]


def test_bounce_lighting_variants(mixed):
    """Antialiasing (4 rays per pixel, each with its own RNG), debug_pixel_cost (secondary rays carry the override too),
    a camera inside the Space, a sharded frame, and explicit rays through aicb_trace_rays."""
    base = dict(lighting_display=aicb200.LIGHT_BOUNCE, bounce_samples=2, view_distance=40.0)
    for kw in (dict(antialiasing_always=True), dict(debug_pixel_cost=True), dict(fog=FOG_COMPROMISE)):
        opts = GraphicsOptions(**base, **kw)
        cam = scenes.standard_camera(mixed, opts, 48, 32)
        gpu, img, ref = render_both(mixed, cam, opts)
        compare(gpu, ref, str(kw))
        same_srgb8(img, ref)
    opts = GraphicsOptions(**base)
    cam = scenes.standard_camera(mixed, opts, 64, 48, direction=(0.3, -1, -0.7), distance_scale=0.2)
    gpu, img, ref = render_both(mixed, cam, opts)
    compare(gpu, ref, "inside")
    cam = scenes.standard_camera(mixed, opts, 64, 48)
    gpu, img, ref = render_both(mixed, cam, opts, shard=(4, 1, 3))
    compare(gpu, ref, "shard")
    rng = np.random.default_rng(5)
    lo = np.array(mixed.lower, dtype=np.float64)
    size = np.array(mixed.size, dtype=np.float64)
    origin = lo + size * rng.uniform(-0.5, 1.5, (500, 3))
    target = lo + size * rng.uniform(0.1, 0.9, (500, 3))
    od = np.concatenate([origin, target - origin], axis=1)
    rt = SpaceRaytracer(mixed, opts)
    got = rt.trace_rays(od, want_steps=True)
    want = orc.OracleScene(mixed).trace_rays(od, opts)
    assert orc.ulp_diff(got["colorbuf"], want["colorbuf"]).max() == 0
    assert np.array_equal(got["steps"], want["steps"])


def test_bounce_needs_a_sample_count(mixed):
    opts = GraphicsOptions(lighting_display=aicb200.LIGHT_BOUNCE, bounce_samples=0, view_distance=40.0)
    cam = scenes.standard_camera(mixed, opts, 16, 16)
    r = RtRenderer(cam)
    r.update(mixed)
    with pytest.raises(aicb200.AicbError):
        r.draw()


def test_bounce_voxel_blocks():
    """Recursive blocks: the bounce starts from the intersection point on a voxel face (surface.rs:406-407)."""
    space = scenes.config_c1(n=12, seed=5, n_voxel_blocks=8, with_light=True, resolution=8)
    opts = GraphicsOptions(lighting_display=aicb200.LIGHT_BOUNCE, bounce_samples=2, view_distance=60.0)
    cam = scenes.standard_camera(space, opts, 80, 60)
    gpu, img, ref = render_both(space, cam, opts)
    compare(gpu, ref, "voxel blocks")
    same_srgb8(img, ref)
    assert gpu["info"].cubes_traced == ref["cubes_traced"]


def test_bench_dump_outputs_is_the_timed_frame(tmp_path):
    """bench.py --dump-outputs writes the sRGB8 frame of the last timed step: the frame a plain render of the same
    workload gives, and the same in two runs."""
    import subprocess
    import sys
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    sys.path.insert(0, root)
    import bench
    outs = []
    for k in range(2):
        out = tmp_path / f"run{k}"
        r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--workload", "c0", "--steps", str(2 + k),
                            "--warmup", "1", "--cpu-seconds", "0.5", "--dump-outputs", str(out)],
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        assert json.loads(r.stdout.strip().splitlines()[-1])["steps"] == 2 + k
        outs.append(np.load(out / "srgb8.npy"))
    assert outs[0].dtype == np.float32
    assert np.array_equal(outs[0], outs[1])
    space, opts, w, h, _ = bench.make_workload("c0")
    r = RtRenderer(scenes.standard_camera(space, opts, w, h))
    r.update(space)
    assert np.array_equal(outs[0], r.draw().data.reshape(-1, 4).astype(np.float32))
