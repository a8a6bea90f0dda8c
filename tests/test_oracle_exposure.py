"""The exposure oracle (oracle_exposure/) against the reference's own known answers (exposure.rs:168-241), the ray
pattern of State::step, its walk rules and no-ops; the correctly rounded f32 ln of exact_math.cuh against glibc's
logf; Camera.set_measured_exposure; and the aicb_exposure_state layout.  No GPU."""
import ctypes as C
import json
import math
import os
import subprocess
from decimal import Context, Decimal

import numpy as np
import pytest

import aicb200
import exposureorc
import lightorc
from aicb200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "all-is-cubes_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

IDENTITY = (0.0, 0.0, 0.0, 1.0)
STONE = aicb200.Block(color=(0.5, 0.5, 0.5, 1.0))
# Sky::Octants with eight distinct grey levels: octant k has luminance 0.25 * (k + 1) (a grey's luminance is its level
# up to the f32 sum's rounding)
OCTANTS = [(0.25 * (k + 1),) * 3 for k in range(8)]


@pytest.fixture(params=[0, 1], ids=["glibc", "cr"])
def libm(request):
    exposureorc.set_libm(request.param)
    yield request.param
    exposureorc.set_libm(1)


def f32_lum(rgb):
    r, g, b = (np.float32(v) for v in rgb)
    return g * np.float32(0.7152) + (r * np.float32(0.2126) + b * np.float32(0.0722))


def lut(v):
    """PackedLight::scalar_out (data.rs:232-243)."""
    return np.float32(0.0) if v == 0 else np.float32(2.0 ** ((np.float32(v) - np.float32(144.0)) / np.float32(10.0)))


def eye(translation, rotation=IDENTITY):
    return aicb200.view_transform_matrix(rotation, translation).reshape(1, 16)


def step(space, states, m, dt=0.1, ticks=1):
    sc = exposureorc.ExposureScene(space)
    out = None
    for _ in range(ticks):
        states, out = sc.step(states, m, dt)
    return states, out


def box_space(n, ids, light=None, sky=((1.0, 1.0, 1.0),), light_max_distance=30, blocks=None):
    table = [aicb200.Block.air(), STONE] if blocks is None else blocks
    ids = np.broadcast_to(np.asarray(ids, dtype=np.uint16), (n, n, n)).copy()
    return aicb200.Space((0, 0, 0), ids, table, light=light, sky_colors=list(sky), light_max_distance=light_max_distance)


def hollow_box_ids(n, fill=1):
    ids = np.full((n, n, n), fill, dtype=np.uint16)
    ids[1:-1, 1:-1, 1:-1] = 0
    return ids


def uniform_light(n, rgb_status):
    return np.broadcast_to(np.asarray(rgb_status, dtype=np.uint8), (n, n, n, 4)).copy()


def expected_direction(index, m):
    """exposure.rs:91-99 restated in Python floats (IEEE f64, as the reference): the un-normalised direction."""
    indexf = float(index)
    vx = math.fmod(indexf, 10.0) / 10.0 * 2.0 - 1.0
    vy = math.trunc(indexf / 10.0) / 10.0 * 2.0 - 1.0
    vz = -1.0
    return tuple(vx * m[0 + a] + vy * m[4 + a] + vz * m[8 + a] for a in range(3))


def octant(d):
    return (int(d[0] >= 0.0) << 2) + (int(d[1] >= 0.0) << 1) + int(d[2] >= 0.0)


def test_target_exposure():
    # exposure.rs:168-174
    got = [exposureorc.target_exposure(v) for v in (0.0, 0.01, 0.5, 1.0, 2.0, 100.0, 1000.0)]
    assert got == [np.float32(v) for v in (2.125, 2.125, 1.3, 0.9625, 0.79375, 0.6625, 0.6625)]
    assert math.isnan(exposureorc.target_exposure(float("nan")))


def test_e2e(libm):
    # exposure.rs:181-241: a 10^3 Space with sky 3, light evaluated, 100 ticks at 10 per second.  The reference's
    # character falls through the empty box meanwhile; every sample there is the sky, wherever the eye is, so a fixed
    # eye at the box's centre is the same test.
    space = box_space(10, 0, sky=((3.0, 3.0, 3.0),))
    lo = lightorc.LightOracle(space)
    lo.fast_evaluate()
    lo.evaluate()
    space.light = lo.field()
    st, out = step(space, aicb200.exposure_states(1), eye((5.0, 5.0, 5.0)), dt=0.1, ticks=100)
    assert exposureorc.luminance_average(st[0]) == np.float32(3.0)
    expected = exposureorc.target_exposure(3.0)
    assert abs(out[0] / expected - 1.0) < 0.001
    assert out[0] == np.float32(math.exp(float(st[0]["exposure_log"]))) or libm == 1


def test_default_states():
    st = aicb200.exposure_states(3)
    assert st.dtype == abi.EXPOSURE_STATE_DTYPE and st.dtype.itemsize == 408
    assert (st["luminance_samples"] == 1.0).all() and (st["luminance_sample_index"] == 0).all()
    assert (st["exposure_log"] == 0.0).all()


@pytest.mark.parametrize("rotation", [IDENTITY, (0.0, 1.0, 0.0, 0.0), (0.3, -0.2, 0.5, 0.78)],
                         ids=["identity", "turned", "tilted"])
def test_sample_pattern_and_ring(rotation):
    # under LightPhysics::None every ray takes the sky in its own direction: the samples show which ring index got
    # which direction (rem_euclid for x, div_euclid for y, z = -1, through the eye's rotation, not normalised)
    space = box_space(4, 0, sky=OCTANTS, light_max_distance=0)
    m = eye((2.0, 2.0, 2.0), rotation)
    st = aicb200.exposure_states(1)
    st["luminance_samples"] = -1.0
    for tick in range(10):
        st, _ = step(space, st, m)
        assert st[0]["luminance_sample_index"] == (10 * tick + 10) % 100
    want = [f32_lum(OCTANTS[octant(expected_direction(i, m[0]))]) for i in range(100)]
    assert np.array_equal(st[0]["luminance_samples"], np.array(want, dtype=np.float32))
    if rotation == IDENTITY:
        # by hand: x >= 0 from column 5 of the 10 x 10 grid, y >= 0 from row 5, z always -1
        for i in range(100):
            assert want[i] == f32_lum(OCTANTS[(4 if i % 10 >= 5 else 0) + (2 if i // 10 >= 5 else 0)])


@pytest.mark.parametrize("index, first", [(95, 96), (99, 0), (2 ** 32 - 1, 96), (12345, 46)])
def test_ring_index_wraps_as_usize(index, first):
    space = box_space(4, 0, sky=OCTANTS, light_max_distance=0)
    st = aicb200.exposure_states(1)
    st["luminance_sample_index"] = index
    st["luminance_samples"] = -1.0
    st, _ = step(space, st, eye((2.0, 2.0, 2.0)))
    written = [(first + k) % 100 for k in range(10)]
    assert st[0]["luminance_sample_index"] == written[-1]
    s = st[0]["luminance_samples"]
    assert all(s[i] != -1.0 for i in written)
    assert all(s[i] == -1.0 for i in range(100) if i not in written)


def test_light_physics_none_samples_the_sky_in_a_closed_box():
    n = 6
    ids = hollow_box_ids(n)
    space = box_space(n, ids, light=uniform_light(n, (150, 150, 150, 255)), sky=((2.0, 2.0, 2.0),),
                      light_max_distance=0)
    st, _ = step(space, aicb200.exposure_states(1), eye((3.0, 3.0, 3.0)))
    s = st[0]["luminance_samples"]
    assert (s[1:11] == f32_lum((2.0, 2.0, 2.0))).all()


def test_closed_box_takes_the_light_in_front_of_the_wall():
    n = 6
    light = uniform_light(n, (150, 150, 150, 255))
    space = box_space(n, hollow_box_ids(n), light=light, sky=((2.0, 2.0, 2.0),))
    st, _ = step(space, aicb200.exposure_states(1), eye((3.0, 3.0, 3.0)))
    assert (st[0]["luminance_samples"][1:11] == f32_lum([lut(150)] * 3)).all()


def test_eye_inside_a_visible_block_takes_its_own_cube():
    n = 4
    light = uniform_light(n, (120, 130, 140, 255))
    light[1, 1, 1] = (160, 100, 90, 255)
    space = box_space(n, 1, light=light)
    st, _ = step(space, aicb200.exposure_states(1), eye((1.5, 1.5, 1.5)))
    assert (st[0]["luminance_samples"][1:11] == f32_lum([lut(160), lut(100), lut(90)])).all()


def invisible_recursive():
    pal = np.zeros((2, 8), dtype=np.float32)
    pal[1, :4] = (0.2, 0.3, 0.4, 1.0)   # an entry no voxel uses
    return aicb200.Block(resolution=4, indices=np.zeros((4, 4, 2), dtype=np.uint16), palette=pal)


def hint_only():
    b = aicb200.Block(color=(0.0, 0.0, 0.0, 0.0))
    b.light_visible = True   # the animation hint: light_visible without a visible voxel
    return b


@pytest.mark.parametrize("make", [invisible_recursive, hint_only], ids=["invisible_recursive", "animation_hint"])
def test_invisible_blocks_are_passed_through(make):
    n = 5
    table = [aicb200.Block.air(), make()]
    space = box_space(n, 1, light=uniform_light(n, (150, 150, 150, 255)), sky=((2.0, 2.0, 2.0),), blocks=table)
    sc = exposureorc.ExposureScene(space)
    assert not sc.visible(1)
    st, _ = sc.step(aicb200.exposure_states(1), eye((2.5, 2.5, 2.5)), 0.1)
    assert (st[0]["luminance_samples"][1:11] == f32_lum((2.0, 2.0, 2.0))).all()


def test_partly_visible_recursive_block_is_visible():
    pal = np.zeros((2, 8), dtype=np.float32)
    pal[1, :4] = (0.2, 0.3, 0.4, 1.0)
    idx = np.zeros((4, 4, 4), dtype=np.uint16)
    idx[3, 3, 3] = 1
    space = box_space(2, 1, blocks=[aicb200.Block.air(), aicb200.Block(resolution=4, indices=idx, palette=pal)])
    assert exposureorc.ExposureScene(space).visible(1)


@pytest.mark.parametrize("status", [0, 1, 128], ids=["uninitialized", "no_rays", "opaque"])
def test_light_that_is_not_visible_continues_the_walk(status):
    # every cube but the eye's is a visible block whose light is not Visible: each ray walks to the bounds, and takes
    # the sky; with the eye's cube lit and the walls' light Visible the first wall decides instead
    n = 5
    ids = np.ones((n, n, n), dtype=np.uint16)
    ids[2, 2, 2] = 0
    light = uniform_light(n, (150, 150, 150, status))
    space = box_space(n, ids, light=light, sky=((2.0, 2.0, 2.0),))
    st, _ = step(space, aicb200.exposure_states(1), eye((2.5, 2.5, 2.5)))
    assert (st[0]["luminance_samples"][1:11] == f32_lum((2.0, 2.0, 2.0))).all()
    light[2, 2, 2] = (170, 170, 170, 255)
    light[:, :, :1] = (110, 110, 110, 255)
    space.light = light
    st, _ = step(space, aicb200.exposure_states(1), eye((2.5, 2.5, 2.5)))
    assert (st[0]["luminance_samples"][1:11] == f32_lum([lut(170)] * 3)).all()


def test_cube_behind_outside_the_bounds_takes_light_outside():
    # the eye above the Space looking down into a slab of stone: cube_behind of the first step is beyond the bounds,
    # where get_light is BlockSky::light_outside (the sky's face texel, PZ here)
    n = 4
    space = box_space(n, 1, light=uniform_light(n, (100, 100, 100, 255)), sky=((2.0, 2.0, 2.0),))
    L = exposureorc.lib()
    L.orc_scene_create.restype = C.c_void_p
    L.orc_scene_create.argtypes = [C.POINTER(abi.SceneDesc)]
    L.orc_scene_block_sky.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_scene_destroy.argtypes = [C.c_void_p]
    desc, keep = space.to_desc()
    h = L.orc_scene_create(C.byref(desc))
    faces = np.zeros((7, 4), dtype=np.uint8)
    L.orc_scene_block_sky(h, faces.ctypes.data)
    L.orc_scene_destroy(h)
    pz = faces[5]
    assert pz[3] == 255
    st, _ = step(space, aicb200.exposure_states(1), eye((2.0, 2.0, 10.0)))
    assert (st[0]["luminance_samples"][1:11] == f32_lum([lut(v) for v in pz[:3]])).all()


def test_no_ops_leave_the_state_bytes():
    space = box_space(4, 0, sky=OCTANTS)
    st0 = aicb200.exposure_states(4)
    rng = np.random.default_rng(5)
    st0["luminance_samples"] = rng.uniform(0.1, 5.0, (4, 100)).astype(np.float32)
    st0["luminance_sample_index"] = [3, 99, 0, 50]
    st0["exposure_log"] = [0.5, -0.25, 0.0, 1.0]
    # dt == 0: nothing at all
    st, out = step(space, st0, np.repeat(eye((2.0, 2.0, 2.0)), 4, axis=0), dt=0.0)
    assert exposureorc.same_bytes(st, st0)
    assert np.array_equal(out, np.exp(st0["exposure_log"].astype(np.float64)).astype(np.float32))
    # !(w > 0): w = 0, w < 0, w NaN, and a NaN m44
    m = np.repeat(eye((2.0, 2.0, 2.0)), 4, axis=0)
    m[0, 15] = 0.0
    m[1, 15] = -1.0
    m[2, 3] = np.inf   # 0 * inf = NaN in w
    m[3, 15] = np.nan
    st, _ = step(space, st0, m)
    assert exposureorc.same_bytes(st, st0)


def test_sum_folds_from_negative_zero():
    # Sum for f32 starts from -0.0 (core::iter's float Sum since Rust 1.83; the reference's toolchain is newer:
    # it uses `[1.0; _]`, stable since 1.89), so 100 samples of -0.0 average -0.0, 0.9 / -0.0 is -inf and the target
    # is clamped up to 0.1: 0.6625, not the 2.125 a +0.0 start would give
    space = box_space(4, 0, sky=((-0.0, -0.0, -0.0),), light_max_distance=0)
    st = aicb200.exposure_states(1)
    st["luminance_samples"] = -0.0
    st, _ = step(space, st, eye((2.0, 2.0, 2.0)), dt=0.5)
    assert exposureorc.luminance_average(st[0]) == 0.0 and np.signbit(exposureorc.luminance_average(st[0]))
    target = exposureorc.target_exposure(-0.0)
    assert target == np.float32(0.6625)
    assert st[0]["exposure_log"] == np.float32(math.log(float(target)))   # (ln target - 0) * 0.5 * 2


def test_view_transform_matrix():
    m = aicb200.view_transform_matrix(IDENTITY, (1.0, 2.0, 3.0)).reshape(4, 4)
    assert np.array_equal(m, [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [1, 2, 3, 1]])
    # a half turn about Y: x and z change sign
    m = aicb200.view_transform_matrix((0.0, 1.0, 0.0, 0.0), (0.0, 0.0, 0.0)).reshape(4, 4)
    assert np.array_equal(m, [[-1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]])


def test_set_measured_exposure():
    vp = aicb200.Viewport.with_scale(1.0, (8, 8))
    fixed = aicb200.Camera(aicb200.GraphicsOptions(exposure=2.0), vp)
    fixed.set_measured_exposure(3.0)
    assert fixed.exposure_value == 2.0 and fixed.data.exposure == np.float32(2.0)
    auto = aicb200.Camera(aicb200.GraphicsOptions(exposure=aicb200.EXPOSURE_AUTOMATIC), vp)
    assert auto.exposure_value == 1.0 and auto.data.exposure == 1.0   # ExposureOption::initial()
    auto.set_measured_exposure(1.75)
    assert auto.data.exposure == np.float32(1.75)
    for bad in (float("nan"), -0.5):
        auto.set_measured_exposure(bad)   # PositiveSign::try_from refuses it: unchanged
        assert auto.data.exposure == np.float32(1.75)
    auto.set_measured_exposure(-0.0)
    assert auto.data.exposure == 0.0 and not np.signbit(auto.data.exposure)
    none = aicb200.Camera(aicb200.GraphicsOptions(exposure=aicb200.EXPOSURE_AUTOMATIC,
                                                  lighting_display=aicb200.LIGHT_NONE), vp)
    none.set_measured_exposure(0.25)
    assert none.data.exposure == 1.0


def test_exposure_state_layout(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "aicb200.h"\n'
                   'int main(){printf("%zu %zu %zu %zu\\n", sizeof(aicb_exposure_state),'
                   'offsetof(aicb_exposure_state, luminance_samples),'
                   'offsetof(aicb_exposure_state, luminance_sample_index),'
                   'offsetof(aicb_exposure_state, exposure_log));return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    d = abi.EXPOSURE_STATE_DTYPE
    assert got == [d.itemsize, d.fields["luminance_samples"][1], d.fields["luminance_sample_index"][1],
                   d.fields["exposure_log"][1]]


LN_DRIVER = r"""
#include <cmath>
#include <cstdio>
#include <cstring>
#include "exact_math.cuh"
using namespace aicb;
static uint32_t bits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
static float from_bits(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
int main() {
    // every f32 in [0.6625, 2.125]: the targets compute_target_exposure can give
    const uint32_t lo = bits(0.6625f), hi = bits(2.125f);
    unsigned long long n = 0, far = 0;
    std::printf("{\"differ\": [");
    bool first = true;
    for (uint32_t b = lo; b <= hi; b++) {
        const float x = from_bits(b), got = logf_exact(x), want = logf(x);
        n++;
        if (bits(got) != bits(want)) {
            const long long d = (long long)bits(got) - (long long)bits(want);
            if (d > 1 || d < -1 || std::signbit(got) != std::signbit(want)) far++;
            std::printf("%s[%u, %u, %u]", first ? "" : ", ", b, bits(got), bits(want));
            first = false;
        }
    }
    std::printf("], \"n\": %llu, \"far\": %llu, \"ln1\": %u}\n", n, far, bits(logf_exact(1.0f)));
    return 0;
}
"""


def test_logf_exact_against_glibc(tmp_path):
    # exact_math.cuh's logf_exact compiled as host code with the project's -fmad=false contract, on every f32 in
    # [0.6625, 2.125]: within 1 ULP of glibc's logf, and where they differ, logf_exact is the nearer to ln x
    src, exe = tmp_path / "ln.cu", tmp_path / "ln"
    src.write_text(LN_DRIVER)
    cmd = [NVCC, "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false",
           "-Xcompiler", "-ffp-contract=off,-fno-fast-math,-O2", "-I", CSRC, "-o", str(exe), str(src)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    t = json.loads(subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout)
    f = lambda u: float(np.array(u, dtype=np.uint32).view(np.float32))
    assert t["n"] == int(np.float32(2.125).view(np.uint32)) - int(np.float32(0.6625).view(np.uint32)) + 1
    assert t["far"] == 0 and t["ln1"] == 0
    ctx = Context(prec=60)
    for xb, gb, wb in t["differ"]:
        exact = ctx.ln(Decimal(f(xb)))
        assert abs(exact - Decimal(f(gb))) < abs(exact - Decimal(f(wb))), (f(xb), f(gb), f(wb))
    print(f"logf_exact: {t['n']} arguments, glibc's logf is not the nearest f32 at {len(t['differ'])}")
