"""The oracle's two libm modes (tests/orc.py: LIBM_PLATFORM = glibc powf / expf, what Rust's std calls on this host;
LIBM_CR = correctly rounded, computed by the CUDA path's exact_math.cuh as host code, what the CUDA path does).

The GPU parity tests hold the CUDA path to the LIBM_CR oracle bit for bit; this module bounds the only remaining
difference to the reference on this platform — the libm — per call and per image, so that the two statements
together give the north_star's +-1 ULP per transcendental call without a tolerance window a kernel bug could hide in:
  * f32::powf in apply_transmittance (raytracer_components.rs:233) and f32::exp in distance_fog (sr.rs:751) are the
    only transcendental calls of the per-ray path (the sRGB encode uses the platform powf on both sides);
  * per call, glibc's result is within 1 ULP of the correctly rounded result, and equal to it on almost all inputs;
  * per image, the two modes give identical hits, steps and depths, and ColorBuf channels whose difference is
    bounded by (calls on the ray) x 1 ULP of the factors involved.
"""
import numpy as np

import orc
from aicb200 import (FOG_ABRUPT, FOG_PHYSICAL, LIGHT_LINEAR, TRANSPARENCY_VOLUMETRIC, GraphicsOptions, scenes)


def test_powf_expf_per_call_within_one_ulp():
    rng = np.random.default_rng(11)
    L = orc.lib()
    n = 200_000
    # unit transmittance 1 - alpha of any alpha in (0, 1), thickness of a span in (0, ~28] (a res-16 voxel .. cube diagonal x16)
    x = (1.0 - rng.uniform(0.0, 1.0, n)).astype(np.float32)
    x[: n // 4] = (1.0 - rng.choice([0.125, 0.25, 0.5, 0.0005, 0.999], n // 4)).astype(np.float32)
    y = np.exp(rng.uniform(np.log(1e-4), np.log(28.0), n)).astype(np.float32)
    a = np.array([L.orc_powf(float(x[i]), float(y[i]), 0) for i in range(n)], dtype=np.float32)
    b = np.array([L.orc_powf(float(x[i]), float(y[i]), 1) for i in range(n)], dtype=np.float32)
    d = orc.ulp_diff(a, b)
    assert d.max() <= 1, f"powf: glibc differs from the correctly rounded value by {d.max()} ULP"
    assert (d == 0).mean() > 0.95
    # fog: exp(-1.6 * rel), rel in [0, 1]
    e = (-1.6 * rng.uniform(0.0, 1.0, n)).astype(np.float32)
    a = np.array([L.orc_expf(float(v), 0) for v in e], dtype=np.float32)
    b = np.array([L.orc_expf(float(v), 1) for v in e], dtype=np.float32)
    d = orc.ulp_diff(a, b)
    assert d.max() <= 1, f"expf: glibc differs from the correctly rounded value by {d.max()} ULP"
    assert (d == 0).mean() > 0.95


def test_images_of_both_modes_agree_to_the_libm_bound():
    space = scenes.config_c2(n=32, n_voxel_blocks=6, with_light=True)
    prev = orc.get_libm()
    try:
        for opts in (GraphicsOptions(view_distance=128.0),
                     GraphicsOptions(view_distance=128.0, fog=FOG_PHYSICAL, lighting_display=LIGHT_LINEAR,
                                     transparency=TRANSPARENCY_VOLUMETRIC)):
            cam = scenes.standard_camera(space, opts, 160, 90)
            sc = orc.OracleScene(space)
            orc.set_libm(orc.LIBM_PLATFORM)
            a = sc.render(cam, opts)
            orc.set_libm(orc.LIBM_CR)
            b = sc.render(cam, opts)
            assert np.array_equal(a["hit"], b["hit"])
            assert np.array_equal(a["depth"], b["depth"])
            # a last-bit difference of T can move the opacity cut by one surface on a rare ray; none here
            assert np.array_equal(a["steps"], b["steps"])
            absd = np.abs(a["colorbuf"].astype(np.float64) - b["colorbuf"].astype(np.float64))
            # every factor differs by <= 1 ULP (6e-8 relative); a ray multiplies at most a few dozen of them
            scale = np.maximum(1.0, np.abs(b["colorbuf"].astype(np.float64)))
            assert (absd <= 64 * 6e-8 * scale).all(), absd.max()
            assert (orc.ulp_diff(a["colorbuf"], b["colorbuf"]) == 0).mean() > 0.98
            d8 = np.abs(a["srgb8"].astype(int) - b["srgb8"].astype(int))
            assert d8.max() <= 1
    finally:
        orc.set_libm(prev)
