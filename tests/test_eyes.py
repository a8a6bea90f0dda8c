"""Characters' eyes without a GPU: aicb_look_rotation against a restatement of Body::look_rotation, the rotation
applied to -Z against the directions set_look_direction was given, the eye structs' layouts against the C header, the
eye-step restatement (tests/eyeorc.py) on hand-derived cases, and the Python helpers that build a batch's camera
parameters and table."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import aicb200
import eyeorc
from aicb200 import GraphicsOptions, Viewport, abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# physics/body.rs:570-595: the directions of the reference's look_direction test, with the yaw and pitch it expects
LOOK_DIRECTIONS = [
    ((0.0, 0.0, -1.0), 0.0, 0.0),
    ((1.0, 0.0, -1.0), 45.0, 0.0),
    ((1.0, 0.0, 0.0), 90.0, 0.0),
    ((0.0, 0.0, 1.0), 180.0, 0.0),
    ((-1.0, 0.0, 0.0), 270.0, 0.0),
    ((0.0, 1.0, 0.0), 180.0, -90.0),
    ((0.0, 1.0, -1.0), 0.0, -45.0),
    ((0.0, -1.0, -1.0), 0.0, 45.0),
    ((0.0, -1.0, 0.0), 180.0, 90.0),
]


def to_degrees(x):
    return x * (180.0 / math.pi)   # f64::to_degrees


def to_radians(x):
    return x * (math.pi / 180.0)   # f64::to_radians


def set_look_direction(d):
    """Body::set_look_direction (physics/body.rs:304-309): (yaw, pitch) in degrees."""
    horizontal = math.hypot(d[0], d[2])
    yaw = math.fmod(180.0 - to_degrees(math.atan2(d[0], d[2])), 360.0)
    if yaw < 0.0:   # rem_euclid
        yaw += 360.0
    return yaw, -to_degrees(math.atan2(d[1], horizontal))


def q_then(s, o):
    """Rotation3D::then (s, then o), quaternions as (i, j, k, r)."""
    si, sj, sk, sr = s
    oi, oj, ok, orr = o
    return (oi * sr + orr * si + oj * sk - ok * sj,
            oj * sr + orr * sj + ok * si - oi * sk,
            ok * sr + orr * sk + oi * sj - oj * si,
            orr * sr - oi * si - oj * sj - ok * sk)


def look_rotation(yaw, pitch):
    """Body::look_rotation: around_x(-pitch.to_radians()).then(around_y(-yaw.to_radians()))."""
    hx = -to_radians(pitch) / 2.0
    hy = -to_radians(yaw) / 2.0
    return q_then((math.sin(hx), 0.0, 0.0, math.cos(hx)), (0.0, math.sin(hy), 0.0, math.cos(hy)))


def transform_vector(q, v):
    """Rotation3D::transform_vector3d."""
    i, j, k, r = q
    cx = (j * v[2] - k * v[1]) * 2.0
    cy = (k * v[0] - i * v[2]) * 2.0
    cz = (i * v[1] - j * v[0]) * 2.0
    return (v[0] + r * cx + j * cz - k * cy, v[1] + r * cy + k * cx - i * cz, v[2] + r * cz + i * cy - j * cx)


def bits(x):
    return np.array(x, dtype=np.float64).view(np.uint64)


def test_set_look_direction_restatement_gives_the_reference_angles():
    for d, yaw, pitch in LOOK_DIRECTIONS:
        assert set_look_direction(d) == (yaw, pitch), d


def test_look_rotation_equals_the_restatement():
    pairs = [(yaw, pitch) for _, yaw, pitch in LOOK_DIRECTIONS]
    pairs += [set_look_direction(d) for d, _, _ in LOOK_DIRECTIONS]
    rng = np.random.default_rng(11)
    pairs += [(float(y), float(p)) for y, p in zip(rng.uniform(0.0, 360.0, 2000), rng.uniform(-90.0, 90.0, 2000))]
    pairs += [(float(y), float(p)) for y, p in zip(rng.uniform(-1e4, 1e4, 500), rng.uniform(-1e3, 1e3, 500))]
    pairs += [(0.0, -0.0), (-0.0, 0.0), (360.0, 90.0), (-90.0, -90.0), (1e-300, -1e-300)]
    for yaw, pitch in pairs:
        got = aicb200.look_rotation(yaw, pitch)
        assert np.array_equal(bits(got), bits(look_rotation(yaw, pitch))), (yaw, pitch)


def test_look_rotation_looks_along_the_direction():
    for d, yaw, pitch in LOOK_DIRECTIONS:
        q = aicb200.look_rotation(*set_look_direction(d))
        along = np.array(transform_vector(q, (0.0, 0.0, -1.0)))
        want = np.array(d) / np.linalg.norm(d)
        assert np.allclose(along, want, rtol=0.0, atol=1e-15), (d, along)
        assert abs(np.linalg.norm(q) - 1.0) < 1e-15
    rng = np.random.default_rng(12)
    for d in rng.normal(size=(500, 3)):
        along = np.array(transform_vector(aicb200.look_rotation(*set_look_direction(d)), (0.0, 0.0, -1.0)))
        assert np.allclose(along, d / np.linalg.norm(d), rtol=0.0, atol=1e-14), d


def test_eye_structs_match_the_c_header(tmp_path):
    src = tmp_path / "eye_layout.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "aicb200.h"\n'
        'int main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %u\\n",'
        "sizeof(aicb_eye),offsetof(aicb_eye,displacement_vel),offsetof(aicb_eye,previous_body_velocity),"
        "sizeof(aicb_eye_view_params),offsetof(aicb_eye_view_params,fov_y_degrees),"
        "offsetof(aicb_eye_view_params,view_distance),offsetof(aicb_eye_view_params,nominal_width),"
        "offsetof(aicb_eye_view_params,nominal_height),offsetof(aicb_eye_view_params,fb_width),"
        "offsetof(aicb_eye_view_params,fb_height),offsetof(aicb_eye_view_params,fixed_exposure),"
        "offsetof(aicb_eye_view_params,automatic_exposure),offsetof(aicb_eye_view_params,lighting_display),"
        "offsetof(aicb_eye_view_params,_pad),AICB_EYE_NOT_INVERTIBLE);return 0;}\n")
    exe = tmp_path / "eye_layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    P = abi.EyeViewParams
    want = [abi.EYE_DTYPE.itemsize, abi.EYE_DTYPE.fields["displacement_vel"][1],
            abi.EYE_DTYPE.fields["previous_body_velocity"][1], C.sizeof(P)]
    want += [getattr(P, f).offset for f in ("fov_y_degrees", "view_distance", "nominal_width", "nominal_height",
                                            "fb_width", "fb_height", "fixed_exposure", "automatic_exposure",
                                            "lighting_display", "_pad")]
    want.append(abi.EYE_NOT_INVERTIBLE)
    assert got == want
    assert got[0] == 72 and got[3] == 48


def one_eye(pos=(0.0, 0.0, 0.0), vel=(0.0, 0.0, 0.0), prev=(0.0, 0.0, 0.0)):
    e = aicb200.eyes(1)
    e["displacement_pos"] = pos
    e["displacement_vel"] = vel
    e["previous_body_velocity"] = prev
    return e


@pytest.mark.parametrize("dt", [1.0 / 60.0, 1.0 / 3.0, 1.0])
def test_eye_at_rest_stays_at_rest(dt):
    b = aicb200.bodies(1, position=(3.0, 4.0, 5.0), velocity=(1.5, -2.0, 0.25))
    e = one_eye(prev=(1.5, -2.0, 0.25))
    for _ in range(10):
        e = eyeorc.step(e, b, dt)
    assert eyeorc.same_bytes(e["displacement_pos"], np.zeros((1, 3)))
    assert eyeorc.same_bytes(e["displacement_vel"], np.zeros((1, 3)))
    assert np.array_equal(e["previous_body_velocity"], b["velocity"])


@pytest.mark.parametrize("dt", [1.0 / 60.0, 1.0 / 3.0, 1.0])
def test_one_impulse_from_rest(dt):
    """Δv from zero displacement: the velocity is -0.04 Δv before the spring (zero at zero displacement) and the
    damping 1e-9^dt; the position moves by the damped velocity times dt."""
    dv = np.array([2.0, -10.0, 0.5])
    b = aicb200.bodies(1, velocity=dv)
    e = eyeorc.step(one_eye(), b, dt)
    before_damping = -(dv * 0.04)
    assert np.array_equal(bits(e["displacement_vel"][0]), bits(before_damping * math.pow(1e-9, dt)))
    assert np.array_equal(bits(e["displacement_pos"][0]), bits(before_damping * math.pow(1e-9, dt) * dt))
    assert np.array_equal(e["previous_body_velocity"][0], dv)
    if dt == 1.0:
        assert np.array_equal(e["displacement_vel"][0], before_damping * 1e-9)


def test_spring_pulls_towards_the_body():
    """Displacement (1, 0, 0) at rest, dt = 1: the spring gives -(1 * (1 + 1)) * 1e21, damped by 1e-9."""
    e = eyeorc.step(one_eye(pos=(1.0, 0.0, 0.0)), aicb200.bodies(1), 1.0)
    assert e["displacement_vel"][0, 0] == (0.0 - (1.0 * 2.0) * 1e21) * 1e-9
    assert e["displacement_pos"][0, 0] == 1.0 + e["displacement_vel"][0, 0] * 1.0
    assert e["displacement_vel"][0, 1] == 0.0 and e["displacement_pos"][0, 2] == 0.0


def test_eye_view_params_and_camera_table():
    vp = Viewport.with_scale(1.0, (40, 30))
    fixed = GraphicsOptions(fov_y=500.0, view_distance=0.5, exposure=1.75)
    p = aicb200.eye_view_params(fixed, vp)
    assert (p.fov_y_degrees, p.view_distance, p.nominal_width, p.nominal_height) == (189.0, 1.0, 40.0, 30.0)
    assert (p.fb_width, p.fb_height, p.fixed_exposure, p.automatic_exposure) == (40, 30, 1.75, 0)
    auto = GraphicsOptions(exposure=aicb200.EXPOSURE_AUTOMATIC, lighting_display=aicb200.LIGHT_NONE)
    p = aicb200.eye_view_params(auto, vp)
    assert (p.automatic_exposure, p.lighting_display) == (1, aicb200.LIGHT_NONE)
    for opts in (fixed, auto):
        table = aicb200.eye_cameras(5, opts, vp)
        assert table.dtype == abi.CAMERA_DTYPE and table.shape == (5,)
        one = bytes(aicb200.Camera(opts, vp).data)
        assert table.tobytes() == one * 5
    assert aicb200.eye_cameras(3, fixed, vp)["exposure"][0] == np.float32(1.75)
    assert aicb200.eye_cameras(3, auto, vp)["exposure"][0] == 1.0
