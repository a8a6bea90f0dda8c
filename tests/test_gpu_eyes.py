"""Characters' eyes on the GPU (aicb_step_eyes_device, aicb_eye_views_device and their group forms): the eye step
against tests/eyeorc.py bit for bit; each eye's matrix, camera, look ray and status against the host camera functions;
the exposure rule against Camera.set_measured_exposure; every NULL-output combination; a whole tick of 64 characters
run as one chain of device calls against the same ticks run with the host calls; groups; and the rejections."""
import ctypes as C
import itertools
import math

import numpy as np
import pytest
import torch

import aicb200
import eyeorc
from aicb200 import GraphicsOptions, SpaceRaytracer, Viewport, abi, scenes
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit
from test_gpu_views import single

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
LIB = aicb200.load_library()


def as_dev(records):
    """A structured numpy array as a uint8 CUDA tensor [n, itemsize]."""
    a = np.ascontiguousarray(records)
    return torch.from_numpy(a.view(np.uint8).reshape(len(a), a.dtype.itemsize).copy()).to(DEV)


def records(t, dtype):
    return t.cpu().numpy().view(dtype).reshape(-1)


def random_batch(n, seed):
    """Eyes and bodies: random displacements (some zero), velocities large, tiny and zero."""
    rng = np.random.default_rng(seed)
    e = aicb200.eyes(n)
    scale = rng.choice([0.0, 1e-300, 1e-8, 0.1, 1.0, 1e6], size=(n, 1))
    e["displacement_pos"] = rng.normal(size=(n, 3)) * scale
    e["displacement_vel"] = rng.normal(size=(n, 3)) * rng.choice([0.0, 1e-3, 1.0, 1e5], size=(n, 1))
    e["previous_body_velocity"] = rng.normal(size=(n, 3)) * rng.choice([0.0, 1e-200, 1.0, 1e8], size=(n, 1))
    b = aicb200.bodies(n, position=rng.uniform(-50, 50, (n, 3)),
                       velocity=rng.normal(size=(n, 3)) * rng.choice([0.0, 1e-250, 1e-3, 10.0, 1e9], size=(n, 1)))
    return e, b


def small_scene():
    return SpaceRaytracer(scenes.small_mixed_scene(n=12, seed=7), GraphicsOptions())


@pytest.mark.parametrize("n", [1, 31, 33, 4096])
@pytest.mark.parametrize("dt", [1.0 / 60.0, 1.0 / 3.0, 1.0], ids=["60th", "3rd", "1"])
def test_step_equals_the_restatement(n, dt):
    rt = small_scene()
    eyes, bodies = random_batch(n, seed=n)
    rng = np.random.default_rng(n + 1)
    de, db = as_dev(eyes), as_dev(bodies)
    for tick in range(100):
        if tick % 3 == 0:   # the body's velocity changes: landing, jumping, pushed
            bodies["velocity"] = bodies["velocity"] * rng.choice([0.0, 0.5, 1.0, -1.0], size=(n, 1)) + \
                rng.normal(size=(n, 3)) * rng.choice([0.0, 1e-6, 5.0], size=(n, 1))
            db = as_dev(bodies)
        eyes = eyeorc.step(eyes, bodies, dt)
        rt.step_eyes(de, db, dt)
        if tick in (0, 1, 9, 99) or n < 64:
            got = records(de, abi.EYE_DTYPE)
            assert eyeorc.same_bytes(got, eyes), f"tick {tick}"
    rt.close()


def host_views(eyes, bodies, rot, params):
    """What the host functions give for each eye: (eye_to_world, camera records with exposure 0, look rays, status)."""
    n = len(eyes)
    t = eyeorc.eye_translation(eyes, bodies)
    m = np.zeros((n, 16))
    cams = np.zeros(n, abi.CAMERA_DTYPE)
    rays = np.zeros((n, 6))
    status = np.zeros(n, np.int32)
    for i in range(n):
        q = (C.c_double * 4)(*rot[i])
        tr = (C.c_double * 3)(*t[i])
        cam = abi.CameraData()
        st = LIB.aicb_camera_from_view(q, tr, params.fov_y_degrees, params.view_distance, params.nominal_width,
                                       params.nominal_height, params.fb_width, params.fb_height, 0.0, C.byref(cam))
        if st != abi.OK:
            status[i] = abi.EYE_NOT_INVERTIBLE
            continue
        m[i] = aicb200.view_transform_matrix(rot[i], t[i])
        cams[i] = np.frombuffer(bytes(cam), abi.CAMERA_DTYPE)[0]
        out = (C.c_double * 6)()
        LIB.aicb_camera_project_ndc(C.byref(cam), 0.0, 0.0, out)
        rays[i] = out[:]
    return m, cams, rays, status


def random_rotations(n, seed):
    rng = np.random.default_rng(seed)
    q = np.array([aicb200.look_rotation(y, p) for y, p in zip(rng.uniform(0, 360, n), rng.uniform(-90, 90, n))])
    q[1::5] = rng.normal(size=(len(q[1::5]), 4))         # not normalised
    q[2::7] = [0.0, 0.0, 0.0, 1.0]
    q[5::17] = 0.0                                        # to_transform's identity: a camera like any other
    q[3::11] = [0.5, 0.5, 0.0, 0.0]                       # degenerate: a singular matrix, no inverse
    q[4::13] = rng.normal(size=(len(q[4::13]), 4)) * 1e-170   # underflowing rotation terms
    return np.ascontiguousarray(q)


VIEWS = [
    (GraphicsOptions(), Viewport.with_scale(1.0, (64, 48))),
    (GraphicsOptions(fov_y=500.0, view_distance=1e6, exposure=1.75), Viewport.with_scale(2.0, (33, 7))),
    (GraphicsOptions(fov_y=0.25, view_distance=0.0, exposure=aicb200.EXPOSURE_AUTOMATIC), Viewport((0.0, 0.0), (1, 1))),
    (GraphicsOptions(exposure=aicb200.EXPOSURE_AUTOMATIC, lighting_display=aicb200.LIGHT_NONE),
     Viewport.with_scale(1.0, (1920, 1080))),
]


def fresh_outputs(n, fill=0xAB):
    return (torch.full((n, 16 * 8), fill, dtype=torch.uint8, device=DEV).view(torch.float64),
            torch.full((n, 144), fill, dtype=torch.uint8, device=DEV),
            torch.full((n, 48), fill, dtype=torch.uint8, device=DEV).view(torch.float64),
            torch.full((n, 4), fill, dtype=torch.uint8, device=DEV).view(torch.int32).reshape(n))


@pytest.mark.parametrize("view", range(len(VIEWS)))
def test_views_equal_the_host_functions(view):
    opts, vp = VIEWS[view]
    params = aicb200.eye_view_params(opts, vp)
    rt = small_scene()
    n = 517
    eyes, bodies = random_batch(n, seed=40 + view)
    rot = random_rotations(n, seed=view)
    m, cams, rays, status = host_views(eyes, bodies, rot, params)
    assert (status == abi.EYE_NOT_INVERTIBLE).sum() >= n // 13
    dm, dc, dr, ds = fresh_outputs(n)
    before = dc.clone()
    exposures = torch.full((n,), 0.625, dtype=torch.float32, device=DEV)
    rt.eye_views(as_dev(eyes), as_dev(bodies), torch.from_numpy(rot).to(DEV), exposures, params, dm, dc, dr, ds)
    got_s = ds.cpu().numpy()
    assert np.array_equal(got_s, status)
    ok = status == 0
    assert eyeorc.same_bytes(dm.cpu().numpy()[ok], m[ok])
    assert eyeorc.same_bytes(dr.cpu().numpy()[ok], rays[ok])
    gc = records(dc, abi.CAMERA_DTYPE)
    want_exposure = np.float32(opts.exposure if opts.exposure != aicb200.EXPOSURE_AUTOMATIC else
                               (1.0 if opts.lighting_display == aicb200.LIGHT_NONE else 0.625))
    cams["exposure"] = want_exposure
    assert eyeorc.same_bytes(gc[ok], cams[ok])
    # a degenerate rotation writes its status alone
    bad = ~ok
    assert (dm.view(torch.uint8).cpu().numpy().reshape(n, -1)[bad] == 0xAB).all()
    assert (dr.view(torch.uint8).cpu().numpy().reshape(n, -1)[bad] == 0xAB).all()
    assert np.array_equal(dc.cpu().numpy()[bad], before.cpu().numpy()[bad])
    rt.close()


MEASUREMENTS = np.array([0.5, np.nan, -1.0, -0.0, np.inf, 0.0, 2.0, -np.inf, 1e-45, 3.25], np.float32)


@pytest.mark.parametrize("kind", ["fixed", "automatic", "automatic-none"])
def test_exposure_rule_equals_set_measured_exposure(kind):
    opts = {"fixed": GraphicsOptions(exposure=0.75),
            "automatic": GraphicsOptions(exposure=aicb200.EXPOSURE_AUTOMATIC),
            "automatic-none": GraphicsOptions(exposure=aicb200.EXPOSURE_AUTOMATIC,
                                              lighting_display=aicb200.LIGHT_NONE)}[kind]
    vp = Viewport.with_scale(1.0, (16, 12))
    params = aicb200.eye_view_params(opts, vp)
    rt = small_scene()
    n = len(MEASUREMENTS)
    eyes, bodies = random_batch(n, seed=3)
    rot = np.array([aicb200.look_rotation(30.0 * i, 5.0 * i - 20.0) for i in range(n)])
    host = [aicb200.Camera(opts, vp) for _ in range(n)]
    table = as_dev(aicb200.eye_cameras(n, opts, vp))
    rng = np.random.default_rng(5)
    de, db, dq = as_dev(eyes), as_dev(bodies), torch.from_numpy(rot).to(DEV)
    for rnd in range(12):
        meas = None if rnd % 4 == 3 else rng.permutation(MEASUREMENTS)
        rt.eye_views(de, db, dq, None if meas is None else torch.from_numpy(meas).to(DEV), params, cameras=table)
        got = records(table, abi.CAMERA_DTYPE)["exposure"]
        for i, cam in enumerate(host):
            if meas is not None:
                cam.set_measured_exposure(meas[i])
        want = np.array([cam.data.exposure for cam in host], np.float32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (rnd, got, want)
    rt.close()


def test_every_null_output_combination():
    opts = GraphicsOptions(exposure=aicb200.EXPOSURE_AUTOMATIC)
    params = aicb200.eye_view_params(opts, Viewport.with_scale(1.0, (40, 30)))
    rt = small_scene()
    n = 70
    eyes, bodies = random_batch(n, seed=8)
    rot = random_rotations(n, seed=8)
    de, db, dq = as_dev(eyes), as_dev(bodies), torch.from_numpy(rot).to(DEV)
    ex = torch.from_numpy(np.resize(MEASUREMENTS, n)).to(DEV)
    full = fresh_outputs(n)
    rt.eye_views(de, db, dq, ex, params, *full)
    full = [t.cpu() for t in full]
    for exposures in (ex, None):
        for mask in itertools.product([False, True], repeat=4):
            outs = fresh_outputs(n)
            given = [t if keep else None for t, keep in zip(outs, mask)]
            rt.eye_views(de, db, dq, exposures, params, *given)
            for t, want, keep, name in zip(outs, full, mask, ("eye_to_world", "cameras", "look_rays", "status")):
                t = t.cpu()
                if not keep:
                    assert (t.view(torch.uint8) == 0xAB).all(), (mask, name)
                elif name == "cameras" and exposures is None:
                    # no measurement: each entry keeps its exposure, the rest is written
                    a, b = t.numpy().view(abi.CAMERA_DTYPE), want.numpy().view(abi.CAMERA_DTYPE)
                    st = full[3].numpy() == 0
                    assert eyeorc.same_bytes(a["inverse_projection_view"][st], b["inverse_projection_view"][st])
                    assert (a["exposure"].view(np.uint32) == 0xABABABAB).all()
                else:
                    assert torch.equal(t.view(torch.uint8), want.view(torch.uint8)), (mask, name)
    rt.close()


@pytest.mark.parametrize("target", TARGETS, ids=TARGET_IDS)
def test_groups_give_one_contexts_bytes(target):
    space = scenes.small_mixed_scene(n=12, seed=7)
    lit = Lit(target, space)
    opts = GraphicsOptions(exposure=aicb200.EXPOSURE_AUTOMATIC)
    params = aicb200.eye_view_params(opts, Viewport.with_scale(1.0, (40, 30)))
    n = 1000
    eyes, bodies = random_batch(n, seed=9)
    rot = random_rotations(n, seed=9)
    want_eyes = eyeorc.step(eyes, bodies, 0.05)
    m, cams, rays, status = host_views(want_eyes, bodies, rot, params)
    de, db = as_dev(eyes), as_dev(bodies)
    side = torch.cuda.Stream(DEV)
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)   # the inputs are written late on the stream the calls are issued on
        de2 = de.clone()
        lit.scene.step_eyes(de2, db, 0.05)
        outs = fresh_outputs(n)
        lit.scene.eye_views(de2, db, torch.from_numpy(rot).to(DEV), torch.full((n,), 2.5, device=DEV), params, *outs)
        copies = [t.clone() for t in (de2,) + outs]
    side.synchronize()
    assert eyeorc.same_bytes(records(copies[0], abi.EYE_DTYPE), want_eyes)
    ok = status == 0
    assert np.array_equal(copies[4].cpu().numpy(), status)
    assert eyeorc.same_bytes(copies[1].cpu().numpy()[ok], m[ok])
    cams["exposure"] = 2.5
    assert eyeorc.same_bytes(records(copies[2], abi.CAMERA_DTYPE)[ok], cams[ok])
    assert eyeorc.same_bytes(copies[3].cpu().numpy()[ok], rays[ok])
    lit.close()


@pytest.mark.parametrize("devices", [None, [0, 0]], ids=["ctx", "group2"])
def test_rejections_write_nothing(devices):
    lit = Lit(devices, scenes.small_mixed_scene(n=12, seed=7))
    s = lit.scene
    pre = "aicb_" if devices is None else "aicb_group_"
    fs, fv = getattr(LIB, pre + "step_eyes_device"), getattr(LIB, pre + "eye_views_device")
    n = 8
    eyes, bodies = random_batch(n, seed=1)
    de, db = as_dev(eyes), as_dev(bodies)
    dq = torch.from_numpy(random_rotations(n, 1)).to(DEV)
    params = aicb200.eye_view_params(GraphicsOptions(), Viewport.with_scale(1.0, (8, 8)))
    for dt in (0.0, -0.1, 1.5, math.nan, math.inf):
        assert fs(s.handle, de.data_ptr(), db.data_ptr(), n, dt, None) == abi.ERR_INVALID
    assert fs(s.handle, None, db.data_ptr(), n, 0.1, None) == abi.ERR_INVALID
    assert fs(s.handle, de.data_ptr(), None, n, 0.1, None) == abi.ERR_INVALID
    assert fs(s.handle, eyes.ctypes.data, db.data_ptr(), n, 0.1, None) == abi.ERR_INVALID   # host memory
    assert fs(s.handle, de.data_ptr() + 4, db.data_ptr(), n, 0.1, None) == abi.ERR_INVALID  # misaligned
    assert fs(s.handle, None, None, 0, 0.1, None) == abi.OK
    outs = fresh_outputs(n)
    ptrs = [t.data_ptr() for t in outs]
    assert fv(s.handle, de.data_ptr(), db.data_ptr(), dq.data_ptr(), None, n, None, *ptrs, None) == abi.ERR_INVALID
    p = C.byref(params)
    assert fv(s.handle, de.data_ptr(), db.data_ptr(), None, None, n, p, *ptrs, None) == abi.ERR_INVALID
    assert fv(s.handle, de.data_ptr(), db.data_ptr(), dq.data_ptr(), None, n, p, ptrs[0] + 4, *ptrs[1:],
              None) == abi.ERR_INVALID
    host_out = np.zeros((n, 6))
    assert fv(s.handle, de.data_ptr(), db.data_ptr(), dq.data_ptr(), None, n, p, ptrs[0], ptrs[1],
              host_out.ctypes.data, ptrs[3], None) == abi.ERR_INVALID
    assert fv(s.handle, None, None, None, None, 0, p, None, None, None, None, None) == abi.OK
    torch.cuda.synchronize()
    assert eyeorc.same_bytes(records(de, abi.EYE_DTYPE), eyes)
    assert all((t.view(torch.uint8) == 0xAB).all() for t in outs)
    lit.close()


def lit_c2():
    s = scenes.config_c2(n=48, seed=3, n_voxel_blocks=8, with_light=True)
    return aicb200.Space(s.lower, s.block_ids, s.blocks, light=s.light, sky_colors=scenes.OCTANT_SKY,
                         light_max_distance=20)


def test_whole_tick_on_the_device_equals_the_host_calls():
    """64 characters, 20 ticks: bodies, exposure, eyes, views, cursor and frames as one chain of device calls on a side
    stream, against host body and exposure steps, host eye arithmetic, aicb_camera_from_view, single-camera
    aicb_render_srgb8 and aicb_cursor_raycast per character."""
    space = lit_c2()
    opts = GraphicsOptions(exposure=aicb200.EXPOSURE_AUTOMATIC, view_distance=40.0)
    vp = Viewport.with_scale(1.0, (24, 16))
    params = aicb200.eye_view_params(opts, vp)
    rt = SpaceRaytracer(space, opts)
    n, dt, gravity = 64, 1.0 / 20.0, (0.0, -20.0, 0.0)
    rng = np.random.default_rng(64)
    bodies = aicb200.bodies(n, position=rng.uniform(4, 44, (n, 3)), collision_box=(-0.3, -0.8, -0.3, 0.3, 0.9, 0.3),
                            velocity=rng.normal(size=(n, 3)) * 4.0, flying=rng.random(n) < 0.2)
    eyes = aicb200.eyes(n)
    states = aicb200.exposure_states(n)
    m = np.zeros((n, 16))
    cams = [aicb200.Camera(opts, vp) for _ in range(n)]
    yaw, pitch = rng.uniform(0, 360, n), rng.uniform(-60, 60, n)
    d_bodies, d_eyes, d_states = as_dev(bodies), as_dev(eyes), as_dev(states)
    d_m = torch.zeros((n, 16), dtype=torch.float64, device=DEV)
    d_table = as_dev(aicb200.eye_cameras(n, opts, vp))
    d_rays = torch.zeros((n, 6), dtype=torch.float64, device=DEV)
    d_status = torch.zeros(n, dtype=torch.int32, device=DEV)
    side = torch.cuda.Stream(DEV)
    for tick in range(20):
        yaw, pitch = (yaw + 7.0) % 360.0, np.clip(pitch + rng.uniform(-5, 5, n), -89.0, 89.0)
        rot = np.array([aicb200.look_rotation(y, p) for y, p in zip(yaw, pitch)])
        # the host calls
        bodies = rt.step_bodies(bodies, dt, gravity)[0]
        states, exposures = rt.step_exposure(states, m, dt)
        eyes = eyeorc.step(eyes, bodies, dt)
        t = eyeorc.eye_translation(eyes, bodies)
        frames, cursors = [], []
        for i, cam in enumerate(cams):
            m[i] = aicb200.view_transform_matrix(rot[i], t[i])
            cam.set_view_transform(rot[i], t[i])
            cam.set_measured_exposure(exposures[i])
            frames.append(single(rt, cam, opts, "srgb8")[0])
            cursors.append(rt.cursor_raycast(cam.project_ndc_into_world(0.0, 0.0).reshape(1, 6), 6.0))
        # the device chain
        with torch.cuda.stream(side):
            d_rot = torch.from_numpy(rot).to(DEV, non_blocking=False)
            d_bodies = rt.step_bodies(d_bodies, dt, gravity, device=True)[0]
            d_states, d_exp = rt.step_exposure(d_states, d_m, dt, device=True)
            rt.step_eyes(d_eyes, d_bodies, dt)
            rt.eye_views(d_eyes, d_bodies, d_rot, d_exp, params, d_m, d_table, d_rays, d_status)
            d_cursor = rt.cursor_raycast(d_rays, 6.0, device=True)
            d_frames = rt.draw_views(d_table, opts, device=True, size=vp.framebuffer_size).result()
            got = [x.clone() for x in (d_bodies, d_states, d_eyes, d_m, d_table, d_cursor, d_frames, d_status)]
        side.synchronize()
        label = f"tick {tick}"
        assert eyeorc.same_bytes(records(got[0], abi.BODY_DTYPE), bodies), label
        assert eyeorc.same_bytes(records(got[1], abi.EXPOSURE_STATE_DTYPE), states), label
        assert eyeorc.same_bytes(records(got[2], abi.EYE_DTYPE), eyes), label
        assert eyeorc.same_bytes(got[3].cpu().numpy(), m), label
        assert (got[7].cpu().numpy() == 0).all(), label
        assert eyeorc.same_bytes(got[4].cpu().numpy(), np.concatenate([np.frombuffer(bytes(c.data), np.uint8)
                                                                        for c in cams]).reshape(n, 144)), label
        assert eyeorc.same_bytes(records(got[5], abi.CURSOR_DTYPE), np.concatenate(cursors)), label
        f = got[6].cpu().numpy().reshape(n, -1, 4)
        for i in range(n):
            assert np.array_equal(f[i], frames[i]), f"{label}: frame {i}"
    assert np.abs(eyes["displacement_pos"]).max() > 0.0   # the eyes moved
    assert len({float(c.data.exposure) for c in cams}) > 1   # the exposures differ between characters
    rt.close()
