"""Batches of views (aicb_render_views_* and aicb_group_render_views_*): every view must equal the single-camera call for
its camera byte for byte, in every output form, and the batch's info must be the sum of the single calls'.  One H100
is enough for the groups: the same device is named several times, each name its own context."""
import ctypes as C

import numpy as np
import pytest

import aicb200
import orc
from aicb200 import (FOG_PHYSICAL, LIGHT_BOUNCE, LIGHT_COARSE, LIGHT_FLAT, LIGHT_LINEAR, LIGHT_NONE, LIGHT_SMOOTHSTEP,
                     TONE_REINHARD, TRANSPARENCY_THRESHOLD, TRANSPARENCY_VOLUMETRIC, AicbError, Block, Context,
                     DeviceGroup, GraphicsOptions, SpaceRaytracer, Space, abi, scenes)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KINDS = ("srgb8", "rgba16f", "colorbuf", "text")


def wide_scene(n=10, n_blocks=16400, seed=11):
    """More than 16384 block ids: the scene keeps 32-bit cells."""
    rng = np.random.default_rng(seed)
    blocks = [Block.air()] + [Block(color=(((i * 37) % 255) / 255.0, ((i * 91) % 255) / 255.0,
                                           ((i * 13) % 255) / 255.0, 1.0)) for i in range(1, n_blocks)]
    ids = rng.integers(0, n_blocks, size=(n, n, n))
    ids = np.where(rng.random((n, n, n)) < 0.25, ids, 0).astype(np.uint16)
    ids[0, 0, 0] = n_blocks - 1
    return Space((0, 0, 0), ids, blocks)


def faint_slab():
    """40 x 24 x 24 cubes of two faint transparent blocks, 19 to 65 surfaces per ray seen end on: more than a fresh
    context's hit stream holds."""
    n, m = 40, 24
    x, y, z = np.meshgrid(np.arange(n), np.arange(m), np.arange(m), indexing="ij")
    ids = (1 + (x + y + z) % 2).astype(np.uint16)
    return Space((0, 0, 0), ids, [Block.air(), Block(color=(0.9, 0.5, 0.2, 0.03)), Block(color=(0.2, 0.4, 0.9, 0.02))])


@pytest.fixture(scope="module")
def spaces():
    return {
        "mixed": scenes.small_mixed_scene(n=12, seed=7),                      # transparent, voxels, light, octant sky
        "c2": scenes.config_c2(n=16, n_voxel_blocks=6),                       # mixed transparent, res-1 and res-16
        "res16": scenes.config_c1(n=16, n_voxel_blocks=8, resolution=16),    # voxel bricks
        "wide": wide_scene(),                                                  # 32-bit cells
    }


DIRECTIONS = [(1.0, 0.6, 1.0), (-1.0, 0.3, 0.5), (0.2, -1.0, 0.4), (0.7, 0.1, -1.0), (-0.4, 0.8, -0.6),
              (1.0, -0.2, -0.3), (0.0, 1.0, 0.1)]


def cameras_for(space, opts, w, h, n):
    """n cameras of one size: distinct directions and exposures; the third inside the Space, the fifth with a far
    point whose w is not positive (its rays are NaN)."""
    cams = []
    for v in range(n):
        cam = scenes.standard_camera(space, opts, w, h, direction=DIRECTIONS[v % len(DIRECTIONS)],
                                     distance_scale=1.0 + 0.15 * (v // len(DIRECTIONS)))
        if v % 7 == 2:   # inside the Space, at its centre
            centre = [space.lower[a] + space.size[a] / 2.0 for a in range(3)]
            cam.look_at_y_up(np.array(centre) + 0.3, np.array(centre) + np.array(DIRECTIONS[v % 7]))
        cam.data.exposure = [1.0, 0.5, 1.75, 2.5, 0.8, 1.25, 3.0][v % 7]
        if v % 7 == 4:   # w(far) <= 0
            m = cam.data.inverse_projection_view
            m[3], m[7], m[11], m[15] = 0.0, 0.0, -2.0, 1.0
        cams.append(cam)
    return cams


def single(rt, cam, opts, kind):
    """The single-camera host call of `kind` on the scene: (outputs, RenderInfo)."""
    lib = aicb200.load_library()
    n = cam.data.fb_width * cam.data.fb_height
    info = abi.RenderInfo()
    o = opts.to_abi(True)
    if kind == "colorbuf":
        cb, depth = np.empty((n, 4), np.float32), np.empty(n, np.float64)
        hit, steps = np.empty((n, 8), np.int32), np.empty(n, np.uint32)
        assert lib.aicb_render_colorbuf(rt.handle, C.byref(cam.data), C.byref(o), None, cb.ctypes.data,
                                        depth.ctypes.data, hit.ctypes.data, steps.ctypes.data, n,
                                        C.byref(info)) == abi.OK, lib.aicb_last_error()
        return {"colorbuf": cb, "depth": depth, "hit": hit, "steps": steps}, aicb200.RenderInfo.from_abi(info)
    dtype, width = {"srgb8": (np.uint8, 4), "rgba16f": (np.uint16, 4), "text": (np.int32, 1)}[kind]
    out = np.empty((n, width), dtype)
    fn = getattr(lib, "aicb_render_" + kind)
    args = (rt.handle, C.byref(cam.data), C.byref(o)) + ((None,) if kind != "text" else ())
    assert fn(*args, out.ctypes.data, n, C.byref(info)) == abi.OK, lib.aicb_last_error()
    return out, aicb200.RenderInfo.from_abi(info)


def as_bytes(x):
    x = x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x)
    return np.ascontiguousarray(x).tobytes()


def check_batch(got, refs, kind, label):
    """got: the batch's output of `kind` (dict for colorbuf); refs: the single calls' outputs, view by view."""
    for v, ref in enumerate(refs):
        if kind == "colorbuf":
            for name in ("colorbuf", "depth", "hit", "steps"):
                assert as_bytes(got[name][v]) == as_bytes(ref[name]), f"{label}: view {v} {name}"
        else:
            assert as_bytes(got[v]) == as_bytes(ref), f"{label}: view {v}"


def check_info(info, infos, label):
    assert info.cubes_traced == sum(i.cubes_traced for i in infos), label
    assert info.rays == sum(i.rays for i in infos), label
    for k in range(6):
        assert info.counters[k] == sum(i.counters[k] for i in infos), (label, k)
    assert info.flaws == 0


def batch_and_singles(rt, cams, opts, kind):
    singles = [single(rt, c, opts, kind) for c in cams]
    return [s[0] for s in singles], [s[1] for s in singles]


OPTIONS = {
    "none": dict(lighting_display=LIGHT_NONE),
    "flat": dict(lighting_display=LIGHT_FLAT),
    "coarse": dict(lighting_display=LIGHT_COARSE),
    "linear_fog": dict(lighting_display=LIGHT_LINEAR, fog=FOG_PHYSICAL),
    "smoothstep": dict(lighting_display=LIGHT_SMOOTHSTEP),
    "bounce": dict(lighting_display=LIGHT_BOUNCE, bounce_samples=2),
    "volumetric": dict(transparency=TRANSPARENCY_VOLUMETRIC),
    "threshold": dict(transparency=TRANSPARENCY_THRESHOLD, transparency_threshold=0.4),
    "aa": dict(antialiasing_always=True),
    "reinhard": dict(tone_mapping=TONE_REINHARD, maximum_intensity=0.7),
    "debug_pixel_cost": dict(debug_pixel_cost=True),
}


@pytest.mark.parametrize("option", sorted(OPTIONS))
def test_each_view_equals_the_single_call_for_every_option(spaces, option):
    space = spaces["mixed"]
    opts = GraphicsOptions(view_distance=60.0, **OPTIONS[option])
    rt = SpaceRaytracer(space, opts)
    cams = cameras_for(space, opts, 37, 23, 7)
    for kind in KINDS:
        refs, infos = batch_and_singles(rt, cams, opts, kind)
        got = {"srgb8": rt.draw_views, "rgba16f": rt.draw_views_rgba16f, "colorbuf": rt.draw_views_colorbuf,
               "text": rt.render_views_text}[kind](cams, opts)
        if kind == "rgba16f":
            got = got.view(np.uint16)
        check_batch(got, refs, kind, f"{option} {kind}")
        if kind == "colorbuf":
            check_info(got["info"], infos, f"{option} info")
    rt.close()


def test_no_sky():
    space = scenes.small_mixed_scene(n=12, seed=7)
    opts = GraphicsOptions(lighting_display=LIGHT_LINEAR, view_distance=60.0)
    rt = SpaceRaytracer(space, opts)
    cams = cameras_for(space, opts, 16, 16, 3)
    o = opts.to_abi(False)
    lib = aicb200.load_library()
    table = aicb200.camera_table(cams)
    out = np.empty((3 * 256, 4), np.float32)
    assert lib.aicb_render_views_colorbuf(rt.handle, table.ctypes.data, 3, C.byref(o), out.ctypes.data, None, None,
                                          None, out.shape[0], None) == abi.OK
    for v, cam in enumerate(cams):
        ref = np.empty((256, 4), np.float32)
        assert lib.aicb_render_colorbuf(rt.handle, C.byref(cam.data), C.byref(o), None, ref.ctypes.data, None, None,
                                        None, 256, None) == abi.OK
        assert out[v * 256:(v + 1) * 256].tobytes() == ref.tobytes(), v
    rt.close()


@pytest.mark.parametrize("name", ["c2", "res16", "wide"])
@pytest.mark.parametrize("n_views,size", [(1, (64, 64)), (2, (1, 1)), (7, (37, 23)), (33, (16, 12))])
def test_scenes_and_shapes(spaces, name, n_views, size):
    space = spaces[name]
    opts = GraphicsOptions(lighting_display=LIGHT_FLAT, view_distance=100.0)
    rt = SpaceRaytracer(space, opts)
    cams = cameras_for(space, opts, size[0], size[1], n_views)
    for kind in ("srgb8", "colorbuf"):
        refs, infos = batch_and_singles(rt, cams, opts, kind)
        got = rt.draw_views(cams, opts) if kind == "srgb8" else rt.draw_views_colorbuf(cams, opts)
        check_batch(got, refs, kind, f"{name} {n_views} {size} {kind}")
        if kind == "colorbuf":
            check_info(got["info"], infos, name)
    rt.close()


def test_empty_batches(spaces):
    space = spaces["mixed"]
    opts = GraphicsOptions()
    rt = SpaceRaytracer(space, opts)
    lib = aicb200.load_library()
    o = opts.to_abi(True)
    info = abi.RenderInfo()
    assert lib.aicb_render_views_srgb8(rt.handle, None, 0, C.byref(o), None, 0, C.byref(info)) == abi.OK
    assert info.rays == 0 and info.cubes_traced == 0
    cams = cameras_for(space, opts, 8, 5, 3)
    for cam in cams:
        cam.data.fb_width = 0
    assert rt.draw_views(cams, opts).shape == (3, 5, 0, 4)
    d = rt.draw_views(cams, opts, device=True).result()
    assert tuple(d.shape) == (3, 5, 0, 4)
    assert rt.draw_views([], opts, device=True, size=(4, 4)).result().numel() == 0
    rt.close()


def test_a_batch_of_several_chunks(spaces):
    """3 views of 1024 x 768 with 4 samples: 9.4 M tasks, past the 4 M task chunk, whose boundary falls inside a
    view."""
    space = spaces["c2"]
    opts = GraphicsOptions(lighting_display=LIGHT_FLAT, antialiasing_always=True, view_distance=100.0)
    rt = SpaceRaytracer(space, opts)
    cams = cameras_for(space, opts, 1024, 768, 3)
    refs, infos = batch_and_singles(rt, cams, opts, "colorbuf")
    got = rt.draw_views_colorbuf(cams, opts)
    check_batch(got, refs, "colorbuf", "chunks")
    check_info(got["info"], infos, "chunks")
    refs8, _ = batch_and_singles(rt, cams, opts, "srgb8")
    check_batch(rt.draw_views(cams, opts), refs8, "srgb8", "chunks srgb8")
    rt.close()


def test_a_deep_batch_is_reissued():
    """The faint slab overflows a fresh context's hit stream: the host call re-issues the batch, and the device call
    returns AICB_ERR_RETRY from aicb_render_finish until the stream is large enough."""
    space = faint_slab()
    opts = GraphicsOptions(lighting_display=LIGHT_NONE, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0)
    cams = [scenes.standard_camera(space, opts, 128, 96, direction=d, distance_scale=0.5)
            for d in [(1.0, 0.04, 0.03), (1.0, -0.05, 0.02), (-1.0, 0.03, -0.04)]]
    warm = SpaceRaytracer(space, opts)
    refs, infos = batch_and_singles(warm, cams, opts, "colorbuf")
    refs8, _ = batch_and_singles(warm, cams, opts, "srgb8")
    for form in ("host", "device"):
        ctx = Context()
        try:
            rt = SpaceRaytracer(space, opts, ctx)
            if form == "host":
                got = rt.draw_views_colorbuf(cams, opts)
                check_batch(got, refs, "colorbuf", "deep host")
                check_info(got["info"], infos, "deep host")
            else:
                lib = aicb200.load_library()
                table = torch.from_numpy(aicb200.camera_table(cams).view(np.uint8).reshape(3, -1)).cuda()
                buf = torch.empty((3, 96, 128, 4), dtype=torch.uint8, device="cuda")
                outs = abi.DeviceOutputs(srgb8=buf.data_ptr(), len=buf.numel() // 4)
                o = opts.to_abi(True)
                issue = lambda: lib.aicb_render_views_device(rt.handle, table.data_ptr(), 3, 128, 96, C.byref(o),
                                                             C.byref(outs), None)
                assert issue() == abi.OK
                assert lib.aicb_render_finish(rt.handle, None) == abi.ERR_RETRY
                statuses = []
                while not statuses or statuses[-1] == abi.ERR_RETRY:
                    assert issue() == abi.OK and len(statuses) < 4
                    statuses.append(lib.aicb_render_finish(rt.handle, None))
                assert statuses[-1] == abi.OK
                check_batch(buf, [r.reshape(96, 128, 4) for r in refs8], "srgb8", "deep device")
            rt.close()
        finally:
            ctx.close()
    warm.close()


def test_device_form_on_a_side_stream(spaces):
    space = spaces["mixed"]
    opts = GraphicsOptions(lighting_display=LIGHT_LINEAR, view_distance=60.0)
    rt = SpaceRaytracer(space, opts)
    cams = cameras_for(space, opts, 37, 23, 7)
    side = torch.cuda.Stream()
    for kind in KINDS:
        refs, infos = batch_and_singles(rt, cams, opts, kind)
        with torch.cuda.stream(side):
            table = torch.from_numpy(aicb200.camera_table(cams).view(np.uint8).reshape(7, -1)).to("cuda")
            call = {"srgb8": rt.draw_views, "rgba16f": rt.draw_views_rgba16f, "colorbuf": rt.draw_views_colorbuf,
                    "text": rt.render_views_text}[kind]
            r = call(table, opts, device=True, size=(37, 23))
            got = r.result()
        side.synchronize()
        if kind == "rgba16f":
            got = got.view(torch.int16)
            refs = [x.view(np.int16) for x in refs]
        check_batch(got, refs, kind, f"device {kind}")
        if kind == "colorbuf":
            check_info(r.info, infos, "device info")
    # a list of cameras goes through the same call
    refs, _ = batch_and_singles(rt, cams, opts, "srgb8")
    check_batch(rt.draw_views(cams, opts, device=True).result(), refs, "srgb8", "device list")
    rt.close()


def test_device_form_rejects_host_and_misaligned_pointers(spaces):
    space = spaces["mixed"]
    opts = GraphicsOptions()
    rt = SpaceRaytracer(space, opts)
    cams = cameras_for(space, opts, 8, 8, 2)
    lib = aicb200.load_library()
    o = opts.to_abi(True)
    host_table = aicb200.camera_table(cams)
    dev_table = torch.from_numpy(host_table.view(np.uint8).reshape(2, -1)).cuda()
    raw = torch.zeros(2 * 144 + 8, dtype=torch.uint8, device="cuda")
    buf = torch.full((2 * 64, 4), 7, dtype=torch.uint8, device="cuda")
    outs = abi.DeviceOutputs(srgb8=buf.data_ptr(), len=128)
    assert lib.aicb_render_views_device(rt.handle, host_table.ctypes.data, 2, 8, 8, C.byref(o), C.byref(outs),
                                        None) == abi.ERR_INVALID
    assert lib.aicb_render_views_device(rt.handle, raw.data_ptr() + 4, 2, 8, 8, C.byref(o), C.byref(outs),
                                        None) == abi.ERR_INVALID
    host_out = np.zeros((128, 4), np.uint8)
    bad = abi.DeviceOutputs(srgb8=host_out.ctypes.data, len=128)
    assert lib.aicb_render_views_device(rt.handle, dev_table.data_ptr(), 2, 8, 8, C.byref(o), C.byref(bad),
                                        None) == abi.ERR_INVALID
    mis = abi.DeviceOutputs(srgb8=buf.data_ptr() + 2, len=128)
    assert lib.aicb_render_views_device(rt.handle, dev_table.data_ptr(), 2, 8, 8, C.byref(o), C.byref(mis),
                                        None) == abi.ERR_INVALID
    wrong_len = abi.DeviceOutputs(srgb8=buf.data_ptr(), len=127)
    assert lib.aicb_render_views_device(rt.handle, dev_table.data_ptr(), 2, 8, 8, C.byref(o), C.byref(wrong_len),
                                        None) == abi.ERR_INVALID
    torch.cuda.synchronize()
    assert bool((buf == 7).all())
    rt.close()


def test_rejected_batches_write_nothing(spaces):
    space = spaces["mixed"]
    opts = GraphicsOptions()
    rt = SpaceRaytracer(space, opts)
    lib = aicb200.load_library()
    o = opts.to_abi(True)
    cams = cameras_for(space, opts, 8, 8, 3)
    odd = cameras_for(space, opts, 8, 9, 1)
    table = aicb200.camera_table(cams[:2] + odd)
    out = np.full((3 * 64, 4), 7, np.uint8)
    assert lib.aicb_render_views_srgb8(rt.handle, table.ctypes.data, 3, C.byref(o), out.ctypes.data, 3 * 64,
                                       None) == abi.ERR_INVALID                              # mismatched sizes
    table = aicb200.camera_table(cams)
    assert lib.aicb_render_views_srgb8(rt.handle, table.ctypes.data, 3, C.byref(o), out.ctypes.data, 3 * 64 - 1,
                                       None) == abi.ERR_INVALID                              # wrong out_len
    assert lib.aicb_render_views_srgb8(rt.handle, None, 3, C.byref(o), out.ctypes.data, 3 * 64,
                                       None) == abi.ERR_INVALID                              # NULL cameras
    big = cameras_for(space, opts, 8192, 8192, 1)[0]
    big_table = aicb200.camera_table([big] * 65)   # 65 * 2^26 tasks >= 2^32
    assert lib.aicb_render_views_srgb8(rt.handle, big_table.ctypes.data, 65, C.byref(o), None, 65 * 8192 * 8192,
                                       None) == abi.ERR_INVALID
    assert b"2^32" in lib.aicb_last_error()
    aa = GraphicsOptions(antialiasing_always=True).to_abi(True)
    big_table = aicb200.camera_table([big] * 16)   # 16 * 2^26 * 4 samples
    assert lib.aicb_render_views_srgb8(rt.handle, big_table.ctypes.data, 16, C.byref(aa), None, 16 * 8192 * 8192,
                                       None) == abi.ERR_INVALID
    assert b"2^32" in lib.aicb_last_error()
    assert (out == 7).all()
    with pytest.raises(AicbError):
        rt.draw_views(cams[:2] + odd, opts)
    rt.close()


@pytest.mark.parametrize("devices", [[0], [0, 0], [0, 0, 0]])
@pytest.mark.parametrize("n_views", [2, 7])
def test_groups_equal_one_context(spaces, devices, n_views):
    space = spaces["mixed"]
    opts = GraphicsOptions(lighting_display=LIGHT_LINEAR, antialiasing_always=n_views == 7, view_distance=60.0)
    rt = SpaceRaytracer(space, opts)
    cams = cameras_for(space, opts, 37, 23, n_views)
    ref = {kind: batch_and_singles(rt, cams, opts, kind) for kind in KINDS}
    g = DeviceGroup(devices)
    try:
        g.update(space)
        for kind in KINDS:
            refs, infos = ref[kind]
            call = {"srgb8": g.draw_views, "rgba16f": g.draw_views_rgba16f, "colorbuf": g.draw_views_colorbuf,
                    "text": g.render_views_text}[kind]
            got = call(cams, opts)
            check_batch(got.view(np.uint16) if kind == "rgba16f" else got, refs, kind, f"group {len(devices)} {kind}")
            if kind == "colorbuf":
                check_info(got["info"], infos, "group info")
            dev = call(cams, opts, device=True)
            torch.cuda.synchronize()
            check_batch(dev.view(torch.int16) if kind == "rgba16f" else dev,
                        [r.view(np.int16) for r in refs] if kind == "rgba16f" else refs, kind,
                        f"group device {len(devices)} {kind}")
    finally:
        g.close()
        rt.close()


def test_three_views_against_the_oracle(spaces):
    space = spaces["mixed"]
    opts = GraphicsOptions(fog=aicb200.FOG_ABRUPT, lighting_display=LIGHT_LINEAR,
                           transparency=TRANSPARENCY_VOLUMETRIC, view_distance=60.0)
    cams = [scenes.standard_camera(space, opts, 24, 16, direction=d) for d in DIRECTIONS[:3]]
    for cam, e in zip(cams, (1.0, 0.6, 1.4)):
        cam.data.exposure = e
    rt = SpaceRaytracer(space, opts)
    got = rt.draw_views(cams, opts)
    cb = rt.draw_views_colorbuf(cams, opts)
    orc.set_libm(orc.LIBM_CR)
    oracle = orc.OracleScene(space)
    for v, cam in enumerate(cams):
        ref = oracle.render(cam, opts)
        assert np.array_equal(cb["hit"][v], ref["hit"]), v
        assert np.array_equal(cb["steps"][v], ref["steps"]), v
        assert orc.max_ulp_diff(cb["colorbuf"][v], ref["colorbuf"]) == 0, v
        assert np.array_equal(got[v].reshape(-1, 4), ref["srgb8"]), v
    rt.close()
