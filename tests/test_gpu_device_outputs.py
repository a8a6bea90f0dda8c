"""Outputs in the caller's device memory (aicb_render_device, aicb_trace_rays_device, aicb_render_layers_device and their
group forms), through the Python layer's device=True / CUDA-tensor calls: every output must equal the host call's byte
for byte, with the same counters; the asynchronous calls follow the caller's stream, finish with one re-issue after a
hit-stream overflow, and reject host memory, another device's memory, wrong lengths and output sets no call gives before
anything is issued.  One H100 is enough: groups name the same device several times."""
import ctypes as C

import numpy as np
import pytest

import aicb200
from aicb200 import (FOG_NONE, FOG_PHYSICAL, LIGHT_BOUNCE, LIGHT_FLAT, LIGHT_LINEAR, LIGHT_NONE,
                     TRANSPARENCY_VOLUMETRIC, Block, Context, DeviceGroup, GraphicsOptions, RtRenderer, Space,
                     SpaceRaytracer, abi, scenes)

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

GROUPS = ([0, 0], [0, 0, 0])
NO_WORLD = (0.74, 0.74, 0.74, 1.0)


@pytest.fixture(scope="module")
def spaces():
    return {"mixed": scenes.small_mixed_scene(n=12, seed=7),
            "voxel": scenes.config_c1(n=16, n_voxel_blocks=8, resolution=16),
            "c2": scenes.config_c2(n=16, n_voxel_blocks=6)}


def host(x):
    return x.cpu().numpy() if torch.is_tensor(x) else x


def faint_slab():
    """test_gpu_resolve's deep scene: 40 x 24 x 24 cubes of two faint transparent blocks, 19 to 65 surfaces per ray
    seen end on, more than a fresh context's hit stream holds."""
    n, m = 40, 24
    x, y, z = np.meshgrid(np.arange(n), np.arange(m), np.arange(m), indexing="ij")
    ids = (1 + (x + y + z) % 2).astype(np.uint16)
    return Space((0, 0, 0), ids, [Block.air(), Block(color=(0.9, 0.5, 0.2, 0.03)), Block(color=(0.2, 0.4, 0.9, 0.02))])


def same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    a, b = np.ascontiguousarray(host(a)), np.ascontiguousarray(host(b))
    return a.nbytes == b.nbytes and a.tobytes() == b.tobytes()


def same_counts(a, b):
    return (a.cubes_traced, a.rays, a.counters, a.algorithmic_bytes) == \
        (b.cubes_traced, b.rays, b.counters, b.algorithmic_bytes)


def text_info(r, cam, opts):
    out = np.zeros(cam.data.fb_width * cam.data.fb_height, dtype=np.int32)
    info, o = abi.RenderInfo(), opts.to_abi(True)
    assert aicb200.load_library().aicb_render_text(r.rt.handle, C.byref(cam.data), C.byref(o), out.ctypes.data,
                                                   out.size, C.byref(info)) == abi.OK
    return aicb200.RenderInfo.from_abi(info)


# (space, options, framebuffer size, shard)
FRAMES = {
    "mixed": ("mixed", {}, (48, 40), None),
    "voxel": ("voxel", {}, (40, 33), None),
    "c2": ("c2", {}, (48, 40), None),
    "aa": ("mixed", dict(antialiasing_always=True), (40, 33), None),
    "odd_37x23": ("mixed", dict(antialiasing_always=True), (37, 23), None),
    "flat": ("mixed", dict(lighting_display=LIGHT_FLAT), (40, 33), None),
    "linear_fog": ("mixed", dict(lighting_display=LIGHT_LINEAR, fog=FOG_PHYSICAL), (40, 33), None),
    "bounce": ("mixed", dict(lighting_display=LIGHT_BOUNCE, bounce_samples=2), (40, 33), None),
    "debug_pixel_cost": ("mixed", dict(debug_pixel_cost=True), (40, 33), None),
    "shard": ("mixed", {}, (40, 50), (16, 1, 3)),
}


@pytest.mark.parametrize("case", list(FRAMES))
def test_world_frames_equal_the_host_calls(spaces, case):
    name, kw, (w, h), shard = FRAMES[case]
    space = spaces[name]
    opts = GraphicsOptions(view_distance=40.0, exposure=1.5, **kw)
    cam = scenes.standard_camera(space, opts, w, h)
    r = RtRenderer(cam)
    r.update(space)
    ref = r.draw(shard=shard)
    ref_16 = r.draw_rgba16f(shard=shard)
    ref_cb = r.draw_colorbuf(shard=shard)
    got = r.draw(shard=shard, device=True).result()
    assert got.data.is_cuda and same_bits(got.data, ref.data) and same_counts(got.info, ref.info), case
    assert same_bits(r.draw_rgba16f(shard=shard, device=True).result(), ref_16), case
    cb = r.draw_colorbuf(shard=shard, device=True).result()
    for k in ("colorbuf", "depth", "hit", "steps"):
        assert same_bits(cb[k], ref_cb[k]), f"{case} {k}"
    assert same_counts(cb["info"], ref_cb["info"]), case
    some = r.draw_colorbuf(shard=shard, want_depth=False, want_steps=False, device=True).result()
    assert some["depth"] is None and same_bits(some["hit"], ref_cb["hit"]), case
    if shard is None:
        ref_text = r.render_text()
        call = r.render_text(device=True)
        assert same_bits(call.result(), ref_text), case
        assert same_counts(call.info, text_info(r, cam, opts)), case
        for devices in GROUPS:
            g = DeviceGroup(devices)
            g.update(space)
            gd = g.draw(cam, opts, device=True)
            assert same_bits(gd.data, ref.data) and same_counts(gd.info, ref.info), f"{case} {devices}"
            assert same_bits(g.draw_rgba16f(cam, opts, device=True), ref_16), f"{case} {devices}"
            gcb = g.draw_colorbuf(cam, opts, device=True)
            for k in ("colorbuf", "depth", "hit", "steps"):
                assert same_bits(gcb[k], ref_cb[k]), f"{case} {devices} {k}"
            assert same_counts(gcb["info"], ref_cb["info"]), f"{case} {devices}"
            assert same_bits(g.render_text(cam, opts, device=True), ref_text), f"{case} {devices}"
            g.close()
    r.rt.close()


def test_full_frame_stores_the_shard_at_framebuffer_positions(spaces):
    space = spaces["mixed"]
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(space, opts, 40, 50)
    r = RtRenderer(cam)
    r.update(space)
    whole = r.draw().data
    frame = torch.zeros((50, 40, 4), dtype=torch.uint8, device="cuda")
    lib, o = aicb200.load_library(), opts.to_abi(True)
    for index in range(3):
        outs = abi.DeviceOutputs(srgb8=frame.data_ptr(), len=40 * 50, full_frame=1)
        s = abi.Shard(16, index, 3)
        assert lib.aicb_render_device(r.rt.handle, C.byref(cam.data), C.byref(o), C.byref(s), C.byref(outs),
                                      None) == abi.OK
        assert lib.aicb_render_finish(r.rt.handle, None) == abi.OK
    assert same_bits(frame, whole)
    r.rt.close()


def ray_batch(space, n, seed):
    rng = np.random.default_rng(seed)
    lo, size = np.array(space.lower, np.float64), np.array(space.size, np.float64)
    o = lo + rng.uniform(-0.5, 1.5, size=(n, 3)) * size
    d = rng.normal(size=(n, 3))
    d[rng.random(n) < 0.02] = 0.0
    return np.concatenate([o, d], axis=1)


@pytest.mark.parametrize("n", [0, 1, 33, 100_003])
def test_ray_batches_from_a_cuda_tensor_equal_the_host_batch(spaces, n):
    space = spaces["mixed"]
    rt = SpaceRaytracer(space, GraphicsOptions(view_distance=40.0))
    rays = ray_batch(space, n, seed=n + 5)
    d_rays = torch.from_numpy(rays).cuda()
    for sky in (True, False):
        ref = rt.trace_rays(rays, sky, True, True, True)
        got = rt.trace_rays(d_rays, sky, True, True, True).result()
        for k in ("colorbuf", "depth", "hit", "steps"):
            assert same_bits(got[k], ref[k]), f"n={n} sky={sky} {k}"
        assert same_counts(got["info"], ref["info"])
        for devices in GROUPS:
            g = DeviceGroup(devices)
            g.update(space)
            gg = g.trace_rays(d_rays, rt.graphics_options, sky, True, True, True)
            for k in ("colorbuf", "depth", "hit", "steps"):
                assert same_bits(gg[k], ref[k]), f"n={n} {devices} sky={sky} {k}"
            assert same_counts(gg["info"], ref["info"])
            g.close()
    rt.close()


def layer_setup(aa):
    mixed = scenes.small_mixed_scene(n=12, seed=7)
    ui_space = scenes.small_mixed_scene(n=6, seed=11, lower=(0, 0, 0))
    wopts = GraphicsOptions(view_distance=40.0, antialiasing_always=aa, exposure=1.75)
    uopts = GraphicsOptions(view_distance=30.0, fog=FOG_NONE, lighting_display=LIGHT_FLAT, exposure=0.625,
                            antialiasing_always=aa)
    wcam = scenes.standard_camera(mixed, wopts, 64, 48)
    ucam = scenes.standard_camera(ui_space, uopts, 64, 48, direction=(0.2, 0.1, 1.0), distance_scale=1.6)
    return mixed, ui_space, wopts, uopts, wcam, ucam


LAYER_CASES = [(True, True, None), (True, True, (0.1, 0.3, 0.6, 0.5)), (True, False, (0.1, 0.3, 0.6, 0.5)),
               (True, False, None), (False, True, None)]


def check_layers(world, ui, backdrop, m, px, call, label):
    """Every layered output of `call` (a device-output function) against the host calls on one context."""
    ref = aicb200.render_layers(world, ui, backdrop, NO_WORLD)
    got = call("srgb8", world, ui, backdrop)
    assert same_bits(got.data, ref.data) and same_counts(got.info, ref.info), label
    ref_t = aicb200.render_layers_terminal(world, ui, backdrop, NO_WORLD)
    got_t = call("terminal", world, ui, backdrop)
    for k in ("text", "layer", "rgba"):
        assert same_bits(got_t[k], ref_t[k]), f"{label} terminal {k}"
    assert same_counts(got_t["info"], ref_t["info"]), label
    for pixels in (None, px):
        ref_rgba, ref_depth, ref_info = aicb200.render_layers_texture(world, ui, backdrop, NO_WORLD, m, pixels=pixels)
        rgba, depth, info = call("texture", world, ui, backdrop, m, pixels)
        assert same_bits(rgba, ref_rgba) and same_bits(depth, ref_depth), f"{label} texture list={pixels is not None}"
        assert same_counts(info, ref_info), label


@pytest.mark.parametrize("aa", [False, True])
def test_layered_outputs_equal_the_host_calls(aa):
    mixed, ui_space, wopts, uopts, wcam, ucam = layer_setup(aa)
    wrt = SpaceRaytracer(mixed, wopts)
    urt = SpaceRaytracer(ui_space, uopts, wrt.ctx)
    m = wcam.depth_transform()
    rng = np.random.default_rng(3)
    px = np.concatenate([aicb200.pixel_picker_order(64, 48, 700), rng.integers(0, 64 * 48, size=333)]).astype(np.uint32)
    d_px = torch.from_numpy(px.view(np.int32)).cuda()   # repeats included

    def one_context(kind, world, ui, backdrop, m=None, pixels=None):
        if kind == "srgb8":
            h = aicb200.render_layers(world, ui, backdrop, NO_WORLD, device=True)
        elif kind == "terminal":
            h = aicb200.render_layers_terminal(world, ui, backdrop, NO_WORLD, device=True)
        else:
            h = aicb200.render_layers_texture(world, ui, backdrop, NO_WORLD, m,
                                              pixels=None if pixels is None else d_px, device=True)
        return h.result()

    for w, u, bd in LAYER_CASES:
        check_layers((wrt, wcam, wopts) if w else None, (urt, ucam, uopts) if u else None, bd, m, px, one_context,
                     f"aa={aa} world={w} ui={u} backdrop={bd}")
    for devices in GROUPS:
        g = DeviceGroup(devices)
        gw, gu = g.add_scene(mixed), g.add_scene(ui_space)

        def on_group(kind, world, ui, backdrop, m=None, pixels=None):
            world = (gw,) + world[1:] if world else None
            ui = (gu,) + ui[1:] if ui else None
            if kind == "srgb8":
                return g.render_layers(world, ui, backdrop, NO_WORLD, device=True)
            if kind == "terminal":
                return g.render_layers_terminal(world, ui, backdrop, NO_WORLD, device=True)
            return g.render_layers_texture(world, ui, backdrop, NO_WORLD, m, pixels=None if pixels is None else d_px,
                                           device=True)

        for w, u, bd in LAYER_CASES:
            check_layers((wrt, wcam, wopts) if w else None, (urt, ucam, uopts) if u else None, bd, m, px,
                         lambda kind, world, ui, backdrop, *a: on_group(kind, world, ui, backdrop, *a),
                         f"{devices} aa={aa} world={w} ui={u} backdrop={bd}")
        g.close()
    urt.close()
    wrt.close()


def test_stream_order_without_synchronising(spaces):
    """A frame issued on a side stream, a reduction of it queued behind it on that stream: the reduction sees the
    finished frame with no synchronisation but the one result() makes.  A second frame into the same tensors after a
    scene update shows the new cells."""
    space = spaces["mixed"]
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(space, opts, 96, 64)
    r = RtRenderer(cam)
    r.update(space)
    ref = r.draw_colorbuf()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        out = {"colorbuf": torch.full((96 * 64, 4), float("nan"), device="cuda"),
               "depth": torch.empty(96 * 64, dtype=torch.float64, device="cuda")}
        call = r.draw_colorbuf(want_hit=False, want_steps=False, device=True, out=out)
        total = out["colorbuf"].double().sum(dim=0)
        depth_max = out["depth"].max()
    call.result()
    side.synchronize()
    assert np.array_equal(total.cpu().numpy(), torch.from_numpy(ref["colorbuf"]).double().sum(dim=0).numpy())
    assert float(depth_max) == float(ref["depth"].max())
    # the scene changes: every cube holds block 1; the second frame goes into the same tensors
    lo, size = space.lower, space.size
    cubes = np.array([[lo[0] + x, lo[1] + y, lo[2] + z] for x in range(size[0]) for y in range(size[1])
                      for z in range(size[2])], dtype=np.int32)
    r.rt.update_cubes(cubes, np.full(len(cubes), 1, dtype=np.uint16))
    with torch.cuda.stream(side):
        again = r.draw_colorbuf(want_hit=False, want_steps=False, device=True, out=out)
        total2 = out["colorbuf"].double().sum(dim=0)
    again.result()
    side.synchronize()
    ref2 = r.draw_colorbuf()
    assert not same_bits(ref2["colorbuf"], ref["colorbuf"])   # the new cells show
    assert same_bits(out["colorbuf"], ref2["colorbuf"]) and same_bits(out["depth"], ref2["depth"])
    assert np.array_equal(total2.cpu().numpy(), torch.from_numpy(ref2["colorbuf"]).double().sum(dim=0).numpy())
    r.rt.close()


def test_group_calls_start_behind_the_callers_stream(spaces):
    """A group call's devices start after the work queued on the caller's stream before the call: the ray batch is
    still being written there (behind a ~0.1 s spin) when the call is made, and every device must read the written
    rays.  Work queued after the call on that stream sees the outputs."""
    space = spaces["mixed"]
    rt = SpaceRaytracer(space, GraphicsOptions(view_distance=40.0))
    rays = ray_batch(space, 20_000, seed=11)
    ref = rt.trace_rays(rays, True, True, True, True)
    good = torch.from_numpy(rays).cuda()
    for devices in GROUPS:
        g = DeviceGroup(devices)
        g.update(space)
        d_rays = torch.zeros_like(good)   # zero rays: every output would differ from the reference
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(200_000_000)
            d_rays.copy_(good)
            got = g.trace_rays(d_rays, rt.graphics_options, True, True, True, True)
            total = got["colorbuf"].double().sum(dim=0)
        side.synchronize()
        for k in ("colorbuf", "depth", "hit", "steps"):
            assert same_bits(got[k], ref[k]), f"{devices} {k}"
        assert np.array_equal(total.cpu().numpy(), torch.from_numpy(ref["colorbuf"]).double().sum(dim=0).numpy())
        g.close()
    rt.close()


def test_an_overflowed_frame_is_reissued_by_result():
    """The faint slab's first frame on a fresh context outgrows the hit stream: aicb_render_finish returns
    AICB_ERR_RETRY once, the re-issued call finishes, and result() returns what the host call returns."""
    space = faint_slab()
    opts = GraphicsOptions(lighting_display=LIGHT_NONE, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0,
                           exposure=1.5)
    cam = scenes.standard_camera(space, opts, 128, 96, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    lib = aicb200.load_library()
    # at the ABI: RETRY once, then OK on re-issue
    ctx = Context()
    try:
        rt = SpaceRaytracer(space, opts, ctx)
        buf = torch.empty((128 * 96, 4), dtype=torch.uint8, device="cuda")
        outs = abi.DeviceOutputs(srgb8=buf.data_ptr(), len=128 * 96)
        o = opts.to_abi(True)
        issue = lambda: lib.aicb_render_device(rt.handle, C.byref(cam.data), C.byref(o), None, C.byref(outs), None)
        assert issue() == abi.OK
        assert lib.aicb_render_finish(rt.handle, None) == abi.ERR_RETRY
        statuses = []
        while not statuses or statuses[-1] == abi.ERR_RETRY:   # each re-issue has a larger hit stream (x4)
            assert issue() == abi.OK and len(statuses) < 4
            statuses.append(lib.aicb_render_finish(rt.handle, None))
        assert statuses[-1] == abi.OK
        assert same_bits(buf.reshape(96, 128, 4), ref_ctx_free_draw(space, opts, cam))
        rt.close()
    finally:
        ctx.close()
    # through result(): each call on a fresh context, against the host call on a warmed one
    warm = RtRenderer(cam)
    warm.update(space)
    ref, ref_cb = warm.draw(), warm.draw_colorbuf()
    mcam = cam.depth_transform()
    px = aicb200.pixel_picker_order(128, 96, 1500)
    ref_tex = aicb200.render_layers_texture((warm.rt, cam, opts), None, None, NO_WORLD, mcam, pixels=px)
    ref_lay = aicb200.render_layers((warm.rt, cam, opts), (warm.rt, cam, opts), None, NO_WORLD)
    for call in ("draw", "colorbuf", "texture", "layers_two_passes"):
        ctx = Context()
        try:
            r = RtRenderer(cam, ctx)
            r.update(space)
            if call == "draw":
                h = r.draw(device=True)
                assert same_bits(h.result().data, ref.data) and same_counts(h.info, ref.info)
            elif call == "colorbuf":
                got = r.draw_colorbuf(device=True).result()
                for k in ("colorbuf", "depth", "hit", "steps"):
                    assert same_bits(got[k], ref_cb[k]), k
                assert same_counts(got["info"], ref_cb["info"])
            elif call == "texture":
                rgba, depth, info = aicb200.render_layers_texture((r.rt, cam, opts), None, None, NO_WORLD, mcam,
                                                                  pixels=torch.from_numpy(px.view(np.int32)).cuda(),
                                                                  device=True).result()
                assert same_bits(rgba, ref_tex[0]) and same_bits(depth, ref_tex[1])
                assert same_counts(info, ref_tex[2])
            else:   # the UI pass overflows; the world pass continues its frame
                got = aicb200.render_layers((r.rt, cam, opts), (r.rt, cam, opts), None, NO_WORLD, device=True).result()
                assert same_bits(got.data, ref_lay.data) and same_counts(got.info, ref_lay.info)
            r.rt.close()
        finally:
            ctx.close()
    warm.rt.close()


def test_retry_reads_the_arguments_of_the_issue():
    """A re-issue after an overflow reads the same backdrop, no-world colour and depth transform as the first issue,
    however much host memory is allocated and written between the issue and result()."""
    space = faint_slab()
    opts = GraphicsOptions(lighting_display=LIGHT_NONE, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0,
                           exposure=1.5)
    cam = scenes.standard_camera(space, opts, 96, 64, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    m, backdrop = cam.depth_transform(), (0.1, 0.3, 0.6, 0.5)
    warm = RtRenderer(cam)
    warm.update(space)
    ref = aicb200.render_layers_texture((warm.rt, cam, opts), None, backdrop, NO_WORLD, m)
    ctx = Context()
    try:
        rt = SpaceRaytracer(space, opts, ctx)
        call = aicb200.render_layers_texture((rt, cam, opts), None, backdrop, NO_WORLD, m, device=True)
        junk = [np.full(k, 7.5, dtype=t) for _ in range(200) for k, t in ((4, np.float32), (16, np.float64))]
        rgba, depth, info = call.result()
        assert info.counters[2] > 8 * info.rays   # the first issue overflowed: result() re-issued it
        assert same_bits(rgba, ref[0]) and same_bits(depth, ref[1]) and same_counts(info, ref[2])
        del junk
        rt.close()
    finally:
        ctx.close()
    warm.rt.close()


def test_the_next_call_on_the_context_finishes_an_issued_one():
    """A context tracks one frame: a call issued before the previous asynchronous call's result() finishes that one
    first, re-issuing it after an overflow, so neither reports the other's frame."""
    space = faint_slab()
    opts = GraphicsOptions(lighting_display=LIGHT_NONE, transparency=TRANSPARENCY_VOLUMETRIC, view_distance=200.0)
    cam = scenes.standard_camera(space, opts, 96, 64, direction=(1.0, 0.04, 0.03), distance_scale=0.5)
    warm = RtRenderer(cam)
    warm.update(space)
    ref, ref_cb = warm.draw(), warm.draw_colorbuf()
    ctx = Context()
    try:
        r = RtRenderer(cam, ctx)
        r.update(space)
        first = r.draw(device=True)            # overflows the fresh context's hit stream
        second = r.draw_colorbuf(device=True)  # finishes `first` before it is issued
        assert first.info is not None
        host = r.draw()                        # a host call finishes `second`
        assert second.info is not None
        assert same_bits(first.result().data, ref.data) and same_counts(first.info, ref.info)
        got = second.result()
        for k in ("colorbuf", "depth", "hit", "steps"):
            assert same_bits(got[k], ref_cb[k]), k
        assert same_counts(got["info"], ref_cb["info"])
        assert same_bits(host.data, ref.data)
        r.rt.close()
    finally:
        ctx.close()
    warm.rt.close()


def ref_ctx_free_draw(space, opts, cam):
    r = RtRenderer(cam, Context())
    r.update(space)
    img = r.draw().data
    r.rt.close()
    r.ctx.close()
    return img


def test_rejected_outputs(spaces):
    """Host memory, a wrong length, an output set no call gives, a tensor on another device: AICB_ERR_INVALID before
    anything is issued (the next call finishes normally)."""
    space = spaces["mixed"]
    opts = GraphicsOptions(view_distance=40.0)
    cam = scenes.standard_camera(space, opts, 40, 30)
    r = RtRenderer(cam)
    r.update(space)
    ref = r.draw()
    lib, o = aicb200.load_library(), opts.to_abi(True)
    n = 40 * 30
    dev = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    hst = np.empty((n, 4), dtype=np.float32)
    pinned = torch.empty((n, 4), dtype=torch.float32).pin_memory()
    text = torch.empty(n, dtype=torch.int32, device="cuda")
    srgb = torch.empty((n, 4), dtype=torch.uint8, device="cuda")

    def render(**kw):
        outs = abi.DeviceOutputs(**{k: (v.data_ptr() if torch.is_tensor(v) else v) for k, v in kw.items()})
        return lib.aicb_render_device(r.rt.handle, C.byref(cam.data), C.byref(o), None, C.byref(outs), None)

    assert render(colorbuf=hst.ctypes.data, len=n) == abi.ERR_INVALID
    assert render(colorbuf=pinned, len=n) == abi.ERR_INVALID
    assert render(colorbuf=dev, len=n - 1) == abi.ERR_INVALID
    assert render(colorbuf=dev, text=text, len=n) == abi.ERR_INVALID
    assert render(srgb8=srgb, colorbuf=dev, len=n) == abi.ERR_INVALID
    assert render(terminal=dev, len=n) == abi.ERR_INVALID
    assert render(len=n) == abi.ERR_INVALID
    rays = torch.zeros((n, 6), dtype=torch.float64, device="cuda")
    outs = abi.DeviceOutputs(colorbuf=dev.data_ptr(), len=n)
    host_rays = np.zeros((n, 6))
    assert lib.aicb_trace_rays_device(r.rt.handle, host_rays.ctypes.data, n, C.byref(o), C.byref(outs),
                                      None) == abi.ERR_INVALID
    bad = abi.DeviceOutputs(srgb8=srgb.data_ptr(), len=n)
    assert lib.aicb_trace_rays_device(r.rt.handle, rays.data_ptr(), n, C.byref(o), C.byref(bad),
                                      None) == abi.ERR_INVALID
    with pytest.raises(ValueError):
        r.draw(device=True, out=torch.empty((30, 40, 4), dtype=torch.float32, device="cuda"))
    # layered: a terminal and an sRGB8 frame at once, a pixel list with a frame, a host pixel list
    wl = abi.Layer(r.rt.handle, C.pointer(cam.data), C.pointer(o))
    both = abi.DeviceOutputs(srgb8=srgb.data_ptr(), terminal=dev.data_ptr(), len=n)
    assert lib.aicb_render_layers_device(C.byref(wl), None, None, None, None, None, 0, C.byref(both),
                                         None) == abi.ERR_INVALID
    frame = abi.DeviceOutputs(srgb8=srgb.data_ptr(), len=n)
    assert lib.aicb_render_layers_device(C.byref(wl), None, None, None, None, text.data_ptr(), n, C.byref(frame),
                                         None) == abi.ERR_INVALID
    m = cam.depth_transform().astype(np.float64).ravel()
    hpx = np.zeros(n, dtype=np.uint32)
    tex = abi.DeviceOutputs(texel_rgba16f=srgb.data_ptr(), texel_depth=text.data_ptr(), len=n)
    assert lib.aicb_render_layers_device(C.byref(wl), None, None, None, m.ctypes.data, hpx.ctypes.data, n,
                                         C.byref(tex), None) == abi.ERR_INVALID
    g = DeviceGroup([0, 0])
    g.update(space)
    gi = abi.RenderInfo()
    assert lib.aicb_group_render_device(g.scene.handle, C.byref(cam.data), C.byref(o),
                                        C.byref(abi.DeviceOutputs(colorbuf=hst.ctypes.data, len=n)), None,
                                        C.byref(gi)) == abi.ERR_INVALID
    assert lib.aicb_group_render_device(g.scene.handle, C.byref(cam.data), C.byref(o),
                                        C.byref(abi.DeviceOutputs(depth=dev.data_ptr(), len=n)), None,
                                        C.byref(gi)) == abi.ERR_INVALID   # a group's ColorBuf set needs colorbuf
    g.close()
    if torch.cuda.device_count() > 1:
        other = torch.empty((n, 4), dtype=torch.uint8, device="cuda:1")
        assert render(srgb8=other, len=n) == abi.ERR_INVALID
    # pointers below their stores' width: a float32 [n, 4] view at a 4-byte offset, an sRGB8 frame at an odd byte
    base = torch.empty(4 * n + 1, dtype=torch.float32, device="cuda")
    with pytest.raises(aicb200.AicbError) as e:
        r.draw_colorbuf(device=True, want_depth=False, want_hit=False, want_steps=False,
                        out={"colorbuf": base[1:].view(n, 4)})
    assert e.value.status == abi.ERR_INVALID and "aligned" in str(e.value)
    raw = torch.empty(4 * n + 1, dtype=torch.uint8, device="cuda")
    assert render(srgb8=raw.data_ptr() + 1, len=n) == abi.ERR_INVALID
    odd_rays = torch.zeros(6 * n + 1, dtype=torch.float64, device="cuda")
    assert lib.aicb_trace_rays_device(r.rt.handle, odd_rays.data_ptr() + 4, n, C.byref(o), C.byref(outs),
                                      None) == abi.ERR_INVALID
    # a host pixel list with device=True is checked as the host call checks it
    with pytest.raises(aicb200.AicbError) as e:
        aicb200.render_layers_texture((r.rt, cam, opts), None, None, NO_WORLD, cam.depth_transform(),
                                      pixels=np.array([0, n], dtype=np.uint32), device=True)
    assert e.value.status == abi.ERR_INVALID
    assert r.ctx.device_id == torch.cuda.current_device()   # Context(-1): the device current at its creation
    # nothing was issued: the context's next frame is an ordinary one
    assert same_bits(r.draw(device=True).result().data, ref.data)
    r.rt.close()
