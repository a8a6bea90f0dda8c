"""The cursor on the GPU (aicb_cursor_raycast, aicb_project_cursor, their _device and group forms) against the cursor
oracle, every field bit for bit (f64s by their bits), on one context and on groups [0], [0, 0] and [0, 0, 0]; and the
selectability flags leave every existing output as it was."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import aicb200
import cursororc
from aicb200 import Block, GraphicsOptions, Space, SpaceRaytracer, abi, scenes
from test_gpu_append_blocks import assert_same, every_output, narrow_space, wide_blocks
from test_gpu_device_blocks import on_device
from test_gpu_device_inputs import T, unlit
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
OPTS = GraphicsOptions(view_distance=60.0, lighting_display=aicb200.LIGHT_LINEAR)
INF = float("inf")


@pytest.fixture(params=TARGETS, ids=TARGET_IDS)
def target(request):
    return request.param


def with_flags(space, seed, p_block=0.3, p_voxel=0.4):
    """The Space with a random share of its blocks and voxels not selectable (block 0 stays AIR)."""
    rng = np.random.default_rng(seed)
    blocks = []
    for b in space.blocks:
        c = copy.copy(b)
        c.selectable = (not b.is_air) and bool(rng.random() >= p_block)
        c.palette = np.array(b.palette, dtype=np.float32, copy=True)
        c.palette.view(np.uint32)[:, 7] = (rng.random(c.palette.shape[0]) < p_voxel).astype(np.uint32)
        blocks.append(c)
    return Space(space.lower, space.block_ids, blocks, light=space.light, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


def voxel_space(seed=5):
    """Voxel blocks of resolution 2 to 128 with partial bounds, among single and invisible blocks."""
    n = 10
    blocks = [Block.air(), Block(color=(0.8, 0.2, 0.1, 1.0)), Block(color=(0.0, 0.0, 0.0, 0.0)),
              Block(color=(0.2, 0.5, 0.9, 0.5))]
    for k, res in enumerate((2, 4, 8, 16, 32, 64, 128)):
        blocks.append(scenes.make_voxel_block(seed + k, resolution=res, alpha=(1.0, 0.5)[k % 2], partial_bounds=True))
    h = scenes.grid_hash(seed, (n, n, n))
    ids = np.where((h & np.uint64(3)) == 0, (h >> np.uint64(8)) % np.uint64(len(blocks)), 0).astype(np.uint16)
    return Space((-4, 0, 3), ids, blocks, light=scenes.noise_light(seed, ids, blocks), sky_colors=scenes.OCTANT_SKY,
                 light_max_distance=20)


def space_of(kind):
    if kind == "c1":
        return scenes.config_c1(n=20, seed=2, n_voxel_blocks=6, with_light=True)
    if kind == "c1_none":
        return unlit(scenes.config_c1(n=20, seed=2, n_voxel_blocks=6, with_light=True))
    if kind == "mixed":
        return scenes.small_mixed_scene(n=12, seed=7)
    if kind == "voxels":
        return voxel_space()
    if kind == "wide":   # more than 32768 palette entries: u32 brick words
        s = voxel_space()
        rng = np.random.default_rng(11)
        pal = np.zeros((40000, 8), np.float32)
        pal[:, :3] = rng.uniform(0, 1, (40000, 3))
        pal[:, 3] = rng.choice(np.array([0.0, 0.5, 1.0], np.float32), 40000)
        s.blocks[5] = Block(resolution=16, indices=rng.integers(0, 40000, (16, 16, 16)).astype(np.uint16), palette=pal,
                            voxel_lower=(0, 0, 0))
        return s
    assert kind == "u32"   # more than 16384 blocks: u32 cells
    s = narrow_space()
    ids = s.block_ids.copy()
    ids[1, 2, :5] = [16383, 16384, 16390, 16400, 16419]
    return Space(s.lower, ids, s.blocks + wide_blocks(), light=s.light, sky_colors=s.sky_colors)


def random_rays(space, n, seed):
    """Rays from inside, from outside (aimed at the bounds or anywhere), missing, axis-parallel, and with a zero
    direction."""
    rng = np.random.default_rng(seed)
    lo = np.array(space.lower, np.float64)
    size = np.array(space.size, np.float64)
    o = lo + rng.uniform(-0.5, 1.5, (n, 3)) * size
    aim = lo + rng.uniform(0.0, 1.0, (n, 3)) * size
    d = aim - o
    kind = rng.integers(0, 6, n)
    d[kind == 1] = rng.normal(size=(int((kind == 1).sum()), 3))                       # anywhere
    axis = rng.integers(0, 3, n)
    par = np.zeros((n, 3))
    par[np.arange(n), axis] = rng.choice([-1.0, 1.0], n) * rng.uniform(0.1, 3.0, n)
    d[kind == 2] = par[kind == 2]                                                     # axis-parallel
    d[kind == 3] = 0.0                                                                # zero direction
    o[kind == 4] = lo + rng.uniform(0.0, 1.0, (int((kind == 4).sum()), 3)) * size     # from inside
    d[kind == 5] *= rng.uniform(1e-3, 1e3, (int((kind == 5).sum()), 1))               # any length
    return np.ascontiguousarray(np.concatenate([o, d], axis=1))


def distances(oracle, rays, seed):
    """Per ray: at, just below and just above its selected step's t, NaN, negative, or none."""
    rng = np.random.default_rng(seed)
    t = oracle.cursor_raycast(rays)["distance"]
    pick = rng.integers(0, 6, len(rays))
    md = np.where(pick == 0, t, np.where(pick == 1, np.nextafter(t, -INF), np.where(pick == 2, np.nextafter(t, INF),
                  np.where(pick == 3, np.nan, np.where(pick == 4, -rng.uniform(0, 2, len(rays)), INF)))))
    return np.ascontiguousarray(md)


def check(scene, space, rays, max_distance=None, label=""):
    want = cursororc.CursorScene(space).cursor_raycast(rays, max_distance)
    got = scene.cursor_raycast(rays, max_distance)
    diff = np.nonzero((np.asarray(got).view(np.uint8).reshape(-1, 80) !=
                       np.asarray(want).view(np.uint8).reshape(-1, 80)).any(axis=1))[0]
    assert len(diff) == 0, f"{label}: {len(diff)} queries differ, first {diff[:3]}: {got[diff[:1]]} vs " \
        f"{want[diff[:1]]}"
    return want


@pytest.mark.parametrize("kind", ["c1", "c1_none", "mixed", "voxels", "wide", "u32"])
def test_random_rays_match_the_oracle(target, kind):
    space = with_flags(space_of(kind), seed=3)
    lit = Lit(target, space)
    rays = random_rays(space, 4000, seed=len(kind))
    want = check(lit.scene, space, rays, None, kind)
    assert (want["block_id"] != abi.CURSOR_NONE).sum() > 200, "too few rays select a cube"
    assert (want["face_entered"] == abi.FACE_WITHIN)[want["block_id"] != abi.CURSOR_NONE].any()
    md = distances(cursororc.CursorScene(space), rays, seed=9)
    check(lit.scene, space, rays, md, kind + " with distances")
    lit.close()


def test_device_form_on_a_side_stream(target):
    space = with_flags(space_of("voxels"), seed=4)
    lit = Lit(target, space)
    rays = random_rays(space, 3000, seed=12)
    md = distances(cursororc.CursorScene(space), rays, seed=13)
    want = cursororc.CursorScene(space).cursor_raycast(rays, md)
    side = torch.cuda.Stream(DEV)
    base, mdt = T(rays), T(md)
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)                 # the rays are written late on the stream the call is issued on
        od = base * 1.0                               # a torch kernel produces them
        out = lit.scene.cursor_raycast(od, mdt, device=True)
        copy_out = out.clone()
    side.synchronize()
    assert cursororc.same_bits(copy_out.cpu().numpy().view(abi.CURSOR_DTYPE).reshape(-1), want)
    lit.close()


def test_updates_are_seen(target):
    """After every kind of update, host and device (a redefinition with new flags, pools compacted, an append, a
    fill_uniform), the cursor sees the new cells and flags."""
    space = with_flags(space_of("voxels"), seed=6)
    lit = Lit(target, space)
    s = lit.scene
    rays = random_rays(space, 2000, seed=21)
    rng = np.random.default_rng(8)
    ids = space.block_ids.copy()
    blocks = list(space.blocks)

    def current(label):
        sp = Space(space.lower, ids.copy(), list(blocks), light=lit.field(), sky_colors=space.sky_colors,
                   light_max_distance=space.light_max_distance)
        check(s, sp, rays, None, label)

    # host cube update
    cubes = np.stack([rng.integers(0, n, 60) for n in space.size], axis=1)
    new = rng.integers(0, len(blocks), 60).astype(np.uint16)
    s.update_cubes((cubes + np.array(space.lower)).astype(np.int32), new)
    for c, v in zip(cubes, new):
        ids[tuple(c)] = v
    current("update_cubes")
    # device cube update: the mirror goes stale, and the cursor sees the cells without it
    cubes = np.stack([rng.integers(0, n, 60) for n in space.size], axis=1)
    new = rng.integers(0, len(blocks), 60).astype(np.uint16)
    s.update_cubes(T((cubes + np.array(space.lower)).astype(np.int32)), T(new))
    torch.cuda.synchronize()
    for c, v in zip(cubes, new):
        ids[tuple(c)] = v
    current("update_cubes_device")
    # a redefinition with new flags (host), then one from device memory, then an append
    b = copy.copy(blocks[4])
    b.selectable = not b.selectable
    blocks[4] = b
    s.update_blocks(np.array([4], np.uint16), [b])
    current("update_blocks")
    nb = with_flags(Space(space.lower, ids, [Block.air(), scenes.make_voxel_block(99, resolution=8)]), seed=2).blocks[1]
    db = on_device(nb)
    db.selectable = nb.selectable
    blocks[5] = nb
    s.update_blocks(np.array([5], np.uint16), [db])
    torch.cuda.synchronize()
    current("update_blocks_device")
    for k in range(6):   # redefinitions until the pools compact
        b = copy.copy(blocks[6 + k % 3])
        b.palette = b.palette.copy()
        b.palette.view(np.uint32)[:, 7] ^= 1
        blocks[6 + k % 3] = b
        s.update_blocks(np.array([6 + k % 3], np.uint16), [b])
    current("compacted")
    app = Block(color=(0.1, 0.9, 0.3, 1.0))
    s.append_blocks([app])
    blocks.append(app)
    ids[0, 0, 0] = len(blocks) - 1
    s.update_cubes(np.array([space.lower], np.int32), np.array([len(blocks) - 1], np.uint16))
    current("append_blocks")
    # fill_uniform with an unselectable block: every query selects nothing
    off = Block(color=(0.5, 0.5, 0.5, 1.0), selectable=False)
    s.fill_uniform(off)
    blocks = [off]
    ids[:] = 0
    current("fill_uniform")
    lit.close()


def test_cursor_leaves_a_frame_in_flight_alone():
    space = with_flags(space_of("mixed"), seed=1)
    cam = scenes.standard_camera(space, OPTS, 160, 120)
    rt = SpaceRaytracer(space, OPTS)
    lib = aicb200.load_library()
    n = cam.data.fb_width * cam.data.fb_height
    o = OPTS.to_abi(True)
    d_out = torch.zeros((n, 4), dtype=torch.uint8, device=DEV)
    stream = torch.cuda.Stream(DEV)
    infos = []
    rays = random_rays(space, 500, seed=2)
    for with_cursor in (False, True):
        assert lib.aicb_render_srgb8_device(rt.handle, C.byref(cam.data), C.byref(o), None, d_out.data_ptr(), n,
                                            C.c_void_p(stream.cuda_stream)) == abi.OK
        if with_cursor:
            out = np.zeros(len(rays), dtype=abi.CURSOR_DTYPE)
            assert lib.aicb_cursor_raycast(rt.handle, rays.ctypes.data, None, len(rays), out.ctypes.data) == abi.OK
            assert cursororc.same_bits(out, cursororc.CursorScene(space).cursor_raycast(rays))
        info = abi.RenderInfo()
        assert lib.aicb_render_finish(rt.handle, C.byref(info)) == abi.OK
        infos.append((info.cubes_traced, info.flaws, d_out.cpu().numpy().tobytes()))
    assert infos[0] == infos[1]
    rt.close()


@pytest.mark.parametrize("devices", [None, [0, 0]], ids=["ctx", "group2"])
def test_rejections(devices):
    space = space_of("mixed")
    lit = Lit(devices, space)
    s = lit.scene
    lib = aicb200.load_library()
    pre = "aicb_" if devices is None else "aicb_group_"
    fn = getattr(lib, pre + "cursor_raycast")
    fd = getattr(lib, pre + "cursor_raycast_device")
    rays = random_rays(space, 64, seed=1)
    out = np.full(64, 0xAB, dtype=np.uint8).repeat(80)
    assert fn(s.handle, None, None, 64, out.ctypes.data) == abi.ERR_INVALID
    assert fn(s.handle, rays.ctypes.data, None, 64, None) == abi.ERR_INVALID
    assert fn(s.handle, None, None, 0, None) == abi.OK
    assert (out == 0xAB).all()
    d_rays, d_out = T(rays), torch.full((64 * 80 + 8,), 0xAB, dtype=torch.uint8, device=DEV)
    d_md = torch.zeros(65, dtype=torch.float64, device=DEV)
    assert fd(s.handle, rays.ctypes.data, None, 64, d_out.data_ptr(), None) == abi.ERR_INVALID   # host memory
    assert fd(s.handle, d_rays.data_ptr(), None, 64, out.ctypes.data, None) == abi.ERR_INVALID
    assert fd(s.handle, d_rays.data_ptr() + 4, None, 63, d_out.data_ptr(), None) == abi.ERR_INVALID   # misaligned
    assert fd(s.handle, d_rays.data_ptr(), None, 64, d_out.data_ptr() + 4, None) == abi.ERR_INVALID
    assert fd(s.handle, d_rays.data_ptr(), d_md.data_ptr() + 4, 64, d_out.data_ptr(), None) == abi.ERR_INVALID
    assert fd(s.handle, None, None, 64, d_out.data_ptr(), None) == abi.ERR_INVALID
    assert fd(s.handle, None, None, 0, None, None) == abi.OK
    torch.cuda.synchronize()
    assert (d_out.cpu().numpy() == 0xAB).all() and (out == 0xAB).all()
    # project_cursor: NULL ndc / out, a layer without a camera, layers on two contexts
    cam = scenes.standard_camera(space, OPTS, 32, 32)
    ndc = np.zeros((4, 2))
    o4 = np.zeros(4, dtype=abi.CURSOR_DTYPE)
    if devices is None:
        other = SpaceRaytracer(space, OPTS, aicb200.Context(0))
        L, P = abi.Layer, lib.aicb_project_cursor
        w, u = L(s.handle, C.pointer(cam.data), None), L(other.handle, C.pointer(cam.data), None)
    else:
        other = aicb200.DeviceGroup([0]).add_scene(space)
        L, P = abi.GroupLayer, lib.aicb_group_project_cursor
        w, u = L(s.handle, C.pointer(cam.data), None), L(other.handle, C.pointer(cam.data), None)
    assert P(C.byref(w), None, None, 4, 6.0, o4.ctypes.data) == abi.ERR_INVALID
    assert P(C.byref(w), None, ndc.ctypes.data, 4, 6.0, None) == abi.ERR_INVALID
    assert P(C.byref(w), C.byref(u), ndc.ctypes.data, 4, 6.0, o4.ctypes.data) == abi.ERR_INVALID
    nocam = L(s.handle, None, None)
    assert P(C.byref(nocam), None, ndc.ctypes.data, 4, 6.0, o4.ctypes.data) == abi.ERR_INVALID
    assert P(C.byref(w), None, None, 0, 6.0, None) == abi.OK
    assert not np.asarray(o4).view(np.uint8).any()
    lit.close()


def test_project_cursor_matches_the_oracle(target):
    world_space = with_flags(space_of("mixed"), seed=5)
    ui_space = with_flags(space_of("voxels"), seed=6, p_block=0.5)
    cam_w = scenes.standard_camera(world_space, OPTS, 64, 48)
    cam_u = scenes.standard_camera(ui_space, OPTS, 64, 48, direction=(-1.0, 0.3, 0.5))
    rng = np.random.default_rng(3)
    ndc = rng.uniform(-1.1, 1.1, (3000, 2))
    ow, ou = cursororc.CursorScene(world_space), cursororc.CursorScene(ui_space)
    if target is None:
        ctx = aicb200.Context.default()
        w, u = SpaceRaytracer(world_space, OPTS, ctx), SpaceRaytracer(ui_space, OPTS, ctx)
        project = aicb200.project_cursor
    else:
        g = aicb200.DeviceGroup(target)
        w, u = g.add_scene(world_space), g.add_scene(ui_space)
        project = g.project_cursor
    layers = set()
    for wmax in (6.0, 30.0, INF):
        want = cursororc.project_cursor((ow, cam_w), (ou, cam_u), ndc, wmax)
        got = project((w, cam_w), (u, cam_u), ndc, wmax)
        assert cursororc.same_bits(got, want), wmax
        layers |= set(np.unique(want["layer"]).tolist())
        assert cursororc.same_bits(project((w, cam_w), None, ndc, wmax),
                                   cursororc.project_cursor((ow, cam_w), None, ndc, wmax))
    assert layers == {0, 1, 2}
    assert cursororc.same_bits(project(None, (u, cam_u), ndc), cursororc.project_cursor(None, (ou, cam_u), ndc))


@pytest.mark.parametrize("kind", ["c1", "voxels", "wide"])
def test_flags_change_no_existing_output(kind):
    """Every frame output, the light field after propagation and device_bytes of a scene with flags set equal those of
    the same scene with its flags cleared."""
    plain = space_of(kind)
    flagged = with_flags(plain, seed=2, p_block=0.5, p_voxel=0.5)
    cam = scenes.standard_camera(plain, OPTS, 48, 40)
    out = []
    for sp in (plain, flagged):
        rt = SpaceRaytracer(sp, OPTS)
        o = every_output(rt, OPTS, cam)
        o["device_bytes"] = np.array([rt.device_bytes])
        if sp.light_max_distance:
            rt.light_fast_evaluate()
            rt.light_evaluate()
            o["light"] = rt.light_download()
        out.append(o)
        rt.close()
    assert_same(out[0], out[1], kind)
