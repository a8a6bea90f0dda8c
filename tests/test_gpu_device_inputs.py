"""The scene calls fed from device memory (aicb_scene_update_cubes_device .. aicb_light_download_device and their group
forms): with the same data as CUDA tensors, each must leave the scene byte for byte as its host twin does.  Every
check builds two scenes from one Space on the same target (one context, groups of 1, 2 and 3 contexts of one device),
updates one through the host calls and the other through the device calls, and compares after every step: block ids,
light, queue, the set of changed cubes, n_changed, device_bytes, an sRGB8 frame and a ColorBuf ray batch."""
import ctypes as C

import numpy as np
import pytest
import torch

import aicb200
from aicb200 import AicbError, Block, GraphicsOptions, Space, abi, scenes
from editlists import edit_list
from test_gpu_append_blocks import narrow_space, wide_blocks
from test_gpu_light import compare_fields, light_scene
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit
from test_gpu_region import with_light

pytestmark = pytest.mark.gpu

OPTS = GraphicsOptions(view_distance=60.0, lighting_display=aicb200.LIGHT_LINEAR)
QUEUED = ((0, 2, 5), (6, 8, 6), 230)   # cubes queued before the edits, so that cancellations show
DEV = torch.device("cuda", 0)


def T(a):
    """A numpy array as a CUDA tensor of the same dtype on device 0 (uint16 through an int16 view)."""
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint16:
        return torch.from_numpy(a.view(np.int16)).to(DEV).view(torch.uint16)
    return torch.from_numpy(a).to(DEV)


def rays_for(space, n=700, seed=3):
    """A fixed ray batch (origin, direction) from a sphere around the Space towards points inside it."""
    rng = np.random.default_rng(seed)
    lo, size = np.array(space.lower, float), np.array(space.size, float)
    centre = lo + size / 2
    d = rng.normal(size=(n, 3))
    origin = centre + d / np.linalg.norm(d, axis=1, keepdims=True) * size.max() * 1.5
    target = lo + rng.uniform(0, 1, (n, 3)) * size
    return np.concatenate([origin, target - origin], axis=1)


class Pair:
    """Two scenes of one Space on one target: `host` updated through the host calls, `dev` through the device calls."""

    def __init__(self, devices, space):
        self.space = space
        self.devices = devices
        self.host, self.dev = Lit(devices, space), Lit(devices, space)
        self.cam = scenes.standard_camera(space, OPTS, 48, 40)
        self.rays = rays_for(space)

    def state(self, lit):
        s = lit.scene
        out = {"ids": s.block_ids(), "srgb8": lit.frame(self.cam, OPTS),
               "colorbuf": aicb200._trace_rays(s, self.rays, OPTS.to_abi(True), True, True, False)["colorbuf"]}
        if self.space.light_max_distance:
            out["light"] = lit.field()
            out["queue"] = s.light_download_queue()
            out["changes"] = np.concatenate([a.reshape(-1).view(np.uint8) for a in s.light_take_changes()])
        elif self.space.light is not None:
            out["light"] = lit.field()
        if lit.group is None:
            out["device_bytes"] = np.array([s.device_bytes])
        return out

    def check(self, label):
        a, b = self.state(self.host), self.state(self.dev)
        assert a.keys() == b.keys()
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), f"{label}: {k} differs"
        return a

    def close(self):
        self.host.close()
        self.dev.close()


def unlit(space):
    """The Space without a light volume and with LightPhysics::None."""
    return Space(space.lower, space.block_ids, space.blocks, sky_colors=space.sky_colors)


def cube_lists(space, seed, with_light):
    """Lists with repeated cubes, cubes set to their own block, an opaque block and back, and an empty list."""
    rng = np.random.default_rng(seed)
    lo, size = np.array(space.lower), np.array(space.size)
    n_blocks = len(space.blocks)
    for k in range(3):
        if len(space.blocks) <= 8:   # light_scene: edit_list's segments (chains between kinds, corners, lamps)
            cubes, ids = edit_list(space, seed=seed + k)
        else:   # a small pool of cubes named many times, and cubes scattered over the bounds, ids from the whole table
            pool = rng.integers(0, size, (24, 3))
            cubes = np.concatenate([pool[rng.integers(0, 24, 120)], rng.integers(0, size, (200, 3))]) + lo
            ids = rng.integers(0, n_blocks, len(cubes)).astype(np.uint16)
        cubes = cubes.astype(np.int32)
        dup = rng.integers(0, len(cubes), len(cubes) // 10)
        cubes = np.concatenate([cubes, cubes[dup]]).astype(np.int32)
        ids = np.concatenate([ids, rng.integers(0, n_blocks, len(dup)).astype(np.uint16)])
        same = rng.integers(0, size, (20, 3))
        cubes = np.concatenate([cubes, (same + lo).astype(np.int32)])
        ids = np.concatenate([ids, space.block_ids[tuple(same.T)]])   # same-block sets (of the original Space)
        c = (rng.integers(0, size, 3) + lo).astype(np.int32)
        cubes = np.concatenate([cubes, [c, c, c]]).astype(np.int32)
        ids = np.concatenate([ids, np.array([1, 0, 1], dtype=np.uint16)])   # opaque, back, opaque
        light = rng.integers(0, 256, (len(cubes), 4)).astype(np.uint8) if with_light else None
        yield cubes, ids, light
    yield np.zeros((0, 3), np.int32), np.zeros(0, np.uint16), (np.zeros((0, 4), np.uint8) if with_light else None)


def spaces(kind):
    if kind == "lit":
        return light_scene(seed=9)
    if kind == "unlit":
        return unlit(light_scene(seed=9))
    return narrow_space()   # "wide": 32-bit cells once append_blocks passes 16384 ids


def grow_wide(pair):
    for lit in (pair.host, pair.dev):
        lit.append_blocks(wide_blocks())
    pair.space = Space(pair.space.lower, pair.space.block_ids, pair.space.blocks + wide_blocks(),
                       light=pair.space.light, sky_colors=pair.space.sky_colors)


@pytest.mark.parametrize("kind", ["lit", "unlit", "wide"])
@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_update_cubes_equals_host(devices, kind):
    p = Pair(devices, spaces(kind))
    if kind == "wide":
        grow_wide(p)
    for step, (cubes, ids, light) in enumerate(cube_lists(p.space, 11, kind != "unlit")):
        p.host.update_cubes(cubes, ids, light)
        p.dev.update_cubes(T(cubes), T(ids), None if light is None else T(light))
        p.check(f"update_cubes step {step}")
    p.close()


@pytest.mark.parametrize("kind", ["lit", "unlit", "wide"])
@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_update_region_and_light_equal_host(devices, kind):
    p = Pair(devices, spaces(kind))
    if kind == "wide":
        grow_wide(p)
    rng = np.random.default_rng(5)
    n_blocks = len(p.space.blocks)
    lo = np.array(p.space.lower)
    for step, (off, size) in enumerate([((1, 2, 0), (5, 4, 9)), ((0, 0, 3), (3, 7, 1)), ((2, 1, 1), (0, 3, 3))]):
        ids = rng.integers(0, n_blocks, size).astype(np.uint16)
        light = rng.integers(0, 256, tuple(size) + (4,)).astype(np.uint8)
        lower = tuple(int(v) for v in lo + off)
        p.host.update_region(lower, size, ids, light)
        p.dev.update_region(lower, size, T(ids), T(light))
        p.check(f"region step {step}")
        p.host.update_region(lower, size, 2, light)
        p.dev.update_region(lower, size, 2, T(light))
        p.check(f"uniform region with light, step {step}")
        p.host.update_region(lower, size, ids)
        p.dev.update_region(lower, size, T(ids))
        p.check(f"region without light, step {step}")
    if p.space.light is not None or p.space.light_max_distance:
        whole = rng.integers(0, 256, p.space.size + (4,)).astype(np.uint8)
        p.host.upload_light(whole)
        p.dev.upload_light(T(whole))
        st = p.check("upload_light")
        got = p.dev.scene.light_download(device=True)
        assert got.device == DEV and got.dtype == torch.uint8
        assert got.cpu().numpy().tobytes() == st["light"].tobytes()
    ids_t = p.dev.scene.block_ids(device=True)
    assert ids_t.dtype == torch.uint16 and ids_t.device == DEV
    assert ids_t.view(torch.int16).cpu().numpy().view(np.uint16).tobytes() == p.host.scene.block_ids().tobytes()
    p.close()


def test_upload_light_gives_a_volume_to_an_unlit_scene():
    """As aicb_scene_upload_light: a scene created without a light volume gets one (device_bytes grows alike)."""
    space = unlit(light_scene(seed=9))
    p = Pair(None, space)
    light = np.random.default_rng(2).integers(0, 256, space.size + (4,)).astype(np.uint8)
    p.host.upload_light(light)
    p.dev.upload_light(T(light))
    p.space = Space(space.lower, space.block_ids, space.blocks, light=light, sky_colors=space.sky_colors)
    p.check("upload into an unlit scene")
    p.close()


@pytest.fixture(scope="module")
def converged_space():
    from resumeorc import LightOracle
    space = light_scene(seed=9)
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    return with_light(space, ol.field())


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_light_edits_equal_host_and_converge(converged_space, devices):
    p = Pair(devices, converged_space)
    for lit in (p.host, p.dev):
        lit.light_queue_region(*QUEUED)
    lo = np.array(p.space.lower)
    for step, (cubes, ids, _) in enumerate(cube_lists(p.space, 21, False)):
        a = p.host.light_edit_cubes(cubes, ids)
        b = p.dev.light_edit_cubes(T(cubes), T(ids))
        assert a == b, f"edit step {step}: n_changed {a} != {b}"
        p.check(f"light_edit_cubes step {step}")
    rng = np.random.default_rng(8)
    for step, (off, size) in enumerate([((1, 1, 1), (4, 5, 6)), ((0, 3, 2), (7, 2, 5))]):
        ids = rng.choice(np.array([0, 1, 3, 5], np.uint16), size).astype(np.uint16)
        lower = tuple(int(v) for v in lo + off)
        a = p.host.light_edit_region(lower, size, ids)
        b = p.dev.light_edit_region(lower, size, T(ids))
        assert a == b, f"region step {step}: n_changed {a} != {b}"
        p.check(f"light_edit_region step {step}")
        a = p.host.light_edit_region(lower, size, 1)
        b = p.dev.light_edit_region(lower, size, 1)
        assert a == b
        p.check(f"uniform light_edit_region step {step}")
    # propagation after the edits: the host sequence's field, under the light tests' convergence contract
    p.host.light_evaluate(1)
    p.dev.light_evaluate(1)
    compare_fields(p.dev.field(), p.host.field())
    p.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_rejections_change_nothing(devices):
    space = light_scene(seed=9)
    p = Pair(devices, space)
    s = p.dev.scene
    before = p.state(p.dev)
    lo, size = np.array(space.lower), np.array(space.size)
    good_c = T(np.array([lo + 1, lo + 2], np.int32))
    good_i = T(np.array([1, 2], np.uint16))
    bad_c = T(np.array([lo + 1, lo + size], np.int32))
    bad_i = T(np.array([1, len(space.blocks)], np.uint16))
    stream = aicb200._stream(DEV)
    host_c = np.ascontiguousarray(np.array([lo + 1, lo + 2], np.int32))
    host_i = np.array([1, 2], np.uint16)
    region_ids = T(np.full((2, 2, 2), len(space.blocks), np.uint16))
    raw = torch.zeros(64, dtype=torch.uint8, device=DEV)

    def region(lower, sz):
        r = abi.Aab()
        r.lower[:] = [int(v) for v in lower]
        r.size[:] = [int(v) for v in sz]
        return r

    n = C.c_size_t(0)
    cases = {
        "cube out of bounds": lambda: s.update_cubes(bad_c, good_i),
        "id past the table": lambda: s.update_cubes(good_c, bad_i),
        "edit cube out of bounds": lambda: s.light_edit_cubes(bad_c, good_i),
        "edit id past the table": lambda: s.light_edit_cubes(good_c, bad_i),
        "region ids past the table": lambda: s.update_region(tuple(lo), (2, 2, 2), region_ids),
        "edit region ids past the table": lambda: s.light_edit_region(tuple(lo), (2, 2, 2), region_ids),
        "region outside the bounds": lambda: s.update_region(tuple(lo + size - 1), (2, 2, 2), region_ids),
        "host cubes": lambda: aicb200._check(s._fn("scene_update_cubes_device")(
            s.handle, host_c.ctypes.data, good_i.data_ptr(), None, 2, stream)),
        "host ids": lambda: aicb200._check(s._fn("light_edit_cubes_device")(
            s.handle, good_c.data_ptr(), host_i.ctypes.data, 2, C.byref(n), stream)),
        "misaligned cubes": lambda: aicb200._check(s._fn("scene_update_cubes_device")(
            s.handle, raw.data_ptr() + 2, good_i.data_ptr(), None, 2, stream)),
        "misaligned ids": lambda: aicb200._check(s._fn("light_edit_cubes_device")(
            s.handle, good_c.data_ptr(), raw.data_ptr() + 1, 2, C.byref(n), stream)),
        "misaligned light": lambda: aicb200._check(s._fn("scene_upload_light_device")(
            s.handle, raw.data_ptr() + 2, int(np.prod(space.size)), stream)),
        "misaligned output": lambda: aicb200._check(s._fn("light_download_device")(
            s.handle, raw.data_ptr() + 1, int(np.prod(space.size)), stream)),
        "host region ids": lambda: aicb200._check(s._fn("scene_update_region_device")(
            s.handle, C.byref(region(lo, (1, 1, 2))), host_i.ctypes.data, 0, None, stream)),
    }
    for label, call in cases.items():
        with pytest.raises(AicbError) as e:
            call()
        assert e.value.status == abi.ERR_INVALID, label
        now = p.state(p.dev)
        for k in before:
            if k != "changes":
                assert now[k].tobytes() == before[k].tobytes(), f"{label}: {k} changed"
    with pytest.raises(ValueError):
        s.update_cubes(good_c.to(torch.int64), good_i)
    if torch.cuda.device_count() > 1:   # a pointer of another device
        on_other = good_c.to(torch.device("cuda", 1))
        with pytest.raises(AicbError):
            aicb200._check(s._fn("scene_update_cubes_device")(s.handle, on_other.data_ptr(), good_i.data_ptr(), None,
                                                              2, stream))
    p.close()
    # LightPhysics::None: the light edits are rejected after the list checks, as the host twins reject them
    q = Pair(devices, unlit(space))
    before = q.state(q.dev)
    for call in (lambda: q.dev.scene.light_edit_cubes(good_c, good_i),
                 lambda: q.dev.scene.light_edit_region(tuple(lo), (2, 2, 2), T(np.ones((2, 2, 2), np.uint16)))):
        with pytest.raises(AicbError) as e:
            call()
        assert e.value.status == abi.ERR_INVALID
        assert "LightPhysics::None" in str(e.value)
    now = q.state(q.dev)
    for k in before:
        assert now[k].tobytes() == before[k].tobytes(), f"None: {k} changed"
    q.close()


def test_messages_are_the_host_twins():
    space = light_scene(seed=9)
    p = Pair(None, space)
    lo, size = np.array(space.lower), np.array(space.size)
    cubes = np.array([lo + 1, lo + size, lo + 2], np.int32)
    ids = np.array([len(space.blocks), 1, 1], np.uint16)   # entry 0's id is bad before entry 1's cube
    for host, dev in ((p.host.update_cubes, p.dev.update_cubes), (p.host.light_edit_cubes, p.dev.light_edit_cubes)):
        with pytest.raises(AicbError) as a:
            host(cubes, ids)
        with pytest.raises(AicbError) as b:
            dev(T(cubes), T(ids))
        assert str(a.value) == str(b.value)
    p.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_host_calls_after_device_updates_see_a_current_mirror(converged_space, devices):
    """Device updates leave the host mirror stale; host light_edit_cubes, light_edit_region, update_blocks +
    light_relight_blocks and fill_uniform then give what the all-host sequence gives."""
    p = Pair(devices, converged_space)
    lo = np.array(p.space.lower)
    cubes, ids, light = next(cube_lists(p.space, 31, True))
    p.host.update_cubes(cubes, ids, light)
    p.dev.update_cubes(T(cubes), T(ids), T(light))
    rids = np.random.default_rng(4).integers(0, len(p.space.blocks), (3, 4, 5)).astype(np.uint16)
    p.host.update_region(tuple(lo + 1), (3, 4, 5), rids)
    p.dev.update_region(tuple(lo + 1), (3, 4, 5), T(rids))
    e_c, e_i, _ = next(cube_lists(p.space, 41, False))
    p.host.light_edit_cubes(e_c, e_i)
    p.dev.light_edit_cubes(T(e_c), T(e_i))
    p.check("device updates")
    # the same host calls on both: the device-updated scene rebuilds its mirror first
    c2, i2, _ = next(cube_lists(p.space, 51, False))
    assert p.host.light_edit_cubes(c2, i2) == p.dev.light_edit_cubes(c2, i2)
    p.check("host light_edit_cubes")
    p.dev.update_cubes(T(c2), T(i2))
    p.host.update_cubes(c2, i2)
    for lit in (p.host, p.dev):
        lit.light_edit_region(tuple(lo), (4, 3, 2), np.full((4, 3, 2), 3, np.uint16))
    p.check("host light_edit_region")
    p.dev.update_region(tuple(lo + 2), (2, 2, 2), T(np.full((2, 2, 2), 4, np.uint16)))
    p.host.update_region(tuple(lo + 2), (2, 2, 2), np.full((2, 2, 2), 4, np.uint16))
    # a block whose kind changes: update_blocks re-encodes its cubes from the mirror
    voxel = scenes.make_voxel_block(3, resolution=4, alpha=0.5)
    for lit in (p.host, p.dev):
        lit.update_blocks([4], [voxel])
        lit.light_relight_blocks([4], 1)
    p.space = Space(p.space.lower, p.space.block_ids, p.space.blocks[:4] + [voxel] + p.space.blocks[5:],
                    light=p.space.light, sky_colors=p.space.sky_colors, light_max_distance=p.space.light_max_distance)
    a, b = p.host.field(), p.dev.field()
    compare_fields(b, a)
    assert p.host.scene.block_ids().tobytes() == p.dev.scene.block_ids().tobytes()
    p.dev.update_cubes(T(c2), T(i2))
    p.host.update_cubes(c2, i2)
    for lit in (p.host, p.dev):
        lit.fill_uniform(Block(color=(0.4, 0.5, 0.6, 1.0)))
    assert p.host.scene.block_ids().tobytes() == p.dev.scene.block_ids().tobytes()
    for lit in (p.host, p.dev):
        lit.light_edit_cubes(c2[:5], np.zeros(5, np.uint16))
    assert p.host.scene.block_ids().tobytes() == p.dev.scene.block_ids().tobytes()
    assert p.host.field().tobytes() == p.dev.field().tobytes()
    p.close()


@pytest.mark.parametrize("devices", TARGETS, ids=TARGET_IDS)
def test_inputs_written_on_a_side_stream_are_read_in_stream_order(devices):
    """A torch kernel on a side stream writes the ids after a delay; the device call issued on that stream reads
    them without a host synchronise in between."""
    space = light_scene(seed=9)
    p = Pair(devices, space)
    rng = np.random.default_rng(12)
    lo, size = np.array(space.lower), np.array(space.size)
    cubes = (rng.integers(0, size, (4000, 3)) + lo).astype(np.int32)
    ids = rng.integers(0, len(space.blocks), 4000).astype(np.uint16)
    src = T(ids)
    c = T(cubes)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        out = torch.zeros(4000, dtype=torch.int16, device=DEV)
        torch.cuda._sleep(50_000_000)   # tens of milliseconds of GPU time before the ids exist
        out.copy_(src.view(torch.int16))
        p.dev.update_cubes(c, out.view(torch.uint16))
        n = p.dev.light_edit_cubes(c[:500], out.view(torch.uint16)[:500].flip(0).contiguous())
    p.host.update_cubes(cubes, ids)
    assert n == p.host.light_edit_cubes(cubes[:500], ids[:500][::-1].copy())
    p.check("side stream")
    p.close()
