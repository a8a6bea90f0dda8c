"""Automatic exposure on the GPU (aicb_step_exposure, its _device and group forms) against the exposure oracle with
correctly rounded ln / exp, the states' bytes and the exposures bit for bit after 1, 10 and 100 ticks, on one context
and on groups [0], [0, 0] and [0, 0, 0]; device-side edits; what the call leaves alone; and the device's ln."""
import ctypes as C
import json
import subprocess

import numpy as np
import pytest
import torch

import __graft_entry__ as g
import aicb200
import exposureorc
from aicb200 import Block, GraphicsOptions, Space, SpaceRaytracer, abi, scenes
from test_gpu_cursor import voxel_space
from test_gpu_device_blocks import on_device
from test_gpu_device_inputs import T, unlit
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
OPTS = GraphicsOptions(view_distance=60.0, lighting_display=aicb200.LIGHT_LINEAR)


@pytest.fixture(autouse=True)
def correctly_rounded():
    exposureorc.set_libm(1)   # ln and exp as the device evaluates them


@pytest.fixture(params=TARGETS, ids=TARGET_IDS)
def target(request):
    return request.param


def invisible_recursive():
    pal = np.zeros((2, 8), dtype=np.float32)
    pal[1, :4] = (0.2, 0.3, 0.4, 1.0)   # used by no voxel
    return Block(resolution=8, indices=np.zeros((8, 3, 8), dtype=np.uint16), palette=pal, voxel_lower=(0, 2, 0))


def partly_visible():
    pal = np.zeros((2, 8), dtype=np.float32)
    pal[1, :4] = (0.7, 0.2, 0.2, 1.0)
    idx = np.zeros((4, 4, 4), dtype=np.uint16)
    idx[1, 2, 3] = 1
    return Block(resolution=4, indices=idx, palette=pal)


def hint_only():
    b = Block(color=(0.0, 0.0, 0.0, 0.0))
    b.light_visible = True   # light_visible (the animation hint) without a visible voxel
    return b


def exposure_voxel_space():
    """voxel_space's blocks of resolution 2-128, plus invisible, partly visible and animation-hint blocks."""
    s = voxel_space(seed=7)
    blocks = s.blocks + [invisible_recursive(), partly_visible(), hint_only()]
    ids = s.block_ids.copy()
    rng = np.random.default_rng(3)
    extra = rng.random(ids.shape) < 0.15
    ids[extra] = rng.integers(len(s.blocks), len(blocks), int(extra.sum()))
    return Space(s.lower, ids, blocks, light=scenes.noise_light(7, ids, blocks), sky_colors=scenes.OCTANT_SKY,
                 light_max_distance=20)


def space_of(kind):
    if kind == "c4":
        return scenes.config_c4(n=32, seed=4)
    if kind == "voxels":
        return exposure_voxel_space()
    if kind == "octants":
        return scenes.small_mixed_scene(n=12, seed=7)
    assert kind == "none"
    return unlit(scenes.config_c1(n=20, seed=2, n_voxel_blocks=6, with_light=True))


def random_quat(rng, n):
    q = rng.normal(size=(n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def random_eyes(space, n, seed):
    """Eyes inside, outside and on the bounds with random rotations; raw random matrices; w <= 0 and NaN."""
    rng = np.random.default_rng(seed)
    lo = np.array(space.lower, np.float64)
    size = np.array(space.size, np.float64)
    m = np.zeros((n, 16))
    kind = rng.integers(0, 6, n)
    q = random_quat(rng, n)
    for i in range(n):
        if kind[i] == 0:     # inside
            t = lo + rng.uniform(0, 1, 3) * size
        elif kind[i] == 1:   # outside
            t = lo + rng.uniform(-0.5, 1.5, 3) * size
        elif kind[i] == 2:   # on the bounds: integer coordinates on a face
            t = lo + np.floor(rng.uniform(0, 1, 3) * (size + 1))
            a = rng.integers(0, 3)
            t[a] = lo[a] + rng.choice([0.0, size[a]])
        else:
            t = lo + rng.uniform(0, 1, 3) * size
        if kind[i] <= 3:
            m[i] = aicb200.view_transform_matrix(q[i] if kind[i] != 3 else (0.0, 0.0, 0.0, 1.0), t)
        else:                # raw random matrices: any w, some NaN or infinite entries
            m[i] = rng.normal(size=16) * rng.choice([0.1, 1.0, 10.0])
            m[i, 12:15] = lo + rng.uniform(0, 1, 3) * size
            m[i, 15] = rng.choice([1.0, 0.5, 0.0, -1.0, 2.0])
            if kind[i] == 5:
                m[i, rng.integers(0, 16)] = rng.choice([np.nan, np.inf, -np.inf])
    return np.ascontiguousarray(m)


def random_states(n, seed):
    rng = np.random.default_rng(seed)
    st = aicb200.exposure_states(n)
    pick = rng.random(n) < 0.5
    st["luminance_samples"][pick] = rng.uniform(0.0, 4.0, (int(pick.sum()), 100)).astype(np.float32)
    st["luminance_sample_index"] = np.where(rng.random(n) < 0.9, rng.integers(0, 100, n), rng.integers(0, 2 ** 32, n))
    st["exposure_log"] = np.where(rng.random(n) < 0.5, 0.0, rng.uniform(-2.0, 1.5, n)).astype(np.float32)
    return st


def first_diff(a, b, width):
    a = np.ascontiguousarray(a).view(np.uint8).reshape(-1, width)
    b = np.ascontiguousarray(b).view(np.uint8).reshape(-1, width)
    return np.nonzero((a != b).any(axis=1))[0]


def run_ticks(scene, space, states, m, dt, ticks=(1, 10, 100), label=""):
    """Steps oracle and scene side by side; compares states and exposures after each tick count in `ticks`."""
    orc = exposureorc.ExposureScene(space)
    want, got = states, states
    for t in range(1, max(ticks) + 1):
        want, we = orc.step(want, m, dt)
        got, ge = scene.step_exposure(got, m, dt)
        if t in ticks:
            d = first_diff(got, want, 408)
            assert len(d) == 0, f"{label} tick {t}: {len(d)} states differ, first {d[:3]}: {got[d[:1]]} vs {want[d[:1]]}"
            d = first_diff(ge, we, 4)
            assert len(d) == 0, f"{label} tick {t}: exposures differ at {d[:3]}: {ge[d[:3]]} vs {we[d[:3]]}"
    return got, ge


@pytest.mark.parametrize("kind", ["c4", "voxels", "octants", "none"])
def test_random_eyes_match_the_oracle(kind):
    space = space_of(kind)
    rt = SpaceRaytracer(space, OPTS)
    if kind == "c4":   # light evaluated on the device, and the oracle given the device's light
        rt.light_fast_evaluate()
        rt.light_evaluate()
        space = Space(space.lower, space.block_ids, space.blocks, light=rt.light_download(),
                      sky_colors=space.sky_colors, light_max_distance=space.light_max_distance)
    m = random_eyes(space, 3000, seed=len(kind))
    st, _ = run_ticks(rt, space, random_states(3000, seed=1), m, 0.05, label=kind)
    changed = (st["exposure_log"] != random_states(3000, seed=1)["exposure_log"]).mean()
    assert changed > 0.5, "too few eyes stepped"
    rt.close()


def test_e2e_on_the_device():
    # exposure.rs:181-241 (see tests/test_oracle_exposure.py): sky 3, light evaluated, 100 ticks at 0.1 s
    light = np.zeros((10, 10, 10, 4), np.uint8)
    light[..., 3] = 1   # NoRays until evaluated
    space = Space((0, 0, 0), np.zeros((10, 10, 10), np.uint16), [Block.air()], light=light,
                  sky_colors=[(3.0, 3.0, 3.0)], light_max_distance=30)
    rt = SpaceRaytracer(space, OPTS)
    rt.light_fast_evaluate()
    rt.light_evaluate()
    st = aicb200.exposure_states(1)
    m = aicb200.view_transform_matrix((0, 0, 0, 1), (5, 5, 5)).reshape(1, 16)
    for _ in range(100):
        st, out = rt.step_exposure(st, m, 0.1)
    assert exposureorc.luminance_average(st[0]) == np.float32(3.0)
    assert abs(out[0] / exposureorc.target_exposure(3.0) - 1.0) < 0.001
    rt.close()


def test_device_form_equals_host_form_and_groups_equal_one_context(target):
    space = space_of("voxels")
    lit = Lit(target, space)
    m = random_eyes(space, 4096, seed=5)
    st0 = random_states(4096, seed=6)
    want, we = exposureorc.ExposureScene(space).step(st0, m, 0.1)
    got, ge = lit.scene.step_exposure(st0, m, 0.1)
    assert exposureorc.same_bytes(got, want) and exposureorc.same_bytes(ge, we)
    side = torch.cuda.Stream(DEV)
    base_st = torch.from_numpy(st0.view(np.uint8).reshape(-1, 408).copy()).to(DEV)
    base_m = T(m)
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)   # the inputs are written late on the stream the call is issued on
        dst = base_st.clone()
        dm = base_m * 1.0
        dst, dout = lit.scene.step_exposure(dst, dm, 0.1, device=True)
        st_copy, out_copy = dst.clone(), dout.clone()
    side.synchronize()
    assert exposureorc.same_bytes(st_copy.cpu().numpy().view(abi.EXPOSURE_STATE_DTYPE).reshape(-1), want)
    assert exposureorc.same_bytes(out_copy.cpu().numpy(), we)
    lit.close()


def test_device_edits_are_seen(target):
    """update_cubes_device, and blocks redefined visible <-> invisible by update_blocks_device and
    append_blocks_device, with no host mirror of the block ids."""
    space = space_of("voxels")
    lit = Lit(target, space)
    s = lit.scene
    m = random_eyes(space, 2000, seed=21)
    st = random_states(2000, seed=22)
    ids = space.block_ids.copy()
    blocks = list(space.blocks)
    rng = np.random.default_rng(8)

    def check(label):
        sp = Space(space.lower, ids.copy(), list(blocks), light=lit.field(), sky_colors=space.sky_colors,
                   light_max_distance=space.light_max_distance)
        want, we = exposureorc.ExposureScene(sp).step(st, m, 0.1)
        got, ge = s.step_exposure(st, m, 0.1)
        d = first_diff(got, want, 408)
        assert len(d) == 0 and exposureorc.same_bytes(ge, we), f"{label}: {len(d)} states differ"

    cubes = np.stack([rng.integers(0, n, 300) for n in space.size], axis=1)
    new = rng.integers(0, len(blocks), 300).astype(np.uint16)
    s.update_cubes(T((cubes + np.array(space.lower)).astype(np.int32)), T(new))
    torch.cuda.synchronize()
    for c, v in zip(cubes, new):
        ids[tuple(c)] = v
    check("update_cubes_device")
    # a visible recursive block becomes invisible, the invisible one visible, from device memory
    vis, inv = 4, len(blocks) - 3
    blocks[vis], blocks[inv] = invisible_recursive(), partly_visible()
    s.update_blocks(np.array([vis, inv], np.uint16), [on_device(blocks[vis]), on_device(blocks[inv])])
    torch.cuda.synchronize()
    check("update_blocks_device")
    app = [partly_visible(), invisible_recursive()]
    s.append_blocks([on_device(b) for b in app])
    torch.cuda.synchronize()
    blocks += app
    sel = rng.random(ids.shape) < 0.2
    ids[sel] = rng.integers(len(blocks) - 2, len(blocks), int(sel.sum()))
    cubes = np.argwhere(sel)
    s.update_cubes(T((cubes + np.array(space.lower)).astype(np.int32)), T(ids[sel].astype(np.uint16)))
    torch.cuda.synchronize()
    check("append_blocks_device")
    lit.close()


def test_nothing_else_changes():
    space = scenes.small_mixed_scene(n=12, seed=7)
    space.light_max_distance = 20   # a light state with a queue and changed cubes to compare
    rt = SpaceRaytracer(space, OPTS)
    rt.light_fast_evaluate()
    cubes = np.array([[0, 3, -4], [1, 4, -3]], np.int32)
    rt.light_edit_cubes(cubes, np.array([1, 2], np.uint16))
    before = (rt.light_download().tobytes(), rt.light_download_queue().tobytes(), rt.light_changes_count(),
              rt.device_bytes)
    cam = scenes.standard_camera(space, OPTS, 160, 120)
    lib = aicb200.load_library()
    n = cam.data.fb_width * cam.data.fb_height
    o = OPTS.to_abi(True)
    d_out = torch.zeros((n, 4), dtype=torch.uint8, device=DEV)
    stream = torch.cuda.Stream(DEV)
    m = random_eyes(space, 500, seed=2)
    infos = []
    for with_exposure in (False, True):
        assert lib.aicb_render_srgb8_device(rt.handle, C.byref(cam.data), C.byref(o), None, d_out.data_ptr(), n,
                                            C.c_void_p(stream.cuda_stream)) == abi.OK
        if with_exposure:
            st = aicb200.exposure_states(len(m))
            out = np.zeros(len(m), np.float32)
            assert lib.aicb_step_exposure(rt.handle, st.ctypes.data, m.ctypes.data, len(m), C.c_double(0.1),
                                          out.ctypes.data) == abi.OK
        info = abi.RenderInfo()
        assert lib.aicb_render_finish(rt.handle, C.byref(info)) == abi.OK
        infos.append((info.cubes_traced, info.flaws, d_out.cpu().numpy().tobytes()))
    assert infos[0] == infos[1]
    after = (rt.light_download().tobytes(), rt.light_download_queue().tobytes(), rt.light_changes_count(),
             rt.device_bytes)
    assert before == after
    rt.close()


@pytest.mark.parametrize("devices", [None, [0, 0]], ids=["ctx", "group2"])
def test_rejections(devices):
    space = scenes.small_mixed_scene(n=12, seed=7)
    lit = Lit(devices, space)
    s = lit.scene
    lib = aicb200.load_library()
    pre = "aicb_" if devices is None else "aicb_group_"
    fn = getattr(lib, pre + "step_exposure")
    fd = getattr(lib, pre + "step_exposure_device")
    m = random_eyes(space, 8, seed=1)
    st = aicb200.exposure_states(8)
    out = np.full(8, 7.0, np.float32)
    for dt in (-0.1, float("nan"), float("inf")):
        assert fn(s.handle, st.ctypes.data, m.ctypes.data, 8, dt, out.ctypes.data) == abi.ERR_INVALID
        assert fd(s.handle, None, None, 0, dt, None, None) == abi.ERR_INVALID
    assert fn(s.handle, None, m.ctypes.data, 8, 0.1, out.ctypes.data) == abi.ERR_INVALID
    assert fn(s.handle, st.ctypes.data, None, 8, 0.1, None) == abi.ERR_INVALID
    assert fn(s.handle, None, None, 0, 0.1, None) == abi.OK
    assert (out == 7.0).all() and exposureorc.same_bytes(st, aicb200.exposure_states(8))
    # host memory where device memory is due
    assert fd(s.handle, st.ctypes.data, m.ctypes.data, 8, 0.1, None, None) == abi.ERR_INVALID
    # dt == 0: the states stay, the exposures are written
    st2, out2 = s.step_exposure(random_states(8, 3), m, 0.0)
    assert exposureorc.same_bytes(st2, random_states(8, 3))
    assert np.array_equal(out2, np.exp(random_states(8, 3)["exposure_log"].astype(np.float64)).astype(np.float32))
    lit.close()


LN_DRIVER = r"""
#include <cstdio>
#include <cstring>
#include <vector>
#include "exact_math.cuh"
using namespace aicb;

__global__ void ln_kernel(uint32_t lo, uint32_t n, float *out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = logf_exact(__uint_as_float(lo + i));
}

int main() {
    float a = 0.6625f, b = 2.125f;
    uint32_t lo, hi;
    std::memcpy(&lo, &a, 4);
    std::memcpy(&hi, &b, 4);
    const uint32_t n = hi - lo + 1;
    float *d;
    if (cudaMalloc(&d, n * sizeof(float)) != cudaSuccess) return 3;
    ln_kernel<<<(n + 255) / 256, 256>>>(lo, n, d);
    std::vector<float> got(n);
    if (cudaMemcpy(got.data(), d, n * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) return 4;
    cudaFree(d);
    unsigned long long mismatch = 0;
    uint32_t first = 0;
    for (uint32_t i = 0; i < n; i++) {
        float x, want;
        const uint32_t xb = lo + i;
        std::memcpy(&x, &xb, 4);
        want = logf_exact(x);
        if (std::memcmp(&want, &got[i], 4) != 0 && mismatch++ == 0) first = xb;
    }
    std::printf("{\"n\": %u, \"mismatch\": %llu, \"first\": %u}\n", n, mismatch, first);
    return 0;
}
"""


def test_device_ln_equals_the_host(tmp_path):
    # logf_exact on the device and compiled as host code, with the library's own flags, on every f32 in
    # [0.6625, 2.125] (tests/test_oracle_exposure.py checks the host's against glibc)
    src, exe = tmp_path / "ln.cu", tmp_path / "ln"
    src.write_text(LN_DRIVER)
    flags = [f for f in g.NVCC_FLAGS if f != "-shared"]
    r = subprocess.run([g.NVCC] + flags + ["-I", str(g.PKG) + "/csrc", "-o", str(exe), str(src)], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    t = json.loads(subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout)
    assert t["n"] == int(np.float32(2.125).view(np.uint32)) - int(np.float32(0.6625).view(np.uint32)) + 1
    assert t["mismatch"] == 0, t
