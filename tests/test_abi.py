"""CPU-side checks of the product library: it loads without a GPU, exports every symbol that
include/aicb200.h declares, the ctypes mirror matches the C struct sizes, and compute entry
points fail loudly (no CPU fallback) when there is no device."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import aicb200
from aicb200 import abi
from conftest import has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    lib = aicb200.load_library()
    header = open(os.path.join(ROOT, "include", "aicb200.h")).read()
    declared = set(re.findall(r"\b(aicb_[a-z0-9_]+)\s*\(", header))
    assert declared == set(abi.EXPORTED_SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), f"libaicb200.so does not export {name}"
    assert lib.aicb_abi_version() == abi.ABI_VERSION


def test_struct_layouts_match_c_header(tmp_path):
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include "aicb200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n",'
                   "sizeof(aicb_aab),sizeof(aicb_voxel),sizeof(aicb_block_desc),sizeof(aicb_sky),sizeof(aicb_scene_desc),"
                   "sizeof(aicb_camera),sizeof(aicb_options),sizeof(aicb_shard),sizeof(aicb_render_info),sizeof(aicb_hit));return 0;}\n")
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    sizes = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    mirror = [abi.Aab, abi.Voxel, abi.BlockDesc, abi.Sky, abi.SceneDesc, abi.CameraData, abi.Options, abi.Shard,
              abi.RenderInfo, abi.Hit]
    assert sizes == [C.sizeof(m) for m in mirror]


def test_library_was_built_for_sm_90a_only():
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-lelf", aicb200.LIB_PATH], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    archs = set(re.findall(r"sm_(\d+a?)", out.stdout))
    assert archs == {"90a"}, archs


@pytest.mark.skipif(has_gpu(), reason="this check is for the GPU-less build container")
def test_no_cpu_fallback_without_gpu():
    with pytest.raises(aicb200.AicbError) as e:
        aicb200.Context(-1)
    assert e.value.status == abi.ERR_CUDA
    assert "no CPU fallback" in str(e.value)


def test_shard_pixel_count_partitions_the_frame():
    cam = aicb200.Camera(aicb200.GraphicsOptions(), aicb200.Viewport.with_scale(1.0, (37, 29)))
    lib = aicb200.load_library()
    for count in (1, 2, 3, 8):
        total = 0
        for index in range(count):
            s = abi.Shard(16, index, count)
            total += lib.aicb_shard_pixel_count(C.byref(cam.data), C.byref(s))
        assert total == 37 * 29
    assert lib.aicb_shard_pixel_count(C.byref(cam.data), None) == 37 * 29


def test_scene_hash_is_deterministic():
    from aicb200 import scenes
    a = scenes.config_c0()
    b = scenes.config_c0()
    assert np.array_equal(a.block_ids, b.block_ids)
    assert int(scenes.hash3(1, 2, 3, 4)) == int(scenes.hash3(1, 2, 3, 4))
    assert 0.10 < (a.block_ids != 0).mean() < 0.15  # 12.5 % fill


def test_rust_sys_crate_declares_every_function_of_the_header():
    """bindings/rust/all-is-cubes-b200-sys (source only; no Rust toolchain here) must not drift from include/aicb200.h."""
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "aicb200.h")).read()
    declared = set(re.findall(r"\b(aicb_[a-z0-9_]+)\s*\(", header))
    rust = open(os.path.join(root, "bindings", "rust", "all-is-cubes-b200-sys", "src", "lib.rs")).read()
    bound = set(re.findall(r"pub fn (aicb_[a-z0-9_]+)", rust))
    assert declared == bound, (sorted(declared - bound), sorted(bound - declared))
    assert declared == set(abi.EXPORTED_SYMBOLS)
