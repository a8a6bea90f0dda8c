"""The brick pool's room for more voxel words (csrc/brick_room.h), which both aicb_scene_update_blocks and
aicb_scene_append_blocks consult before they place new definitions.  Brick positions are u32: the live data alone may
not pass 2^32 words (rejected), and when only the dead words push the positions past it, the pool is compacted first.
A scene that reaches these sizes needs 8 GiB of bricks, so the rule is checked here on the host, through a small
driver built from the same header."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER_DIR = os.path.join(ROOT, "all-is-cubes_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

DRIVER = r"""
#include <cstdio>
#include <cstdlib>
#include "brick_room.h"
int main(int argc, char **argv) {
    for (int i = 1; i + 2 < argc; i += 3) {
        const BrickRoom r = brick_room(std::strtoull(argv[i], nullptr, 0), std::strtoull(argv[i + 1], nullptr, 0),
                                       std::strtoull(argv[i + 2], nullptr, 0));
        std::printf("%s\n", r == BrickRoom::fits ? "fits" : r == BrickRoom::compact_first ? "compact_first" : "too_big");
    }
    return 0;
}
"""

LIMIT = 2 ** 32 - 1
RES128 = 128 ** 3

CASES = [
    # (words in use, of which dead, words to add) -> decision
    ((0, 0, RES128), "fits"),
    ((LIMIT - 10, 0, 10), "fits"),
    ((LIMIT - 10, 0, 11), "too_big"),                         # the parent's limit, unchanged without dead words
    ((LIMIT - 10, 5, 11), "compact_first"),
    # an append after updates: the pool holds up to twice its live data, dead <= live
    ((2 ** 32 - 2 ** 20, 2 ** 31 - 2 ** 20, RES128), "compact_first"),
    ((LIMIT - RES128, 2 ** 31 - 2 ** 21, RES128), "fits"),      # exactly 2^32 - 1 words in use afterwards
    ((LIMIT - RES128, 2 ** 31 - 2 ** 21, RES128 + 1), "compact_first"),
    # live data past the limit is rejected whatever is dead
    ((2 ** 32, 2 ** 31, 2 ** 31), "too_big"),
    ((3 * 2 ** 30, 2 ** 30, 2 ** 31 - 1), "compact_first"),
    ((3 * 2 ** 30, 2 ** 30, 2 ** 31), "too_big"),
]


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("brick_room")
    src, exe = d / "driver.cpp", d / "driver"
    src.write_text(DRIVER)
    r = subprocess.run([NVCC, "-std=c++17", "-I", HEADER_DIR, "-o", str(exe), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return str(exe)


def test_brick_room_decisions(driver):
    args = [str(v) for (inputs, _) in CASES for v in inputs]
    out = subprocess.run([driver] + args, capture_output=True, text=True, check=True).stdout.split()
    assert out == [want for _, want in CASES]
