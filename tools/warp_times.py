"""AICB_PROFILE_KERNELS=1: end-time distribution of the marching warps for a full frame and for one shard of 8."""
import os
import sys

os.environ["AICB_PROFILE_KERNELS"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
import bench  # noqa: E402
import aicb200  # noqa: E402
from aicb200 import scenes  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "c2"
space, opts, w, h, desc = bench.make_workload(name)
cam = scenes.standard_camera(space, opts, w, h)
r = aicb200.RtRenderer(cam)
r.update(space)
for shard in (None, (16, 2, 8)):
    print("shard", shard, flush=True)
    for i in range(3):
        r.draw(shard=shard)
