"""Blocks with more than 32768 palette entries (up to 2^16: VoxelIndex is u16, voxel_storage.rs:32), on the oracle: a
Space holding such a block draws exactly as the same Space holding its twin, whose palette is deduplicated below 32768
entries (same voxels).  The GPU tests of wide brick pools rest on this: the twin is drawn with narrow brick words."""
import numpy as np
import pytest

import orc
import widepal
from aicb200 import (LIGHT_FLAT, LIGHT_LINEAR, LIGHT_NONE, TRANSPARENCY_SURFACE, TRANSPARENCY_THRESHOLD,
                     TRANSPARENCY_VOLUMETRIC, GraphicsOptions, scenes)

OPTIONS = [GraphicsOptions(view_distance=40.0, transparency=TRANSPARENCY_VOLUMETRIC, lighting_display=LIGHT_LINEAR),
           GraphicsOptions(view_distance=40.0, transparency=TRANSPARENCY_SURFACE, lighting_display=LIGHT_FLAT),
           GraphicsOptions(view_distance=40.0, transparency=TRANSPARENCY_THRESHOLD, transparency_threshold=0.3,
                           lighting_display=LIGHT_NONE)]


@pytest.mark.parametrize("resolution,n_palette", [(64, 40000), (128, 65536)])
def test_wide_palette_draws_as_its_deduplicated_twin(resolution, n_palette):
    wide, twin = widepal.wide_block(11, resolution, n_palette)
    assert wide.palette.shape[0] == n_palette > 32768 and twin.palette.shape[0] <= 32768
    assert np.array_equal(wide.palette[wide.indices], twin.palette[twin.indices])
    used = np.unique(wide.indices)
    assert used.max() == n_palette - 1
    d = len(twin.palette)
    for kind in (widepal.INVISIBLE, widepal.TRANSLUCENT, widepal.EMISSIVE_CLEAR, widepal.EMISSIVE):
        assert ((used > 32767) & (used % d == kind)).any(), f"no entry above 32767 of kind {kind}"
    ws, ts = widepal.space_with(wide), widepal.space_with(twin)
    ow, ot = orc.OracleScene(ws), orc.OracleScene(ts)
    for opts in OPTIONS:
        cam = scenes.standard_camera(ws, opts, 64, 48)
        a, b = ow.render(cam, opts), ot.render(cam, opts)
        for k in ("srgb8", "colorbuf", "depth", "hit", "steps", "text"):
            assert a[k].tobytes() == b[k].tobytes(), f"transparency {opts.transparency}: {k} differs"
        assert a["cubes_traced"] == b["cubes_traced"]
        # the frame meets the wide block's voxels: no other block of the Space has this resolution
        assert (a["hit"][:, 6] == resolution).sum() > 50, "the frame shows too little of the wide block"
