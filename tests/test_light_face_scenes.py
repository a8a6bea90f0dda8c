"""The voxel scenes of tests/test_gpu_light_voxels.py tell the faces of a block apart, shown on the light oracle alone.

LightBuffer::traverse (updater.rs:760-884) reads the colour and the opacity bit of the face a ray ENTERS a block by.  A
kernel that read the exit face instead, or the Within colour, would give the oracle's answers on atoms, whose faces are
all alike.  Here each block table is altered the way such a kernel would misread it, and compute_light on the same field
must change: so the GPU tests, which demand the oracle's bits on these scenes, would catch that kernel."""
import copy

import pytest

import orc
from aicb200 import Space
from test_gpu_light import all_cubes
from test_gpu_light_voxels import odd_corner_scene, translucent_stack

SCENES = {"odd_corner": odd_corner_scene, "translucent_stack": translucent_stack}


def mirror_colours(b):
    c = b.light_face_colors
    b.light_face_colors = c[3:] + c[:3]           # NX <-> PX, NY <-> PY, NZ <-> PZ


def mirror_opacity(b):
    m = b.light_opaque_faces
    b.light_opaque_faces = ((m & 7) << 3) | (m >> 3)


def opacity_of_next_face(b):
    m = b.light_opaque_faces
    b.light_opaque_faces = ((m << 1) | (m >> 5)) & 0x3F   # the bit of NX read for NY, NY for NZ, ... PZ for NX


def within_colour(b):
    b.light_face_colors = [b.light_color] * 6


def altered(space, alter):
    """The Space with `alter` applied to a copy of every voxel block (atoms are the same from every side)."""
    blocks = []
    for b in space.blocks:
        if b.indices is not None:
            b = copy.copy(b)
            alter(b)
        blocks.append(b)
    return Space(space.lower, space.block_ids, blocks, light=space.light, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


def compute_both(space, alter):
    """compute_light of every cube with the true and with the altered blocks, on the oracle's field after fast_evaluate
    and 600 updates (one of the inputs the GPU tests use)."""
    ol = orc.OracleLight(space)
    ol.fast_evaluate()
    ol.evaluate(0, max_updates=600)
    cubes = all_cubes(space)
    ref = ol.compute(cubes)
    wrong = orc.OracleLight(altered(space, alter))
    wrong.set_field(ol.field())
    return ref, wrong.compute(cubes)


@pytest.mark.parametrize("alter", [mirror_colours, within_colour, opacity_of_next_face])
@pytest.mark.parametrize("name", list(SCENES))
def test_misread_faces_change_compute_light(name, alter):
    ref, got = compute_both(SCENES[name](), alter)
    differ = int((got != ref).any(axis=1).sum())
    lit = int((ref[:, 3] == 255).sum())
    assert differ >= 0.05 * lit, f"{differ} of {lit} lit cubes differ"


@pytest.mark.parametrize("name", list(SCENES))
def test_mirrored_opacity_bits_change_compute_light(name):
    """The opacity bit decides only whether a ray that hits a face with coverage > 0 stops (alpha = 0) or goes on
    (alpha *= 1 - coverage).  Behind an opaque face's full layer, the opposite face is covered completely unless its
    trace stops at transmittance 1/256 first: only the veiled blocks have such a face, its coverage above 1 - 1/256, so
    the light that the correct bit lets through is small and few cubes change, by one unit.  The GPU tests demand the
    oracle's bits, so even one cube catches a kernel that reads the bit of the face a ray leaves by."""
    space = SCENES[name]()
    assert any(b.light_face_colors[(f + 3) % 6][3] < 1.0 for b in space.blocks for f in range(6)
               if (b.light_opaque_faces >> f) & 1), "no block whose face opposite an opaque one is partly covered"
    ref, got = compute_both(space, mirror_opacity)
    differ = int((got != ref).any(axis=1).sum())
    assert differ > 0
