"""The cursor oracle (oracle_cursor/) against the reference's own known answers (cursor.rs:310-436), project_cursor's
layer order, the preceding cube's rules, and aicb_cursor's layout.  No GPU."""
import ctypes as C
import os
import subprocess

import numpy as np

import aicb200
import cursororc
from aicb200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = float("inf")

# cursor.rs's X_RAY: starts in cube [-1, 0, 0], hits [0, 0, 0], [1, 0, 0], ... just above the midpoint
X_RAY = (-0.5, 0.500001, 0.500001, 1.0, 0.0, 0.0)
# SLOPING_RAY: through the left face, then the middle Y plane, of a block at [0, 0, 0]
SLOPING_RAY = (-0.25, 1.0, 0.5, 1.0, -1.0, 0.0)

SOME_BLOCK = dict(color=(0.5, 0.25, 0.125, 1.0))   # make_some_blocks: an opaque atom


def make_slab(numerator, resolution):
    """content.rs:176-210: voxel bounds [0, R) x [0, numerator) x [0, R), a checkerboard of two selectable voxels;
    the voxels above the bounds are AIR (not selectable)."""
    x, y, z = np.meshgrid(np.arange(resolution), np.arange(numerator), np.arange(resolution), indexing="ij")
    indices = ((x + y + z) % 2).astype(np.uint16)
    palette = np.zeros((2, 8), dtype=np.float32)
    palette[0, :4] = (0.6, 0.4, 0.2, 1.0)
    palette[1, :4] = (0.63, 0.42, 0.21, 1.0)
    return aicb200.Block(resolution=resolution, indices=indices, palette=palette)


def row_space(blocks, light=None, sky=(1.0, 1.0, 1.0)):
    """cursor.rs's test_space: the blocks in a row along X from [0, 0, 0]; `blocks` [0] is AIR."""
    table = [aicb200.Block.air()] + list(blocks)
    ids = np.arange(1, len(blocks) + 1, dtype=np.uint16).reshape(-1, 1, 1)
    return aicb200.Space((0, 0, 0), ids, table, light=light, sky_colors=sky)


def cast(space, ray, max_distance=None):
    return cursororc.CursorScene(space).cursor_raycast(np.array([ray]), max_distance)[0]


def test_simple_hit_after_air():
    c = cast(row_space([aicb200.Block.air(), aicb200.Block(**SOME_BLOCK)]), X_RAY)
    assert c["block_id"] == 2
    assert tuple(c["cube"]) == (1, 0, 0)
    assert c["face_selected"] == abi.FACE_NX


def test_maximum_distance_too_short():
    c = cast(row_space([aicb200.Block.air(), aicb200.Block(**SOME_BLOCK)]), X_RAY, 1.0)
    assert c["block_id"] == abi.CURSOR_NONE
    assert c["layer"] == 0 and c["preceding_block_id"] == abi.CURSOR_NONE


def test_ignores_not_selectable_atom():
    c = cast(row_space([aicb200.Block(color=(1, 1, 1, 1), selectable=False), aicb200.Block(**SOME_BLOCK)]), X_RAY)
    assert tuple(c["cube"]) == (1, 0, 0)
    assert c["block_id"] == 2


def test_ignores_not_selectable_voxels():
    c = cast(row_space([make_slab(1, 2), aicb200.Block(**SOME_BLOCK)]), X_RAY)
    assert tuple(c["cube"]) == (1, 0, 0)
    assert c["block_id"] == 2


def test_hits_selectable_voxels():
    c = cast(row_space([aicb200.Block.air(), make_slab(3, 4), aicb200.Block(**SOME_BLOCK)]), X_RAY)
    assert tuple(c["cube"]) == (1, 0, 0)
    assert c["block_id"] == 2


def test_slope_hits_face_of_full_block():
    c = cast(row_space([aicb200.Block(**SOME_BLOCK)]), SLOPING_RAY)
    assert c["face_entered"] == abi.FACE_NX
    assert c["face_selected"] == abi.FACE_NX


def test_slope_hits_face_different_from_entered():
    c = cast(row_space([make_slab(1, 2)]), SLOPING_RAY)
    assert c["face_entered"] == abi.FACE_NX
    assert c["face_selected"] == abi.FACE_PY


def test_voxel_flags_decide_within_a_block():
    # the same slab with its lower voxels made unselectable: the ray through them finds nothing
    slab = make_slab(3, 4)
    slab_off = aicb200.Block(resolution=4, indices=slab.indices, palette=slab.palette, voxel_selectable=False)
    assert cast(row_space([slab_off]), X_RAY)["block_id"] == abi.CURSOR_NONE
    one_on = aicb200.Block(resolution=4, indices=slab.indices, palette=slab.palette, voxel_selectable=[False, True])
    assert cast(row_space([one_on]), X_RAY)["block_id"] == 1
    # a single voxel's own flag, and Evoxel::AIR for a resolution-1 block whose bounds hold no voxel
    assert cast(row_space([aicb200.Block(color=(1, 1, 1, 1), voxel_selectable=False)]), X_RAY)["block_id"] == \
        abi.CURSOR_NONE
    empty = aicb200.Block(resolution=1, indices=np.zeros((0, 0, 0), dtype=np.uint16),
                          palette=np.zeros((1, 8), dtype=np.float32))
    assert cast(row_space([empty]), X_RAY)["block_id"] == abi.CURSOR_NONE
    # an invisible single voxel is selectable unless it says otherwise
    assert cast(row_space([aicb200.Block(color=(0, 0, 0, 0))]), X_RAY)["block_id"] == 1


def test_ray_from_inside_is_within_without_preceding():
    space = row_space([aicb200.Block(**SOME_BLOCK), aicb200.Block(**SOME_BLOCK)])
    ray = (1.25, 0.5, 0.5, 3.0, 0.0, 0.0)
    c = cast(space, ray)
    assert c["face_entered"] == abi.FACE_WITHIN and c["face_selected"] == abi.FACE_WITHIN
    assert tuple(c["cube"]) == (1, 0, 0) and tuple(c["preceding_cube"]) == (1, 0, 0)
    assert c["preceding_block_id"] == abi.CURSOR_NONE
    assert tuple(c["preceding_light"]) == (0, 0, 0, 0)
    assert c["distance"] == 0.0
    assert tuple(c["point_entered"]) == ray[:3]


def test_preceding_cube_outside_is_outside_with_the_sky_texel():
    light = np.zeros((2, 1, 1, 4), dtype=np.uint8)
    light[:] = (10, 20, 30, 255)
    space = aicb200.Space((0, 0, 0), np.array([[[1]], [[1]]], dtype=np.uint16),
                          [aicb200.Block.air(), aicb200.Block(**SOME_BLOCK)], light=light, sky_colors=(1.0, 1.0, 1.0),
                          light_max_distance=20)
    c = cast(space, X_RAY)
    assert tuple(c["cube"]) == (0, 0, 0) and tuple(c["preceding_cube"]) == (-1, 0, 0)
    assert c["preceding_block_id"] == abi.CURSOR_OUTSIDE
    assert tuple(c["light"]) == (10, 20, 30, 255)
    assert tuple(c["preceding_light"]) == (144, 144, 144, 255)   # BlockSky::light_outside, face NX of a white sky
    # without a light volume (LightPhysics::None) every cube's light is PackedLight::ONE
    c = cast(aicb200.Space((0, 0, 0), np.array([[[1]]], dtype=np.uint16),
                           [aicb200.Block.air(), aicb200.Block(**SOME_BLOCK)], sky_colors=(0.0, 0.0, 0.0)), X_RAY)
    assert tuple(c["light"]) == (144, 144, 144, 255) and tuple(c["preceding_light"]) == (144, 144, 144, 255)
    assert c["distance"] == 0.5 and tuple(c["point_entered"]) == (0.0, 0.500001, 0.500001)


def test_distance_limit_compares_t_distance():
    space = row_space([aicb200.Block.air(), aicb200.Block(**SOME_BLOCK)])
    sc = cursororc.CursorScene(space)
    rays = np.array([X_RAY] * 5)
    out = sc.cursor_raycast(rays, [1.5, 1.4999999, float("nan"), -1.0, INF])
    assert list(out["block_id"]) == [2, abi.CURSOR_NONE, 2, abi.CURSOR_NONE, 2]


def _camera(eye, target):
    cam = aicb200.Camera(aicb200.GraphicsOptions(), aicb200.Viewport.with_scale(1.0, (32, 32)))
    cam.look_at_y_up(eye, target)
    return cam


def test_project_cursor_tries_ui_then_world():
    one = lambda block: aicb200.Space((0, 0, 0), np.ones((1, 1, 1), dtype=np.uint16), [aicb200.Block.air(), block])
    cam = _camera((0.5, 0.5, 10.0), (0.5, 0.5, 0.0))
    world = (cursororc.CursorScene(one(aicb200.Block(**SOME_BLOCK))), cam)
    ui_on = (cursororc.CursorScene(one(aicb200.Block(color=(1, 1, 1, 1)))), cam)
    ui_off = (cursororc.CursorScene(one(aicb200.Block(color=(1, 1, 1, 1), selectable=False))), cam)
    ndc = np.array([[0.0, 0.0], [0.9, 0.9]])
    # the UI answers first, with no distance limit (the cube is ~9 away)
    out = cursororc.project_cursor(world, ui_on, ndc, 6.0)
    assert list(out["layer"]) == [1, 0]
    # an unselectable UI block lets the world answer, within world_max_distance only
    assert list(cursororc.project_cursor(world, ui_off, ndc, 20.0)["layer"]) == [2, 0]
    assert list(cursororc.project_cursor(world, ui_off, ndc, 6.0)["layer"]) == [0, 0]
    assert list(cursororc.project_cursor(world, None, ndc, 20.0)["layer"]) == [2, 0]
    # each layer's ray is Camera::project_ndc_into_world of its camera
    ray = cam.project_ndc_into_world(0.0, 0.0)
    direct = world[0].cursor_raycast(np.array([ray]), 20.0)[0]
    got = cursororc.project_cursor(world, None, ndc[:1], 20.0)[0]
    got["layer"] = 0
    assert cursororc.same_bits(got, direct)


def test_cursor_layout_matches_c_header(tmp_path):
    names = [n for n in abi.CURSOR_DTYPE.names]
    src = tmp_path / "cursor.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "aicb200.h"\nint main(){printf("%zu", '
                   'sizeof(aicb_cursor));' + "".join(f'printf(" %zu", offsetof(aicb_cursor, {n}));' for n in names) +
                   'printf(" %zu %zu %zu %zu", sizeof(aicb_voxel), offsetof(aicb_voxel, flags), '
                   'sizeof(aicb_block_desc), offsetof(aicb_block_desc, flags));return 0;}\n')
    exe = tmp_path / "cursor"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [C.sizeof(abi.Cursor)] + [getattr(abi.Cursor, n).offset for n in names]
    want += [C.sizeof(abi.Voxel), abi.Voxel.flags.offset, C.sizeof(abi.BlockDesc), abi.BlockDesc.flags.offset]
    assert got == want
    assert got[0] == 80 == abi.CURSOR_DTYPE.itemsize
    assert [abi.CURSOR_DTYPE.fields[n][1] for n in names] == got[1:1 + len(names)]


def test_ingest_carries_selectable_into_the_flags():
    from aicb200 import ingest

    def blocks_space(blocks, contents, upper):
        return {"type": "SpaceV1", "bounds": {"lower": [0, 0, 0], "upper": upper},
                "physics": {"gravity": [0, 0, 0], "sky": {"type": "UniformV1", "color": [0, 0, 0]},
                            "light": {"type": "NoneV1"}},
                "blocks": blocks, "contents": ingest.gz_encode(np.array(contents, dtype="<u2").tobytes()),
                "light": None}

    air = {"type": "BlockV1", "primitive": {"type": "AirV1"}}
    atom = lambda sel: {"type": "BlockV1", "primitive": {"type": "AtomV1", "color": [1.0, 0.0, 0.0, 1.0]},
                        "modifiers": [] if sel is None else [{"type": "SelectableV1", "selectable": sel}]}
    voxels = blocks_space([air, atom(None), atom(False)], [0, 1, 2, 1], [2, 1, 2])
    recur = {"type": "BlockV1", "primitive": {"type": "RecurV1", "space": {"type": "HandleV1", "Specific": "vox"},
                                              "resolution": 2},
             "modifiers": [{"type": "SelectableV1", "selectable": True}, {"type": "SelectableV1", "selectable": False}]}
    world = blocks_space([air, recur, atom(False), atom(True)], [1, 2, 3], [3, 1, 1])
    u = {"type": "UniverseV1", "members": [{"name": {"Specific": "vox"}, "member_type": "Space", "value": voxels},
                                          {"name": {"Specific": "world"}, "member_type": "Space", "value": world}]}
    w = ingest.spaces_from_universe(u)[ingest.name_key({"Specific": "world"})]
    desc, keep = w.to_desc()
    assert [desc.blocks[i].flags for i in range(4)] == [abi.BLOCK_NOT_SELECTABLE] * 3 + [0]   # AIR included
    # the Recur block's voxels: AirV1 not selectable, the plain atom selectable, the unselectable atom not
    assert list(w.blocks[1].palette.view(np.uint32)[:, 7]) == [abi.VOXEL_NOT_SELECTABLE, 0, abi.VOXEL_NOT_SELECTABLE]
    assert not w.blocks[0].selectable
