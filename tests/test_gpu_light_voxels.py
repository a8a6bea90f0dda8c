"""GPU light propagation on voxel blocks: faces that differ in opacity and colour, partial voxel bounds, hollow blocks.

An atom carries one colour on all six faces and is opaque on all of them or on none, so over atoms a kernel that read
the colour or opacity of another face than the one a ray enters by (LightBuffer::traverse, updater.rs:760-884) gives
the right answers.  The blocks here differ
face by face; each fixture asserts the opacity bits and face colours it derives (block/eval/derived.rs), so a change of
the derivation cannot quietly turn them back into atoms.  The kernels are held to the light oracle on the same Space:
fast_evaluate and compute_light bit for bit, converged and edited fields by the contract of tests/test_gpu_light.py.
tests/test_light_face_scenes.py shows on the oracle alone that these scenes tell the faces apart."""
import numpy as np
import pytest

import aicb200
import orc
from aicb200 import Block, GraphicsOptions, Space, SpaceRaytracer, scenes
from test_gpu_group_light import assert_replicas_identical, c4_slice, group_scene, slab_space, with_field
from test_gpu_light import NO_RAYS, VISIBLE, all_cubes, compare_fields, light_scene
from test_gpu_light_changes import Lit, cubes_set_opaque, opaque_for_light

pytestmark = pytest.mark.gpu

NX, NY, NZ, PX, PY, PZ = range(6)
R = 4            # resolution of the hand-made blocks


def opposite(face):
    return (face + 3) % 6


def layer(face, r=R):
    """The index of the voxel layer that lies on `face`."""
    sl = [slice(None)] * 3
    sl[face % 3] = r - 1 if face >= 3 else 0
    return tuple(sl)


def voxel_block(indices, palette, lower=(0, 0, 0), resolution=R):
    """palette rows: (r, g, b, a) or (r, g, b, a, er, eg, eb); entry 0 is the air voxel."""
    pal = np.zeros((len(palette) + 1, 8), dtype=np.float32)
    for i, row in enumerate(palette):
        pal[i + 1, :len(row)] = row
    return Block(resolution=resolution, voxel_lower=lower, indices=indices.astype(np.uint16), palette=pal)


def rgb(c):
    return np.array(c[:3], dtype=np.float64)


FACE_TINTS = [(0.9, 0.6, 0.2), (0.8, 0.8, 0.1), (0.9, 0.3, 0.5), (0.7, 0.9, 0.2), (0.95, 0.5, 0.1), (0.6, 0.7, 0.3)]
VEIL = (0.1, 0.2, 0.9, 0.9)     # the translucent layer on the open side of a one-face block


def one_face_block(face):
    """Opaque on `face` only: a full opaque layer there, a blue translucent layer on the opposite face, air between."""
    idx = np.zeros((R, R, R), dtype=np.uint16)
    idx[layer(opposite(face))] = 2
    idx[layer(face)] = 1
    b = voxel_block(idx, [FACE_TINTS[face] + (1.0,), VEIL])
    assert b.light_opaque_faces == 1 << face
    assert np.allclose(b.light_face_colors[face], FACE_TINTS[face] + (1.0,), atol=1e-6)
    # seen from the other side the veil comes first: a different colour, the same full coverage
    back = b.light_face_colors[opposite(face)]
    assert back[3] == 1.0 and np.abs(rgb(back) - rgb(FACE_TINTS[face])).max() > 0.2, back
    for f in range(6):
        if f % 3 != face % 3:
            assert 0.25 < b.light_face_colors[f][3] < 0.5, (f, b.light_face_colors[f])   # one opaque column, one veiled
    return b


def half_slab_block():
    """Solid on its lower half, the voxel bounds shrunk to the solid voxels: opaque on NY only, full coverage on NY and
    PY (whose surface lies inside the cube), half coverage on the sides."""
    b = voxel_block(np.ones((R, R // 2, R), dtype=np.uint16), [(0.6, 0.5, 0.3, 1.0)])
    assert b.voxel_size == (R, R // 2, R)
    assert b.light_opaque_faces == 1 << NY
    assert b.light_face_colors[NY][3] == 1.0 and b.light_face_colors[PY][3] == 1.0
    for f in (NX, NZ, PX, PZ):
        assert np.isclose(b.light_face_colors[f][3], 0.5), (f, b.light_face_colors[f])
    return b


def shell_block(open_face=None):
    """A hollow box of opaque voxels, its back wall (NZ) in another colour; `open_face` leaves that wall out."""
    idx = np.ones((R, R, R), dtype=np.uint16)
    idx[layer(NZ)] = 2
    inner = (slice(1, R - 1),) * 3
    idx[inner] = 0
    if open_face is not None:
        hole = list(inner)
        hole[open_face % 3] = R - 1 if open_face >= 3 else 0
        idx[tuple(hole)] = 0
    b = voxel_block(idx, [(0.3, 0.8, 0.4, 1.0), (0.9, 0.1, 0.6, 1.0)])
    want = 0x3F if open_face is None else 0x3F & ~(1 << open_face)
    assert b.light_opaque_faces == want
    assert all(c[3] == 1.0 for c in b.light_face_colors)   # every face is covered, the open one through its hole
    assert b.light_visible and opaque_for_light(b) == (open_face is None)
    return b


def two_colour_block(near=(1.0, 0.05, 0.05), far=(0.05, 0.05, 1.0), axis=0):
    """Translucent all through: a `near` layer on the negative face of `axis`, a `far` layer on the positive face (both
    alpha 0.9), grey alpha-0.5 voxels between.  Its two faces on that axis differ strongly in colour and have equal coverage."""
    idx = np.full((R, R, R), 2, dtype=np.uint16)
    idx[layer(axis)] = 1
    idx[layer(axis + 3)] = 3
    b = voxel_block(idx, [near + (0.9,), (0.5, 0.5, 0.5, 0.5), far + (0.9,)])
    n, p = b.light_face_colors[axis], b.light_face_colors[axis + 3]
    assert b.light_opaque_faces == 0
    assert 0.0 < n[3] < 1.0 and np.isclose(n[3], p[3])
    assert np.abs(rgb(n) - rgb(p)).max() > 0.25, (n, p)
    return b


def one_face_emitter(face=PX):
    """An emissive opaque voxel layer on one face, nothing else."""
    idx = np.zeros((R, R, R), dtype=np.uint16)
    idx[layer(face)] = 1
    b = voxel_block(idx, [(0.9, 0.8, 0.3, 1.0, 3.0, 2.0, 0.5)])
    assert b.light_opaque_faces == 1 << face and max(b.light_emission) > 0.0
    assert b.light_face_colors[face][3] == 1.0 and np.isclose(b.light_face_colors[opposite(face)][3], 1.0)
    return b


def veiled_block(face, r=16):
    """Opaque on `face` only, every other voxel alpha 0.999, the opaque layer glowing.  A trace from the opposite face
    stops once its transmittance falls below 1/256 (trace_for_eval), before it reaches the opaque layer: that face's
    coverage is just below 1, so it matters whether a ray entering there reads that face's opacity bit (not set: alpha
    *= 1 - coverage) or the bit of the face it leaves by (set: alpha = 0)."""
    idx = np.full((r, r, r), 2, dtype=np.uint16)
    idx[layer(face, r)] = 1
    b = voxel_block(idx, [FACE_TINTS[face] + (1.0, 6.0, 5.0, 4.0), (0.3, 0.4, 0.8, 0.999)], resolution=r)
    assert b.light_opaque_faces == 1 << face
    assert b.light_face_colors[face][3] == 1.0
    assert 0.99 < b.light_face_colors[opposite(face)][3] < 1.0, b.light_face_colors[opposite(face)]
    return b


def sparse_block():
    """A hashed voxel block with partial voxel bounds and translucent palette entries."""
    b = scenes.make_voxel_block(31, resolution=8, palette_size=5, transparent_palette_entry=True)
    assert b.voxel_size != (8, 8, 8) and b.light_opaque_faces == 0
    assert all(0.0 < c[3] < 1.0 for c in b.light_face_colors), b.light_face_colors
    return b


def tinted_glass():
    """A translucent voxel block with holes: every face partly covered."""
    b = scenes.make_voxel_block(57, resolution=R, palette_size=3, alpha=0.25, partial_bounds=False)
    assert b.light_opaque_faces == 0
    assert all(0.0 < c[3] < 1.0 for c in b.light_face_colors), b.light_face_colors
    return b


def face_blocks():
    """The voxel blocks of the scenes, by name."""
    out = {f"one_face_{n}": one_face_block(f) for f, n in enumerate(orc.FACES[1:])}
    out.update({f"veiled_{n}": veiled_block(f) for f, n in enumerate(orc.FACES[1:])})
    out.update(half_slab=half_slab_block(), open_shell=shell_block(PZ), closed_shell=shell_block(),
               two_colour=two_colour_block(), two_colour_z=two_colour_block((0.1, 0.9, 0.1), (0.9, 0.2, 0.9), axis=2),
               emitter=one_face_emitter(), sparse=sparse_block(), glass=tinted_glass())
    return out


ATOMS = [Block(color=(0.5, 0.5, 0.5, 1.0)), Block(color=(0.8, 0.3, 0.2, 1.0)), Block(color=(0.3, 0.6, 0.9, 0.25)),
         Block(color=(0.1, 0.1, 0.1, 1.0), emission=(4.0, 3.0, 1.0))]


def unlit(size):
    light = np.zeros(tuple(size) + (4,), dtype=np.uint8)
    light[..., 3] = NO_RAYS
    return light


def odd_corner_scene(max_distance=30, seed=11):
    """(a) 23 x 9 x 17 at (-37, 5, -1000): a floor of atoms, a quarter of the cubes above it filled with the voxel blocks
    and a few atoms."""
    size = (23, 9, 17)
    vox = face_blocks()
    blocks = [Block.air()] + ATOMS + list(vox.values())
    h = scenes.grid_hash(seed, size)
    filled = (h & np.uint64(3)) == 0
    pick = 2 + ((h >> np.uint64(8)) % np.uint64(len(blocks) - 2)).astype(np.int64)
    ids = np.where(filled, pick, 0).astype(np.uint16)
    ids[:, 0, :] = 1
    return Space((-37, 5, -1000), ids, blocks, light=unlit(size), sky_colors=scenes.OCTANT_SKY,
                 light_max_distance=max_distance)


def mixed_scene():
    """(b) scenes.small_mixed_scene, unlit, with the voxel blocks above appended to its table (for the edits)."""
    sp = scenes.small_mixed_scene(with_light=False)
    return Space(sp.lower, sp.block_ids, sp.blocks + list(face_blocks().values()), light=unlit(sp.size),
                 sky_colors=scenes.OCTANT_SKY, light_max_distance=20)


def translucent_stack():
    """(c) slab_space's layout (test_gpu_group_light) in translucent voxel blocks: three walls and a beam that rays cross
    five and more of, an emitter in front of the walls, shells and veiled blocks beside them."""
    n = 14
    vox = face_blocks()
    blocks = [Block.air(), ATOMS[0], vox["two_colour"], vox["glass"], vox["two_colour_z"], vox["emitter"],
              vox["closed_shell"], vox["open_shell"], vox["sparse"], vox["half_slab"], vox["veiled_NX"],
              vox["veiled_PX"], vox["veiled_NZ"]]
    ids = np.zeros((n, n, n), dtype=np.uint16)
    ids[:, 0, :] = 1
    ids[3:11, 2:9, 6] = 4
    ids[3:11, 2:9, 7] = 3
    ids[3:11, 2:9, 8] = 2
    ids[5:9, 9:13, 3:12] = 2
    ids[6, 4, 2] = 5
    ids[2, 1:4, 3] = 6
    ids[11, 1:4, 3] = 7
    ids[2, 1, 10:13] = 8
    ids[11, 1, 10:13] = 9
    ids[4, 1:4, 2] = 10            # veiled faces towards the emitter ...
    ids[8, 1:4, 2] = 11
    ids[5:8, 1:3, 4] = 12          # ... and towards the glass walls
    return Space((0, 0, 0), ids, blocks, light=unlit((n, n, n)), sky_colors=scenes.OCTANT_SKY, light_max_distance=20)


VOXEL_SCENES = {"odd_corner": odd_corner_scene, "small_mixed": mixed_scene, "translucent_stack": translucent_stack}
ATOM_SCENES = {"light_scene": light_scene, "slab_space": slab_space, "c4_slice": c4_slice}


def relaxed_fields(space, stages=(0, 300, 600, 1200)):
    """The oracle's field after fast_evaluate, then after more and more updates of the queue: compute_light inputs."""
    ol = orc.OracleLight(space)
    ol.fast_evaluate()
    done = 0
    for k in stages:
        ol.evaluate(0, max_updates=k - done)
        done = k
        yield ol, ol.field()


# ---- fast_evaluate --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("make", list(VOXEL_SCENES.values()) + list(ATOM_SCENES.values()),
                         ids=list(VOXEL_SCENES) + list(ATOM_SCENES))
def test_fast_evaluate_equals_the_oracle(make):
    space = make()
    ol = orc.OracleLight(space)
    ol.fast_evaluate()
    rt = SpaceRaytracer(space, GraphicsOptions())
    rt.light_fast_evaluate()
    gpu, ref = rt.light_download(), ol.field()
    assert np.array_equal(gpu, ref), np.argwhere((gpu != ref).any(axis=-1))[:5]
    rt.close()


# ---- compute_light --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(VOXEL_SCENES))
def test_compute_light_is_bit_exact_on_voxel_blocks(name):
    """Every cube, on the oracle's field after fast_evaluate and after 300 / 600 / 1200 updates, on one context and on a
    group of two; the translucent stack must send some cubes through the lockstep walk."""
    space = VOXEL_SCENES[name]()
    cubes = all_cubes(space)
    for stage, (ol, field) in enumerate(relaxed_fields(space)):
        ref = ol.compute(cubes)
        rt = SpaceRaytracer(with_field(space, field), GraphicsOptions())
        got = rt.light_compute(cubes)
        assert np.array_equal(got, ref), f"stage {stage}: {np.argwhere((got != ref).any(axis=1))[:5]}"
        overflow = rt.light_stats()["rounds"]
        if name == "translucent_stack":
            assert 0 < overflow < len(cubes), (stage, overflow)
        rt.close()
        g, gs = group_scene([0, 0], with_field(space, field))
        got = gs.light_compute(cubes)
        assert np.array_equal(got, ref), f"group, stage {stage}: {np.argwhere((got != ref).any(axis=1))[:5]}"
        assert gs.light_stats()["rounds"] == overflow
        assert np.array_equal(assert_replicas_identical(gs, 2), field)
        g.close()


@pytest.mark.parametrize("max_distance", [1, 2, 7, 30, 127, 255])
def test_compute_light_is_bit_exact_at_every_max_distance(max_distance):
    """Rays end where the squared distance exceeds max_distance^2 (updater.rs:452-455); the chart ends at t = 127, so
    127 and 255 walk it whole."""
    space = odd_corner_scene(max_distance=max_distance)
    cubes = all_cubes(space)
    for stage, (ol, field) in enumerate(relaxed_fields(space, stages=(0, 600))):
        ref = ol.compute(cubes)
        rt = SpaceRaytracer(with_field(space, field), GraphicsOptions())
        got = rt.light_compute(cubes)
        assert np.array_equal(got, ref), f"stage {stage}: {np.argwhere((got != ref).any(axis=1))[:5]}"
        rt.close()


# ---- convergence, edits and the changed cubes -----------------------------------------------------------------------
@pytest.mark.parametrize("name,n_edits", [("odd_corner", 300), ("small_mixed", 120), ("translucent_stack", 60)])
@pytest.mark.parametrize("devices", [None, [0, 0]], ids=["ctx", "group2"])
def test_converge_then_edit_voxel_blocks(devices, name, n_edits):
    space = VOXEL_SCENES[name]()
    ol = orc.OracleLight(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    s = Lit(devices, space)
    s.light_fast_evaluate()
    s.light_evaluate(0)
    converged = s.field()
    compare_fields(converged, ol.field())
    # quiescent as test_gpu_light's atom scene: statuses stable, nearly every cube unchanged by a recomputation
    cubes = all_cubes(space)
    again = s.light_compute(cubes).reshape(converged.shape)
    vis = converged[..., 3] == VISIBLE
    d = np.abs(again[..., :3].astype(int) - converged[..., :3].astype(int)).max(axis=-1)[vis]
    assert np.array_equal(again[..., 3][vis], converged[..., 3][vis])
    assert (d == 0).mean() > 0.8 and d.max() <= 12, (float((d == 0).mean()), int(d.max()))

    # edits that swap voxel blocks, atoms and air, closed shells among them
    s.light_take_changes(discard=True)
    before = converged.reshape(-1, 4)
    rng = np.random.default_rng(17)
    edit_cubes = np.stack([rng.integers(0, space.size[a], n_edits) + space.lower[a] for a in range(3)], axis=1).astype(np.int32)
    edit_ids = rng.integers(0, len(space.blocks), n_edits).astype(np.uint16)
    closed = next(i for i, b in enumerate(space.blocks)
                  if b.indices is not None and opaque_for_light(b) and (b.indices == 0).any())   # hollow
    edit_ids[::7] = closed
    ol.set_cubes(edit_cubes, edit_ids)
    ol.evaluate(0)
    updates, _ = s.light_edit_and_propagate(edit_cubes, edit_ids, 0)
    assert updates > 0
    after = s.field()
    compare_fields(after, ol.field())
    idx, tx = s.light_take_changes()
    assert np.array_equal(tx, after.reshape(-1, 4)[idx])
    taken = set(idx.tolist())
    changed = np.flatnonzero((before != after.reshape(-1, 4)).any(axis=1))
    missing = [int(i) for i in changed if int(i) not in taken]
    assert not missing, f"{len(missing)} changed texels not announced, e.g. {missing[:5]}"
    opaque = cubes_set_opaque(space, edit_cubes, edit_ids)
    assert opaque <= taken, sorted(opaque - taken)[:5]
    final_ids = space.block_ids.reshape(-1).copy()
    for c, i in zip(edit_cubes, edit_ids):
        final_ids[np.ravel_multi_index(tuple(c - np.array(space.lower)), space.size)] = i
    assert any(final_ids[i] == closed for i in opaque), "no closed shell was set"
    s.close()


# ---- light_on_slab lit by the GPU -----------------------------------------------------------------------------------
_SLAB_LIT = []


def slab_lit_by_gpu():
    """The light_on_slab universe (test_golden_images) with its light from GPU fast_evaluate + evaluate(1), as the
    reference builds it, and the oracle's field of the same calls."""
    if not _SLAB_LIT:
        from test_golden_images import build_light_on_slab_universe
        ref = build_light_on_slab_universe()
        space = Space(ref.lower, ref.block_ids, ref.blocks, light=unlit(ref.size), sky_colors=ref.sky_colors,
                      light_max_distance=30)
        rt = SpaceRaytracer(space, GraphicsOptions())
        rt.light_fast_evaluate()
        rt.light_evaluate(1)
        _SLAB_LIT.append((with_field(ref, rt.light_download()), ref))
        rt.close()
    return _SLAB_LIT[0]


def test_light_on_slab_field_lit_by_gpu_meets_the_contract():
    gpu, ref = slab_lit_by_gpu()
    assert np.array_equal(gpu.light[..., 3], ref.light[..., 3])
    compare_fields(gpu.light, ref.light)


@pytest.mark.parametrize("name,lighting", [("None", aicb200.LIGHT_NONE), ("Flat", aicb200.LIGHT_FLAT),
                                           ("Coarse", aicb200.LIGHT_COARSE), ("Linear", aicb200.LIGHT_LINEAR),
                                           ("Smoothstep", aicb200.LIGHT_SMOOTHSTEP)])
def test_light_on_slab_lit_by_gpu_meets_the_reference_threshold(name, lighting):
    """The reference's light_on_slab images, drawn by the oracle renderer as test_golden_images draws them, from the
    field the GPU propagated: the reference's threshold, 7 on every pixel."""
    from test_golden_images import check_threshold, golden, light_on_slab_camera
    gpu, _ = slab_lit_by_gpu()
    opts = GraphicsOptions.unaltered_colors()
    opts.lighting_display = lighting
    opts.fov_y = 45.0
    img = orc.OracleScene(gpu).render(light_on_slab_camera(opts), opts)["srgb8"].reshape(96, 128, 4)
    check_threshold(img, golden(f"light_on_slab-{name}-all"), [(7, 128 * 96)])
