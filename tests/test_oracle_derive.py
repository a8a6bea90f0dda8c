"""The compute_derived oracle (oracle_derive/) against the reference's own known answers (block/eval/tests.rs), and
against Block's numpy restatement on the synthetic blocks of aicb200/scenes.py.  CPU only."""
import numpy as np
import pytest

import deriveorc
from aicb200 import Block, scenes

F32 = np.float32
TRANSPARENT = (0.0, 0.0, 0.0, 0.0)


@pytest.fixture(autouse=True, scope="module")
def _libm():
    deriveorc.set_libm(deriveorc.LIBM_PLATFORM)   # what Rust's std calls on this host
    yield


def voxels_fn(res, fn, lower=(0, 0, 0), size=None):
    """Block::builder().voxels_fn(res, fn) over the data bounds `lower`, `size` (default the whole block): fn(x, y, z)
    -> (rgba, emission); equal voxels share a palette entry."""
    size = size or (res, res, res)
    pal, idx = {}, np.zeros(size, dtype=np.uint16)
    for x in range(size[0]):
        for y in range(size[1]):
            for z in range(size[2]):
                rgba, em = fn(lower[0] + x, lower[1] + y, lower[2] + z)
                key = tuple(float(F32(v)) for v in rgba) + tuple(float(F32(v)) for v in em)
                idx[x, y, z] = pal.setdefault(key, len(pal))
    palette = np.zeros((len(pal), 8), dtype=np.float32)
    for key, i in pal.items():
        palette[i, :7] = key
    return Block(resolution=res, voxel_lower=lower, indices=idx, palette=palette)


def color(rgba):
    return (lambda x, y, z: (rgba, (0.0, 0.0, 0.0)))


def one(block):
    return deriveorc.derive([block])[0]


def f32s(*v):
    return tuple(float(F32(x)) for x in v)


# ---- block/eval/tests.rs ---------------------------------------------------------------------------------------------
def test_overall_color_ignores_interior():
    outer, inner = (1.0, 0.0, 0.0, 1.0), (0.0, 1.0, 0.0, 1.0)
    b = voxels_fn(8, lambda x, y, z: (inner if all(1 <= c < 7 for c in (x, y, z)) else outer, (0.0, 0.0, 0.0)))
    assert one(b).color == outer


def test_opaque_atom():
    e = one(Block(color=(1.0, 2.0, 3.0, 1.0), emission=(1.0, 1.0, 1.0)))
    assert e.color == (1.0, 2.0, 3.0, 1.0)
    assert e.face_colors == ((1.0, 2.0, 3.0, 1.0),) * 6
    assert e.emission == (1.0, 1.0, 1.0)
    assert e.opaque_faces == 0x3F and e.visible


def test_transparent_atom():
    e = one(Block(color=(1.0, 2.0, 3.0, 0.5)))
    assert e.color == (1.0, 2.0, 3.0, 0.5) and e.face_colors == ((1.0, 2.0, 3.0, 0.5),) * 6
    assert e.emission == (0.0, 0.0, 0.0)
    assert e.opaque_faces == 0 and e.visible


def test_emissive_only_atom():
    e = one(Block(color=TRANSPARENT, emission=(1.0, 2.0, 3.0)))
    assert e.color == TRANSPARENT and e.face_colors == (TRANSPARENT,) * 6
    assert e.emission == (1.0, 2.0, 3.0)
    assert e.opaque_faces == 0 and e.visible


def test_invisible_atom():
    e = one(Block(color=TRANSPARENT))
    assert e.color == TRANSPARENT and e.face_colors == (TRANSPARENT,) * 6
    assert e.opaque_faces == 0 and not e.visible


def test_voxels_checked_individually():
    e = one(voxels_fn(2, lambda x, y, z: ((float(x), float(y), float(z), 1.0), (0.0, 0.0, 0.0))))
    assert e.color == (0.5, 0.5, 0.5, 1.0)
    assert e.face_colors == ((0.0, 0.5, 0.5, 1.0), (0.5, 0.0, 0.5, 1.0), (0.5, 0.5, 0.0, 1.0),
                             (1.0, 0.5, 0.5, 1.0), (0.5, 1.0, 0.5, 1.0), (0.5, 0.5, 1.0, 1.0))
    assert e.opaque_faces == 0x3F and e.visible


@pytest.mark.parametrize("reflectance", [TRANSPARENT, (0.0, 0.5, 1.0, 0.5)])
@pytest.mark.parametrize("resolution", [1, 2, 4, 32])
def test_voxels_emission_equivalence(reflectance, resolution):
    atom_emission = (1.0, 2.0, 3.0)
    b = voxels_fn(resolution, lambda x, y, z: (reflectance, atom_emission))
    total = np.array(one(b).emission, dtype=np.float32)
    difference = total - np.array(atom_emission, dtype=np.float32)
    assert float(np.sqrt(np.sum(difference * difference, dtype=np.float32))) < 0.0001, total


def test_transparent_voxels_simple():
    res, alpha = 4, F32(0.5)
    rgb = (1.0, 0.5, 0.0)
    b = voxels_fn(res, lambda x, y, z: (rgb + ((float(alpha) if x == 0 and z == 0 else 1.0),), (0.0, 0.0, 0.0)))
    e = one(b)
    squared = F32(res * res)
    assert e.color == rgb + f32s(F32(1.0) - alpha / (squared * F32(3.0)))
    one_face = rgb + f32s(F32(1.0) - alpha / squared)
    opaque = rgb + (1.0,)
    assert e.face_colors == (opaque, one_face, opaque, opaque, one_face, opaque)
    assert e.opaque_faces == (1 << 3) | (1 << 5)   # PX, PZ
    assert e.visible


@pytest.mark.xfail(strict=True, reason="the reference ignores this test: 'not sure if code or test is wrong'")
def test_transparent_voxels_weighted():
    c1, c2 = np.array([1.0, 0.0, 0.0], dtype=np.float32), np.array([0.0, 1.0, 0.0], dtype=np.float32)
    colors = [(1.0, 0.0, 0.0, 1.0), (0.0, 1.0, 0.0, 0.5)]
    e = one(voxels_fn(2, lambda x, y, z: (colors[y], (0.0, 0.0, 0.0))))
    surface_area = F32(4.0 * 6.0)
    half_semi_alpha = F32(0.5) ** F32(0.5)
    semi_on_opaque_blend = c1 * (F32(1.0) - half_semi_alpha) + c2 * half_semi_alpha
    expected = (c1 * F32(4.0) + semi_on_opaque_blend * F32(4.0) + c1 * F32(8.0) + c2 * F32(4.0)) * (F32(1.0) / surface_area)
    assert e.color[:3] == tuple(float(v) for v in expected)


def test_voxels_full_but_transparent():
    res = 4
    e = one(voxels_fn(res, lambda x, y, z: ((0.0, 0.0, 0.0, 1.0 if (x, y, z) == (1, 1, 1) else 0.0), (0.0, 0.0, 0.0))))
    assert e.color == (0.0, 0.0, 0.0, float(F32(1.0) / F32(res * res)))
    assert e.opaque_faces == 0 and e.visible


def test_voxels_partial_not_filling():
    e = one(voxels_fn(4, color((1.0, 1.0, 1.0, 1.0)), size=(2, 4, 4)))
    assert e.color == (1.0, 1.0, 1.0, float(F32(8.0) / F32(12.0)))
    assert e.opaque_faces == 1   # NX alone
    assert e.visible


def test_air_data_gives_zeros():
    air = one(Block.air())
    assert air.color == TRANSPARENT and air.face_colors == (TRANSPARENT,) * 6 and air.emission == (0.0, 0.0, 0.0)
    assert air.opaque_faces == 0 and not air.visible


def test_invisible_interior_voxel_is_not_visible_but_emission_is():
    """visible counts every data voxel through its opacity category, not the palette: unused entries do not count,
    hidden emissive voxels do."""
    pal = np.zeros((3, 8), dtype=np.float32)
    pal[1, :4] = (1.0, 1.0, 1.0, 1.0)          # unused
    pal[2, 4:7] = (0.5, 0.0, 0.0)              # transparent, emissive
    idx = np.zeros((4, 4, 4), dtype=np.uint16)
    assert not one(Block(resolution=4, indices=idx, palette=pal)).visible
    idx[2, 2, 2] = 2
    assert one(Block(resolution=4, indices=idx, palette=pal)).visible


# ---- against Block's numpy restatement --------------------------------------------------------------------------------
def ulps(a, b):
    a = np.array(a, dtype=np.float32).view(np.int32).astype(np.int64)
    b = np.array(b, dtype=np.float32).view(np.int32).astype(np.int64)
    a = np.where(a < 0, -(a & 0x7FFFFFFF), a)
    b = np.where(b < 0, -(b & 0x7FFFFFFF), b)
    return int(np.abs(a - b).max())


@pytest.mark.parametrize("alpha", [1.0, 0.5, 0.05])
@pytest.mark.parametrize("resolution", [2, 8, 16, 32])
def test_oracle_agrees_with_the_numpy_restatement(resolution, alpha):
    blocks = [scenes.make_voxel_block(seed, resolution=resolution, alpha=alpha, emissive_every=3,
                                      partial_bounds=seed % 2 == 0, transparent_palette_entry=seed % 3 == 0)
              for seed in range(6)]
    # numpy sums pairwise, the reference one term after another: the two roundings of a sum of up to 6 * res^2 terms
    # differ by about res ULP (measured: 25 at res 16, 83 at 32, 252 at 64)
    for b, e in zip(blocks, deriveorc.derive(blocks)):
        assert e.opaque_faces == b.light_opaque_faces
        assert e.visible == b.light_visible
        assert ulps(e.color, b.light_color) <= 4 * resolution
        assert ulps(e.face_colors, b.light_face_colors) <= 4 * resolution
        assert ulps(e.emission, b.light_emission) <= 4 * resolution


def test_the_reference_panics_on_a_nan_sum():
    pal = np.zeros((3, 8), dtype=np.float32)
    pal[1, :4] = (1.0, 1.0, 1.0, 0.5)
    pal[1, 4:7] = (np.inf, 0.0, 0.0)
    pal[2, :4] = (1.0, 1.0, 1.0, 0.5)
    pal[2, 4:7] = (-np.inf, 0.0, 0.0)   # no Rgb holds it, but the C ABI passes it on: inf + -inf is NaN
    idx = np.ones((4, 4, 4), dtype=np.uint16)
    idx[:, :, 2:] = 2
    good = voxels_fn(2, color((1.0, 1.0, 1.0, 1.0)))
    with pytest.raises(deriveorc.DerivePanic) as e:
        deriveorc.derive([good, Block(resolution=4, indices=idx, palette=pal)])
    assert e.value.position == 1
