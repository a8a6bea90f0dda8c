"""aicb_derive_block_light (Context.derive_block_light): compute_derived's light fields on the GPU, bit for bit equal to
the oracle (oracle_derive/, correctly rounded powf as the device computes it), over resolutions, data bounds, alphas,
emission, wide palettes and overflowing sums; batches, validation, and light propagation fed the device's fields."""
import copy
import ctypes as C

import numpy as np
import pytest

import aicb200
import deriveorc
import orc
from aicb200 import GraphicsOptions, Block, Space, SpaceRaytracer, abi, scenes
from test_gpu_light import all_cubes, compare_fields
from test_gpu_light_voxels import mixed_scene, translucent_stack

pytestmark = pytest.mark.gpu

RESOLUTIONS = [1, 2, 4, 8, 16, 32, 64, 128]
ALPHAS = np.array([0.0, 1e-7, 0.125, 0.5, 0.999, 1.0], dtype=np.float32)


@pytest.fixture(scope="module")
def ctx():
    deriveorc.set_libm(deriveorc.LIBM_CR)   # powf as the device computes it
    c = aicb200.Context(0)
    yield c
    c.close()


def bits(lights):
    """Every field of every BlockLight as u32 bit patterns (floats) and integers, for an exact comparison."""
    out = []
    for bl in lights:
        f = np.array([v for c in bl.face_colors for v in c] + list(bl.color) + list(bl.emission), dtype=np.float32)
        out.append(tuple(f.view(np.uint32).tolist()) + (bl.opaque_faces, int(bl.visible)))
    return out


def assert_equal_to_oracle(ctx, blocks):
    got, ref = ctx.derive_block_light(blocks), deriveorc.derive(blocks)
    for i, (g, r) in enumerate(zip(bits(got), bits(ref))):
        assert g == r, f"block {i}: device {got[i]} != oracle {ref[i]}"
    return got


def random_block(rng, res, bounds="full", palette_size=12, alphas=ALPHAS, emissive=0.3, invisible=0.2, scale=1.0):
    """A block of `res` with random data bounds of the kind `bounds`, and a palette of random colours, alphas drawn
    from `alphas`, some emissive entries, some unused ones; about `invisible` of the voxels use an invisible entry."""
    if bounds == "full" or res == 1:
        lo, size = [0, 0, 0], [res, res, res]
    elif bounds == "partial":
        lo = [int(rng.integers(0, res // 2 + 1)) for _ in range(3)]
        size = [int(rng.integers(1, res - lo[a] + 1)) for a in range(3)]
    elif bounds == "one_face":   # reaches one face of the block only
        a = int(rng.integers(0, 3))
        lo, size = [1, 1, 1], [res - 2, res - 2, res - 2]
        if int(rng.integers(0, 2)):
            lo[a], size[a] = 0, res - 1
        else:
            size[a] = res - 1
        size = [max(s, 1) for s in size]
    elif bounds == "slab":       # one voxel thick
        a = int(rng.integers(0, 3))
        lo, size = [0, 0, 0], [res, res, res]
        lo[a], size[a] = int(rng.integers(0, res)), 1
    pal = np.zeros((palette_size, 8), dtype=np.float32)
    pal[:, :3] = rng.random((palette_size, 3), dtype=np.float32) * np.float32(scale)
    pal[:, 3] = rng.choice(alphas, palette_size)
    emits = rng.random(palette_size) < emissive
    pal[emits, 4:7] = rng.random((int(emits.sum()), 3), dtype=np.float32) * np.float32(3.0)
    pal[0, :] = 0.0                   # the invisible entry
    used = palette_size - 2           # the last two entries stay unused
    idx = rng.integers(1, used, size=tuple(size)).astype(np.uint16)
    idx[rng.random(tuple(size)) < invisible] = 0
    return Block(resolution=res, voxel_lower=lo, indices=idx, palette=pal)


@pytest.mark.parametrize("res", RESOLUTIONS)
def test_every_resolution_equals_the_oracle(ctx, res):
    rng = np.random.default_rng(res)
    kinds = ["full", "partial", "one_face", "slab"]
    n_each = 4 if res <= 32 else 1
    blocks = [random_block(rng, res, k) for k in kinds for _ in range(n_each)]
    # alpha by alpha: every voxel of one alpha, with and without emission
    blocks += [random_block(rng, res, "full", alphas=np.array([a], dtype=np.float32), emissive=e, invisible=0.0)
               for a in (ALPHAS if res <= 32 else ALPHAS[[1, 3, 4]]) for e in (0.0, 1.0)]
    assert_equal_to_oracle(ctx, blocks)


def test_emissive_transparent_voxels(ctx):
    rng = np.random.default_rng(7)
    blocks = [random_block(rng, r, "partial", alphas=np.array([0.0, 1e-7, 0.125], dtype=np.float32), emissive=1.0,
                           invisible=0.0) for r in (2, 8, 16, 32)]
    got = assert_equal_to_oracle(ctx, blocks)
    assert all(any(v > 0.0 for v in g.emission) for g in got)


def test_single_voxels_and_air(ctx):
    blocks = [Block.air(), Block(color=(1.0, 2.0, 3.0, 1.0), emission=(1.0, 1.0, 1.0)), Block(color=(0.2, 0.3, 0.4, 0.5)),
              Block(color=(0.0, 0.0, 0.0, 0.0), emission=(1.0, 2.0, 3.0)), Block(color=(0.5, 0.5, 0.5, 0.0))]
    pal = np.zeros((2, 8), dtype=np.float32)
    pal[1, :4] = (0.25, 0.5, 0.75, 1.0)
    blocks.append(Block(resolution=1, indices=np.ones((1, 1, 1), dtype=np.uint16), palette=pal))
    got = assert_equal_to_oracle(ctx, blocks)
    assert [g.visible for g in got] == [False, True, True, True, False, True]


def test_wide_palette(ctx):
    """A palette over 32 768 entries, most of them used (the scenes keep such a block in 4-byte brick words)."""
    rng = np.random.default_rng(3)
    n = 40000
    pal = np.zeros((n, 8), dtype=np.float32)
    pal[:, :3] = rng.random((n, 3), dtype=np.float32)
    pal[:, 3] = rng.choice(ALPHAS, n)
    pal[::5, 4:7] = 0.5
    idx = rng.integers(0, n, size=(64, 64, 64)).astype(np.uint16)
    idx[0, 0, 0] = n - 1
    assert_equal_to_oracle(ctx, [Block(resolution=64, indices=idx, palette=pal)])


@pytest.mark.parametrize("scale,emission", [(1e28, 1.0), (3e38, 1.0), (1.0, np.inf), (np.inf, 0.0), (1e28, np.inf)])
def test_overflowing_sums_match_the_oracle(ctx, scale, emission):
    """Huge colours and infinite emission: the device's result is the oracle's value, or, where the oracle reports the
    reference's panic, AICB_ERR_INVALID naming the block."""
    rng = np.random.default_rng(11)
    for res in (4, 16):
        for alphas in (np.array([0.5], dtype=np.float32), np.array([1e-7, 1.0], dtype=np.float32), ALPHAS):
            b = random_block(rng, res, "full", alphas=alphas, emissive=0.0, invisible=0.0)
            b.palette[1:, :3] *= np.float32(scale)
            b.palette[1::2, 4:7] = np.float32(emission)
            blocks = [Block(color=(0.1, 0.2, 0.3, 1.0)), b]
            try:
                ref = deriveorc.derive(blocks)
            except deriveorc.DerivePanic as p:
                assert p.position == 1
                with pytest.raises(aicb200.AicbError) as e:
                    ctx.derive_block_light(blocks)
                assert e.value.status == abi.ERR_INVALID and "block 1" in str(e.value)
                continue
            assert bits(ctx.derive_block_light(blocks)) == bits(ref)


def test_nan_sum_fails_and_names_the_block(ctx):
    pal = np.zeros((3, 8), dtype=np.float32)
    pal[1, :4] = (1.0, 1.0, 1.0, 0.5)
    pal[1, 4:7] = (np.inf, 0.0, 0.0)
    pal[2, :4] = (1.0, 1.0, 1.0, 0.5)
    pal[2, 4:7] = (-np.inf, 0.0, 0.0)
    idx = np.ones((4, 4, 4), dtype=np.uint16)
    idx[:, :, 2:] = 2
    blocks = [Block(color=(1.0, 1.0, 1.0, 1.0)), scenes.make_voxel_block(1, resolution=8),
              Block(resolution=4, indices=idx, palette=pal)]
    with pytest.raises(deriveorc.DerivePanic):
        deriveorc.derive(blocks)
    descs = aicb200._block_descs(blocks)
    out = (abi.BlockLight * 3)()
    C.memset(out, 0xA5, C.sizeof(out))
    before = bytes(out)
    lib = aicb200.load_library()
    assert lib.aicb_derive_block_light(ctx.handle, descs, 3, out) == abi.ERR_INVALID
    assert "block 2" in lib.aicb_last_error().decode()
    assert bytes(out) == before


def test_one_call_equals_one_call_per_block(ctx):
    rng = np.random.default_rng(5)
    blocks = [random_block(rng, int(r), str(k)) for r, k in
              zip(rng.choice([1, 2, 4, 8, 16, 32], 40), rng.choice(["full", "partial", "one_face", "slab"], 40))]
    blocks[3:3] = [Block.air(), Block(color=(0.5, 0.5, 0.5, 0.5))]
    together = bits(ctx.derive_block_light(blocks))
    alone = [bits(ctx.derive_block_light([b]))[0] for b in blocks]
    assert together == alone
    assert together == bits(deriveorc.derive(blocks))


def test_no_blocks(ctx):
    assert ctx.derive_block_light([]) == []
    lib = aicb200.load_library()
    assert lib.aicb_derive_block_light(ctx.handle, None, 0, None) == abi.OK


def _bad_blocks():
    good = scenes.make_voxel_block(2, resolution=8)
    pal = good.palette
    cases = {}
    b = copy.copy(good); b.resolution = 3
    cases["resolution"] = (b, abi.ERR_INVALID)
    b = copy.copy(good); b.voxel_lower = (7, 0, 0)
    cases["bounds"] = (b, abi.ERR_INVALID)
    b = copy.copy(good); b.indices = good.indices.copy(); b.indices[0, 0, 0] = pal.shape[0]
    cases["index"] = (b, abi.ERR_INVALID)
    big = np.zeros((65537, 8), dtype=np.float32)
    cases["palette_too_big"] = (Block(resolution=4, indices=np.zeros((4, 4, 4), dtype=np.uint16), palette=big),
                                abi.ERR_UNSUPPORTED)
    return good, cases


@pytest.mark.parametrize("case", ["resolution", "bounds", "index", "palette_too_big", "n_indices", "null_palette"])
def test_invalid_blocks_leave_out_untouched(ctx, case):
    good, cases = _bad_blocks()
    lib = aicb200.load_library()
    if case in cases:
        bad, status = cases[case]
        descs = aicb200._block_descs([good, bad])
    else:
        descs, status = aicb200._block_descs([good, good]), abi.ERR_INVALID
        if case == "n_indices":
            descs[1].n_indices -= 1
        else:
            descs[1].palette = None
    out = (abi.BlockLight * 2)()
    C.memset(out, 0x5A, C.sizeof(out))
    before = bytes(out)
    assert lib.aicb_derive_block_light(ctx.handle, descs, 2, out) == status
    assert "block 1" in lib.aicb_last_error().decode()
    assert bytes(out) == before
    # the same block is refused by scene creation, with the same status
    if case in cases:
        sp = Space((0, 0, 0), np.ones((2, 2, 2), dtype=np.uint16), [Block.air(), cases[case][0]])
        with pytest.raises(aicb200.AicbError) as e:
            SpaceRaytracer(sp, GraphicsOptions())
        assert e.value.status == status


def test_null_pointers(ctx):
    lib = aicb200.load_library()
    descs = aicb200._block_descs([Block.air()])
    out = (abi.BlockLight * 1)()
    assert lib.aicb_derive_block_light(ctx.handle, None, 1, out) == abi.ERR_INVALID
    assert lib.aicb_derive_block_light(ctx.handle, descs, 1, None) == abi.ERR_INVALID
    assert lib.aicb_derive_block_light(None, descs, 1, out) == abi.ERR_INVALID


@pytest.mark.parametrize("make", [mixed_scene, translucent_stack], ids=["small_mixed", "translucent_stack"])
def test_light_from_device_derived_blocks(ctx, make):
    """A voxel scene whose recursive blocks take their light fields from the device: fast_evaluate and compute_light
    on the GPU give the light oracle's texels byte for byte, the oracle being fed the oracle's derived fields; a
    converged field agrees as closely as the reference's own queue order allows (test_gpu_light.compare_fields)."""
    space = make()
    dev_blocks, orc_blocks = [copy.copy(b) for b in space.blocks], [copy.copy(b) for b in space.blocks]
    recursive = [i for i, b in enumerate(space.blocks) if b.indices is not None]
    assert recursive
    for i, bl in zip(recursive, ctx.derive_block_light([dev_blocks[i] for i in recursive])):
        dev_blocks[i].set_light_data(bl)
    for i, bl in zip(recursive, deriveorc.derive([orc_blocks[i] for i in recursive])):
        orc_blocks[i].set_light_data(bl)
    dev = Space(space.lower, space.block_ids, dev_blocks, light=space.light, sky_colors=space.sky_colors,
                light_max_distance=space.light_max_distance)
    ref = Space(space.lower, space.block_ids, orc_blocks, light=space.light, sky_colors=space.sky_colors,
                light_max_distance=space.light_max_distance)
    ol = orc.OracleLight(ref)
    ol.fast_evaluate()
    rt = SpaceRaytracer(dev, GraphicsOptions())
    rt.light_fast_evaluate()
    field = ol.field()
    assert np.array_equal(rt.light_download(), field)
    cubes = all_cubes(dev)
    assert np.array_equal(rt.light_compute(cubes), ol.compute(cubes))
    rt.light_evaluate(0)
    ol.evaluate(0)
    compare_fields(rt.light_download(), ol.field())
    rt.close()
