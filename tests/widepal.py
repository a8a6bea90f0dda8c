"""Blocks whose palettes have more than 32768 entries (a scene's brick pool takes u32 words for them), and their twins:
the same voxels with the palette deduplicated below 32768 entries.  A Space with one draws, lights and reports exactly
as the same Space with the other.  Test infrastructure, shared by the oracle and the GPU tests."""
import numpy as np

from aicb200 import Block, Space, scenes

# The distinct voxels of a wide palette: entry k of a palette is KINDS[k % len(KINDS)].
AIR, INVISIBLE, TRANSLUCENT, EMISSIVE_CLEAR, EMISSIVE = 0, 1, 2, 3, 4


def voxel_kinds(seed, n=97):
    """n distinct voxels: AIR, an invisible non-AIR voxel, a translucent one, an emitter with alpha 0, an opaque
    emitter, then opaque and translucent colours (alpha 1, 0.5, 0.25, 0.125)."""
    pal = np.zeros((n, 8), np.float32)
    pal[5:, :4] = scenes.make_palette(seed, n - 5)[:, :4]
    pal[5:, 3] = np.array([1.0, 0.5, 0.25, 0.125], np.float32)[np.arange(n - 5) % 4]
    pal[INVISIBLE, :4] = (0.6, 0.2, 0.4, 0.0)
    pal[TRANSLUCENT, :4] = (0.2, 0.7, 0.9, 0.375)
    pal[EMISSIVE_CLEAR, 4:7] = (0.4, 1.5, 0.6)
    pal[EMISSIVE, :4] = (0.3, 0.2, 0.1, 1.0)
    pal[EMISSIVE, 4:7] = (2.0, 1.0, 0.25)
    return pal


def wide_block(seed, resolution, n_palette, fill=0.125):
    """A full block of `resolution` whose palette has n_palette entries (each a copy of one of voxel_kinds), with its
    twin.  A fraction `fill` of the voxels is visible; the others are AIR entries.  Voxels take entries from the whole
    palette, so entries above 32767 of every kind are used, and the last entry, n_palette - 1, is used too."""
    kinds = voxel_kinds(seed)
    d = len(kinds)
    rng = np.random.default_rng(seed)
    shape = (resolution,) * 3
    idx = rng.integers(0, n_palette, shape, dtype=np.int64)
    air = rng.random(shape) >= fill
    idx[air] = (idx[air] // d) * d   # an AIR entry near the drawn one
    # the last entry, and one entry above 32767 of each special kind, on the block's near faces
    special = [n_palette - 1] + [((n_palette - 1 - k) // d) * d + k for k in (INVISIBLE, TRANSLUCENT, EMISSIVE_CLEAR,
                                                                                EMISSIVE)]
    for j, e in enumerate(special):
        idx[resolution - 1, :, 4 * j:4 * j + 3] = e
        idx[:, resolution - 1, 4 * j + 1] = e
    idx = idx.astype(np.uint16)
    wide = Block(resolution=resolution, indices=idx, palette=kinds[np.arange(n_palette) % d])
    twin = Block(resolution=resolution, indices=(idx % d).astype(np.uint16), palette=kinds)
    return wide, twin


def space_with(block, n=8, seed=7, at=((7, 7, 7), (7, 5, 6), (6, 7, 4), (5, 6, 7), (7, 4, 3), (3, 7, 7))):
    """small_mixed_scene (every block kind) with `block` as the table's last id, at a few cubes the standard camera sees."""
    base = scenes.small_mixed_scene(n=n, seed=seed)
    ids = base.block_ids.copy()
    wid = len(base.blocks)
    for c in at:
        ids[c] = wid
    blocks = base.blocks + [block]
    return Space(base.lower, ids, blocks, light=scenes.noise_light(seed + 5, ids, blocks), sky_colors=base.sky_colors,
                 light_max_distance=base.light_max_distance)
