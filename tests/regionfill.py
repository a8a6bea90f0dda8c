"""Boxes of cubes for the tests of the box calls (aicb_scene_update_region, aicb_light_edit_region): the cubes of a box in
GridAab::interior_iter order, fills that mix kept and changed cubes, and the Space a fill leaves."""
import numpy as np

from aicb200 import Space

# Boxes inside test_gpu_light.light_scene (14^3 at (-2, 1, 3)), as (lower, size).  The first touches the lower x face
# and starts at an odd z offset with 9 cubes per row; the second touches the upper x, lower y and upper z faces with 11
# cubes per row from z offset 3: every row of both has an unaligned head and tail.
BOXES = (((-2, 3, 4), (5, 6, 9)), ((3, 1, 6), (9, 4, 11)))


def box_cubes(lower, size):
    """The box's cubes in interior_iter order (grid_iter.rs:75-106): z fastest, then y, then x."""
    x, y, z = np.meshgrid(*[np.arange(lower[a], lower[a] + size[a]) for a in range(3)], indexing="ij")
    return np.stack([x.ravel(), y.ravel(), z.ravel()], axis=1).astype(np.int32)


def box_slices(space, lower, size):
    return tuple(slice(lower[a] - space.lower[a], lower[a] - space.lower[a] + size[a]) for a in range(3))


def mixed_fill(space, lower, size, seed):
    """Ids of shape `size`: about a third of the cubes keep their block, the others draw from the whole table."""
    rng = np.random.default_rng(seed)
    old = space.block_ids[box_slices(space, lower, size)]
    drawn = rng.integers(0, len(space.blocks), old.shape).astype(np.uint16)
    return np.where(rng.random(old.shape) < 0.33, old, drawn).astype(np.uint16)


def filled(space, lower, size, ids, light=None):
    """The Space after the fill (`ids`: one id or an array of shape `size`), with `light` or the light it had."""
    out = space.block_ids.copy()
    out[box_slices(space, lower, size)] = ids
    return Space(space.lower, out, space.blocks, light=space.light if light is None else light,
                 sky_colors=space.sky_colors, light_max_distance=space.light_max_distance)
