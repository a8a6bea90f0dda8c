"""The light oracle's side of a block redefinition (oracle_light/: orc_light_update_blocks, orc_light_append_blocks,
orc_light_relight_blocks), on the CPU.  Relighting index L after redefining it must give exactly the field that
placing a new index L' with the same definition in every cube holding L gives (Mutation::set -> modified_cube_needs_update,
space/light/updater.rs:135-173): both queue the same cubes at the same priority, and the oracle pops them in a fixed
order."""
import numpy as np
import pytest

from aicb200 import Block
from lightorc import LightOracle
from test_gpu_light import light_scene

# light_scene's blocks: 1 floor (opaque), 2 opaque, 3 translucent, 4 nearly clear, 5 opaque emitter, 6 invisible emitter,
# 7 invisible
REDEFINITIONS = {
    "opaque_becomes_emissive": (2, Block(color=(0.2, 0.9, 0.3, 1.0), emission=(3.0, 2.0, 1.0))),
    "translucent_becomes_opaque": (3, Block(color=(0.9, 0.2, 0.1, 1.0))),
    "emitter_goes_dark_and_clear": (5, Block(color=(0.1, 0.1, 0.1, 0.25))),
    "face_colour_changes": (1, Block(color=(0.1, 0.3, 0.9, 1.0))),
}


def converged(space):
    ol = LightOracle(space)
    ol.fast_evaluate()
    ol.evaluate(0)
    return ol


def holders(space, index):
    """The cubes holding `index`, in increasing linear index order."""
    at = np.argwhere(space.block_ids == index)   # (row-major: increasing linear index)
    return (at + np.array(space.lower)).astype(np.int32)


@pytest.mark.parametrize("name", sorted(REDEFINITIONS))
def test_relight_equals_placing_a_copy_in_every_holding_cube(name):
    index, block = REDEFINITIONS[name]
    space = light_scene(seed=9)
    relit, placed = converged(space), converged(space)
    assert np.array_equal(relit.field(), placed.field())
    relit.update_blocks([index], [block])
    relit.relight_blocks([index])
    relit_updates = relit.evaluate(0)[0]
    placed.append_blocks([block])
    cubes = holders(space, index)
    assert len(cubes) > 0
    placed.set_cubes(cubes, np.full(len(cubes), len(space.blocks), dtype=np.uint16))
    placed_updates = placed.evaluate(0)[0]
    assert relit_updates == placed_updates > 0
    assert np.array_equal(relit.field(), placed.field())


def test_duplicates_unused_indices_and_none():
    space = light_scene(seed=9)
    once, twice = converged(space), converged(space)
    block = REDEFINITIONS["translucent_becomes_opaque"][1]
    for ol, indices in ((once, [3]), (twice, [3, 3])):
        ol.update_blocks([3], [block])
        ol.relight_blocks(indices)
    assert once.queue_len() == twice.queue_len() > 0
    once.evaluate(0)
    twice.evaluate(0)
    assert np.array_equal(once.field(), twice.field())
    # an index no cube holds queues nothing; neither does an empty list
    assert once.queue_len() == 0
    once.append_blocks([Block(color=(1.0, 1.0, 1.0, 1.0), emission=(1.0, 1.0, 1.0))])
    once.relight_blocks([len(space.blocks)])
    once.relight_blocks([])
    assert once.queue_len() == 0
