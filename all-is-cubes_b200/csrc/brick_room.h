// brick_room.h — whether a scene's brick pool has room for more voxel words (aicb200.cu: flatten_blocks and
// flatten_placeable).  Plain host code with no CUDA, so that a host compiler alone can test it (tests/test_brick_room.py).
#pragma once
#include <cstddef>
#include <cstdint>

// Brick positions are u32 (BlockRec::brick_off, the hit records): the words in use after an append of `added` words,
// live and dead, must stay below 2^32.  The dead words can be compacted away first; the live ones cannot.
enum class BrickRoom {
    fits,            // place as it is
    compact_first,   // the live data fits, its positions would not: compact the brick pool, then flatten again
    too_big,         // the live data alone passes 2^32 words: rejected
};

inline BrickRoom brick_room(uint64_t n_bricks, uint64_t dead_bricks, uint64_t added) {
    const uint64_t LIMIT = 0xffffffffull;
    if (n_bricks - dead_bricks + added > LIMIT) return BrickRoom::too_big;
    if (n_bricks + added > LIMIT) return BrickRoom::compact_first;
    return BrickRoom::fits;
}
