"""Lists of scattered Mutation::set entries for the tests of aicb_light_edit_cubes, and a numpy restatement of how the
library applies one: the entries whose id changes the cube's block at that point of the list, the final cells,
OPAQUE for every changing entry whose own block is opaque for light, then modified_cube_needs_update
(space/light/updater.rs:135-173) for every changing entry against the final cells (DESIGN.md §4b)."""
import numpy as np

from test_gpu_light_changes import opaque_for_light

FACES = ((-1, 0, 0), (0, -1, 0), (0, 0, -1), (1, 0, 0), (0, 1, 0), (0, 0, 1))   # Face6 order: NX NY NZ PX PY PZ
NEWLY_VISIBLE = 250
OPAQUE_TEXEL = (0, 0, 0, 128)


def kinds(space):
    """Block indices of the table by kind: air, opaque for light, glass (transparent, not emitting), lamp (emitting)."""
    blocks = space.blocks
    out = {"air": [0], "opaque": [], "glass": [], "lamp": []}
    for i, b in enumerate(blocks[1:], start=1):
        if opaque_for_light(b):
            out["opaque"].append(i)
        elif any(v != 0.0 for v in b.light_emission):
            out["lamp"].append(i)
        elif b.light_opaque_faces == 0:
            out["glass"].append(i)
    assert all(out.values()), out
    return out


def edit_list(space, seed, n_random=48):
    """A list of (cube, id) entries in segments, the segments in a seeded order: random entries over a small pool of
    cubes (heavy duplication, ids from the whole table), A -> B -> A and B -> A -> B chains between a cube's own block
    and one of another kind, a cube with its three upper neighbours, the corners of the bounds, and one entry of each
    kind (air, opaque, glass, lamp).  Returns (cubes int32 (n, 3), ids uint16 (n,))."""
    rng = np.random.default_rng(seed)
    lo, size = np.array(space.lower), np.array(space.size)
    k = kinds(space)

    def cube():
        return lo + rng.integers(0, size)

    def pick(kind):
        return int(rng.choice(k[kind]))

    def holds(c):
        return int(space.block_ids[tuple(np.asarray(c) - lo)])

    pool = [cube() for _ in range(12)]
    segments = [[(pool[rng.integers(len(pool))], int(rng.integers(len(space.blocks)))) for _ in range(n_random)]]
    for _ in range(3):
        c = cube()
        a = holds(c)
        b = pick("air" if opaque_for_light(space.blocks[a]) else "opaque")
        segments.append([(c, b), (c, a)])             # A -> B -> A
        c = cube()
        a = holds(c)
        b = pick(["opaque", "glass", "lamp", "air"][int(rng.integers(4))])
        segments.append([(c, b), (c, a), (c, b)])     # B -> A -> B (a no-op list when b == a)
    c = lo + rng.integers(0, size - 1)
    segments.append([(c + d, int(rng.integers(len(space.blocks)))) for d in ((0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1))])
    corners = [lo + np.array([x, y, z]) * (size - 1) for x in (0, 1) for y in (0, 1) for z in (0, 1)]
    segments.append([(c, int(rng.integers(len(space.blocks)))) for c in corners])
    segments.append([(cube(), pick(kind)) for kind in ("air", "opaque", "glass", "lamp")])
    entries = [e for s in (segments[i] for i in rng.permutation(len(segments))) for e in s]
    cubes = np.array([c for c, _ in entries], dtype=np.int32).reshape(-1, 3)
    return cubes, np.array([i for _, i in entries], dtype=np.uint16)


def edit_cubes_rule(space, queue, field, cubes, ids):
    """The list applied as aicb_light_edit_cubes applies it, to a copy of the queue (uint8, the volume's shape) and the
    field (uint8, shape + (4,)) of a Space holding space.block_ids.  Returns (number of changing entries, final block
    ids, queue, field, sorted linear indices of the cubes entering the set of changed cubes)."""
    shape, lo = tuple(space.size), np.array(space.lower)
    cur = space.block_ids.copy()
    changing = []
    for c, i in zip(cubes, ids):
        at = tuple(np.asarray(c) - lo)
        if cur[at] == i:
            continue   # Mutation::set of the same block changes nothing
        cur[at] = i
        changing.append((at, int(i)))
    queue, field, changed = queue.copy(), field.copy(), set()
    for at, i in changing:   # every changing entry whose own block is opaque for light
        if opaque_for_light(space.blocks[i]):
            field[at] = OPAQUE_TEXEL
            changed.add(int(np.ravel_multi_index(at, shape)))
    for at, _ in changing:   # modified_cube against the final cells
        block = space.blocks[cur[at]]
        if opaque_for_light(block):
            field[at] = OPAQUE_TEXEL
            changed.add(int(np.ravel_multi_index(at, shape)))
            queue[at] = 0
        else:
            queue[at] = NEWLY_VISIBLE
        for f, d in enumerate(FACES):
            n = tuple(np.asarray(at) + d)
            if not all(0 <= n[a] < shape[a] for a in range(3)):
                continue
            opp = (f + 3) % 6   # the neighbour's own face toward the cube
            if not (space.blocks[cur[n]].light_opaque_faces >> opp) & 1:
                queue[n] = NEWLY_VISIBLE
    return len(changing), cur, queue, field, sorted(changed)
