"""The body oracle (oracle_body/) against the reference's known answers: physics/tests.rs, step.rs:986-1087 and
collision.rs:554-723, and the derived uniform collision of block/eval/derived.rs.  CPU only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import aicb200
from aicb200 import abi
import bodyorc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRAVITY = (0.0, -20.0, 0.0)   # SpacePhysics::DEFAULT (space/physics.rs:43)
POSITION_EPSILON = 1e-6 * 1e-6
AIR = aicb200.Block(is_air=True)
STONE = aicb200.Block(color=(0.5, 0.5, 0.5, 1.0))


def slab(thickness, res):
    """make_slab: the lower `thickness` voxel layers solid (Hard), the rest air (None)."""
    idx = np.zeros((res, res, res), dtype=np.uint16)
    idx[:, thickness:, :] = 1
    pal = np.zeros((2, 8), dtype=np.float32)
    pal[0, :4] = (0.5, 0.5, 0.5, 1.0)
    return aicb200.Block(resolution=res, indices=idx, palette=pal, voxel_collision=[True, False])


def scene(lower, ids, blocks):
    return bodyorc.BodyScene(aicb200.Space(lower, np.asarray(ids, dtype=np.uint16), blocks))


def test_body_struct_layouts_match_c_header(tmp_path):
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "aicb200.h"\nint main(){printf("%zu %zu %zu %zu %zu '
                   '%zu %zu %zu\\n",sizeof(aicb_body),sizeof(aicb_contact),sizeof(aicb_move_segment),'
                   'sizeof(aicb_body_step_info),offsetof(aicb_body,flying),offsetof(aicb_body_step_info,n_contacts),'
                   'offsetof(aicb_body_step_info,uncrush_axes),offsetof(aicb_contact,kind));return 0;}\n')
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [abi.BODY_DTYPE.itemsize, abi.CONTACT_DTYPE.itemsize, abi.MOVE_SEGMENT_DTYPE.itemsize,
            abi.BODY_STEP_INFO_DTYPE.itemsize, abi.BODY_DTYPE.fields["flying"][1],
            abi.BODY_STEP_INFO_DTYPE.fields["n_contacts"][1], abi.BODY_STEP_INFO_DTYPE.fields["uncrush_axes"][1],
            abi.CONTACT_DTYPE.fields["kind"][1]]
    assert got == want


@pytest.mark.parametrize("gravity", [False, True])
def test_freefall(gravity):
    s = scene((0, 0, 0), np.zeros((1, 1, 1)), [AIR])
    b = aicb200.bodies(1, position=(0.0, 2.0, 0.0), velocity=(2.0, 0.0, 0.0), flying=not gravity)
    b, _, _ = s.step_bodies(b, 0.25, GRAVITY)
    p1 = b["position"][0].copy()
    b, _, _ = s.step_bodies(b, 0.25, GRAVITY)
    assert p1.tolist() == [0.5, 0.75 if gravity else 2.0, 0.0]
    assert b["position"][0].tolist() == [1.0, -1.75 if gravity else 2.0, 0.0]


def test_falling_collision():
    s = scene((0, 0, 0), np.ones((1, 1, 1)), [AIR, STONE])
    b = aicb200.bodies(1, position=(0.0, 2.0, 0.0), velocity=(2.0, 0.0, 0.0))
    b, info, contacts = s.step_bodies(b, 1.0, GRAVITY)
    p = b["position"][0]
    assert p[0] == 2.0 and p[2] == 0.0 and abs(p[1] - 1.5) < 1e-6
    assert info["n_contacts"][0] == 1
    assert bodyorc.contact_tuple(contacts[0, 0]) == (abi.CONTACT_BLOCK, (0, 0, 0), 5, 0, (0, 0, 0))


def test_falling_collision_partial_block():
    s = scene((0, 0, 0), np.ones((1, 1, 1)), [AIR, slab(2, 4)])
    b = aicb200.bodies(1, position=(0.0, 2.0, 0.0), velocity=(0.2, 0.0, 0.0))
    b, info, contacts = s.step_bodies(b, 1.0, GRAVITY)
    p = b["position"][0]
    assert p[0] == 0.2 and p[2] == 0.0 and abs(p[1] - 1.0) < 1e-6
    assert info["n_contacts"][0] == 1
    c = contacts[0, 0]
    assert (c["kind"], tuple(c["cube"]), c["resolution"], c["face"]) == (abi.CONTACT_VOXEL, (0, 0, 0), 4, 5)
    b["velocity"][0, 0] = 0.0
    for _ in range(1000):
        b, _, _ = s.step_bodies(b, 1.0, GRAVITY)
        assert abs(b["position"][0, 1] - 1.0) < 1e-6


def test_push_out_simple():
    s = scene((0, 0, 0), np.ones((1, 1, 1)), [AIR, STONE])
    b = aicb200.bodies(1, position=(1.25, 0.5, 0.5), flying=True)
    b, info, _ = s.step_bodies(b, 1.0, GRAVITY)
    assert b["position"][0].tolist() == [1.5 + POSITION_EPSILON, 0.5, 0.5]
    assert b["velocity"][0].tolist() == [0.0, 0.0, 0.0]
    assert info["has_push_out"][0] == 1


def test_velocity_limit():
    s = scene((0, 0, 0), np.zeros((1, 1, 1)), [AIR])
    b = aicb200.bodies(1, velocity=(1e7, 0.0, 0.0), flying=True)
    b, _, _ = s.step_bodies(b, 0.5, GRAVITY)
    assert b["velocity"][0].tolist() == [1e4, 0.0, 0.0]
    assert b["position"][0].tolist() == [0.5 * 1e4, 0.0, 0.0]


def _walled_room():
    ids = np.ones((3, 3, 3))
    ids[1, 1, 1] = 0
    return scene((-1, -1, -1), ids, [AIR, STONE])


def _no_passing(s, velocity):
    start = np.array([0.5, 0.5, 0.5])
    b = aicb200.bodies(1, position=start, collision_box=(-0.375,) * 3 + (0.375,) * 3, flying=True)
    history = []
    for _ in range(5000):
        b["velocity"][0] = velocity
        history.insert(0, tuple(b["position"][0]))
        b, _, _ = s.step_bodies(b, 1.0 / 60.0, GRAVITY)
        p = b["position"][0]
        assert np.max(np.abs(p - start)) < 0.5, p
        if tuple(p) in history:
            break
        del history[10:]
    else:
        return
    assert np.max(np.abs(b["position"][0] - start)) > 0.09


@pytest.mark.parametrize("case", [(1.0, 1.0, 1.0), (1.0, 0.1, 0.1), (0.1, -0.1, -0.047)])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_no_passing_through_blocks(case, sign):
    _no_passing(_walled_room(), np.array(case) * sign)


def test_no_passing_through_blocks_random():
    s = _walled_room()
    rng = np.random.default_rng(1)
    for _ in range(20):
        v = rng.uniform(0.04, 1.0, 3) * rng.choice([-1.0, 1.0], 3)
        if np.linalg.norm(v) < 0.05:
            continue
        _no_passing(s, v)


def test_crush():
    s = scene((0, 0, 0), np.ones((1, 1, 1)), [AIR, STONE])
    b = aicb200.bodies(1, position=(0.0, 1.25, 0.0))[0]
    assert b["occupying"].tolist() == [-0.5, 0.75, -0.5, 0.5, 1.75, 0.5]
    b, info, st = s.crush_if_colliding(b)
    assert st == 0
    assert b["occupying"].tolist() == [-0.5, 1.0, -0.5, 0.5, 1.75, 0.5]
    assert info.tolist() == [0.0, 0.25, 0.0, 0.0, 0.0, 0.0]   # the NY face moved in by 0.25


def test_uncrush_not_needed():
    s = scene((0, 0, 0), np.zeros((1, 1, 1)), [AIR])
    b = aicb200.bodies(1, position=(0.0, 1.25, 0.0))[0]
    after, r, _ = s.uncrush(b)
    assert r == abi.UNCRUSH_NOT_NEEDED and after["occupying"].tolist() == b["occupying"].tolist()


def test_uncrush_unobstructed():
    s = scene((0, 0, 0), np.zeros((1, 1, 1)), [AIR])
    b = aicb200.bodies(1, position=(0.0, 1.25, 0.0))[0]
    expected = [-0.5, 0.75, -0.5, 0.5, 1.75, 0.5]
    b["occupying"] = [-0.4, 0.85, -0.4, 0.4, 1.65, 0.4]
    after, r, _ = s.uncrush(b)
    assert r == abi.UNCRUSH_COMPLETE and after["occupying"].tolist() == expected


def test_uncrush_impossible_intersecting():
    s = scene((0, 0, 0), np.ones((1, 1, 1)), [AIR, STONE])
    b = aicb200.bodies(1, position=(0.5, 0.5, 0.5))[0]
    b["occupying"] = [0.25, 0.25, 0.25, 0.75, 0.75, 0.75]
    after, r, _ = s.uncrush(b)
    assert r == abi.UNCRUSH_NOT_POSSIBLE and after["occupying"].tolist() == [0.25, 0.25, 0.25, 0.75, 0.75, 0.75]


def test_uncrush_partial_success():
    s = scene((0, 0, 0), np.ones((1, 1, 1)), [AIR, STONE])
    b = aicb200.bodies(1, position=(0.5, 1.25, 0.5))[0]
    b["occupying"] = [0.25, 1.125, 0.25, 0.75, 1.75, 0.75]
    after, r, axes = s.uncrush(b)
    assert r == abi.UNCRUSH_PARTIAL and axes.tolist() == [2, 0, 1]   # Z, X, Y: the last maximum wins
    assert after["occupying"].tolist() == [0.0, 1.0, 0.0, 1.0, 1.75, 1.0]


def _tester(initial_y, blocks):
    s = scene((0, 0, 0), np.array([[[0]], [[1]]]), blocks)
    return s.collide_along_ray([0.5, initial_y, 0.0, 0.0, -2.0, 0.0], [0, 0, 0, 1, 1, 1])


def test_collide_along_ray_with_opaque_block():
    end, _ = _tester(1.5, [AIR, STONE])
    assert end[0] == 0.25 and bodyorc.contact_tuple(end[1]) == (abi.CONTACT_BLOCK, (1, 0, 0), 5, 0, (0, 0, 0))


@pytest.mark.parametrize("initial_y,t", [(1.5, 0.5), (0.75, 0.125)])
def test_collide_along_ray_recursive(initial_y, t):
    end, _ = _tester(initial_y, [AIR, slab(1, 2)])
    assert end[0] == t
    assert bodyorc.contact_tuple(end[1]) == (abi.CONTACT_VOXEL, (1, 0, 0), 5, 2, (0, 0, 0))


def test_collide_along_ray_two_recursive():
    end, _ = _tester(0.75, [slab(1, 4), slab(1, 2)])
    assert end[0] == 0.125 and bodyorc.contact_tuple(end[1]) == (abi.CONTACT_VOXEL, (1, 0, 0), 5, 2, (0, 0, 0))
    end, _ = _tester(0.75, [slab(1, 2), slab(1, 4)])
    assert end[0] == 0.125 and bodyorc.contact_tuple(end[1]) == (abi.CONTACT_VOXEL, (0, 0, 0), 5, 2, (1, 0, 0))


def test_already_colliding():
    s = scene((0, 0, 0), np.array([[[0]], [[1]]]), [STONE, slab(1, 2)])
    end, reported = s.collide_along_ray([0.5, 0.0, 0.5, 1.0, 0.0, 0.0], [-1, -1, -1, 2, 1, 1])
    assert end is None
    assert [bodyorc.contact_tuple(c) for c in reported] == [
        (abi.CONTACT_BLOCK, (0, 0, 0), 0, 0, (0, 0, 0)), (abi.CONTACT_VOXEL, (1, 0, 0), 0, 2, (0, 0, 0))]


def _rec(res, lower, size, palette_collision, used):
    """A recursive block whose palette entries have the given collisions and whose voxels use entries `used`."""
    idx = np.zeros(size, dtype=np.uint16)
    flat = idx.reshape(-1)
    flat[:len(used)] = used
    flat[len(used):] = used[-1]
    pal = np.zeros((len(palette_collision), 8), dtype=np.float32)
    pal[:, 3] = 1.0
    return aicb200.Block(resolution=res, voxel_lower=lower, indices=idx, palette=pal, voxel_collision=palette_collision)


def test_uniform_collision_rule():
    HARD, NONE, MIXED = 0, 1, 2
    assert bodyorc.uniform_collision(AIR) == NONE
    assert bodyorc.uniform_collision(STONE) == HARD
    assert bodyorc.uniform_collision(aicb200.Block(color=(1, 1, 1, 1), collision=False)) == NONE
    # a full block: the palette if it agrees, else the entries in use
    assert bodyorc.uniform_collision(_rec(2, (0, 0, 0), (2, 2, 2), [True, True], [0, 1])) == HARD
    assert bodyorc.uniform_collision(_rec(2, (0, 0, 0), (2, 2, 2), [False, False], [0, 1])) == NONE
    assert bodyorc.uniform_collision(_rec(2, (0, 0, 0), (2, 2, 2), [True, False], [0, 1])) == MIXED
    assert bodyorc.uniform_collision(_rec(2, (0, 0, 0), (2, 2, 2), [True, False], [0])) == HARD
    assert bodyorc.uniform_collision(_rec(2, (0, 0, 0), (2, 2, 2), [True, False], [1])) == NONE
    # voxel bounds smaller than the block: the air outside counts as None (block/eval/tests.rs:436's four)
    assert bodyorc.uniform_collision(_rec(2, (0, 0, 0), (2, 1, 2), [True], [0])) == MIXED
    assert bodyorc.uniform_collision(_rec(2, (0, 0, 0), (2, 1, 2), [False], [0])) == NONE
    assert bodyorc.uniform_collision(_rec(2, (0, 0, 0), (2, 1, 2), [True, False], [1])) == NONE
    assert bodyorc.uniform_collision(_rec(2, (0, 0, 0), (2, 1, 2), [True, False], [0])) == MIXED


def test_rejected_bodies():
    s = scene((0, 0, 0), np.zeros((1, 1, 1)), [AIR])
    good = aicb200.bodies(1)
    for field, k, v in [("position", 0, np.nan), ("velocity", 1, np.inf), ("collision_box", 0, 0.5),
                        ("occupying", 3, -0.6), ("occupying", 2, np.inf)]:
        b = good.copy()
        b[field][0, k] = v
        assert s.step_bodies(b, 0.1, GRAVITY) is None
    assert s.step_bodies(good, 0.1, GRAVITY, external_delta_v=[[np.nan, 0, 0]]) is None


def _space_v1(blocks, contents, upper):
    from aicb200 import ingest
    return {"type": "SpaceV1", "bounds": {"lower": [0, 0, 0], "upper": upper},
            "physics": {"gravity": [0, 0, 0], "sky": {"type": "UniformV1", "color": [0, 0, 0]},
                        "light": {"type": "NoneV1"}},
            "blocks": blocks, "contents": ingest.gz_encode(np.array(contents, dtype="<u2").tobytes()), "light": None}


def _ingested_world():
    from aicb200 import ingest
    air = {"type": "BlockV1", "primitive": {"type": "AirV1"}}

    def atom(collision=None):
        prim = {"type": "AtomV1", "color": [1.0, 0.0, 0.0, 1.0]}
        if collision is not None:
            prim["collision"] = collision
        return {"type": "BlockV1", "primitive": prim}

    def recur(name, offset=(0, 0, 0)):
        return {"type": "BlockV1", "primitive": {"type": "RecurV1", "space": {"type": "HandleV1", "Specific": name},
                                                 "offset": list(offset), "resolution": 2}}

    # a slab: the lower voxel layer is a Hard atom, the upper one AirV1 (Z-major contents of a 2x2x2 Space)
    slab_space = _space_v1([air, atom()], [1, 1, 0, 0, 1, 1, 0, 0], [2, 2, 2])
    # a block whose voxels are all NoneV1 atoms, and one that mixes HardV1 with NoneV1 atoms
    none_space = _space_v1([air, atom("NoneV1"), atom("HardV1")], [1] * 8, [2, 2, 2])
    mixed_space = _space_v1([air, atom("NoneV1"), atom("HardV1")], [1, 2] * 4, [2, 2, 2])
    world = _space_v1([air, recur("slab"), recur("none"), recur("mixed"), atom("NoneV1"), atom(),
                       recur("slab", offset=(10, 10, 10))], [1, 2, 3, 4, 5, 6], [6, 1, 1])
    u = {"type": "UniverseV1", "members": [
        {"name": {"Specific": n}, "member_type": "Space", "value": v}
        for n, v in (("slab", slab_space), ("none", none_space), ("mixed", mixed_space), ("world", world))]}
    return ingest.spaces_from_universe(u)[ingest.name_key({"Specific": "world"})]


def test_ingest_carries_collision():
    w = _ingested_world()
    HARD, NONE, MIXED = 0, 1, 2
    # AIR, the slab (Hard below AirV1), all-None voxels, None and Hard voxels, a NoneV1 atom, a HardV1 atom (the
    # default), an empty RecurV1 region
    assert [bodyorc.uniform_collision(b) for b in w.blocks] == [NONE, MIXED, NONE, MIXED, NONE, HARD, NONE]
    # AirV1 voxels are None; column 7 keeps the selectable flags only, the collision is added to the descriptor
    assert list(w.blocks[1].voxel_no_collision) == [True, False]
    assert list(w.blocks[1].palette.view(np.uint32)[:, 7]) == [abi.VOXEL_NOT_SELECTABLE, 0]
    assert list(w.blocks[1].desc_palette().view(np.uint32)[:, 7]) == [
        abi.VOXEL_NOT_SELECTABLE | abi.VOXEL_NO_COLLISION, 0]


def test_ingested_slab_collides_as_a_slab():
    w = _ingested_world()
    s = bodyorc.BodyScene(w)
    b = aicb200.bodies(1, position=(0.5, 2.0, 0.5))
    for _ in range(30):
        b, _, _ = s.step_bodies(b, 0.05, GRAVITY)
    assert abs(b["position"][0, 1] - 1.0) < 1e-6   # the box's bottom rests on the slab's top, y = 0.5
