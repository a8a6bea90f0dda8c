"""Bodies on the GPU (aicb_step_bodies, its _device and group forms) against the body oracle: bodies and
BodyStepDetails bit for bit (f64s by their bits), contact sets and counts, on one context and on groups [0], [0, 0]
and [0, 0, 0]; and collision bits leave every existing output as it was."""
import copy

import numpy as np
import pytest
import torch

import aicb200
import bodyorc
import cursororc
from aicb200 import Block, GraphicsOptions, Space, abi, scenes
from test_gpu_append_blocks import assert_same, every_output
from test_gpu_device_blocks import on_device
from test_gpu_light_changes import TARGET_IDS, TARGETS, Lit

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
GRAVITY = (0.0, -20.0, 0.0)
OPTS = GraphicsOptions(view_distance=60.0, lighting_display=aicb200.LIGHT_LINEAR)


@pytest.fixture(params=TARGETS, ids=TARGET_IDS)
def target(request):
    return request.param


def with_collision(space, seed, p_block=0.25, p_voxel=0.4):
    """The Space with a random share of its single voxels and palette entries without collision."""
    rng = np.random.default_rng(seed)
    blocks = []
    for b in space.blocks:
        c = copy.copy(b)
        c.palette = np.array(b.palette, dtype=np.float32, copy=True)
        col = c.palette.view(np.uint32)[:, 7]
        p = p_block if b.indices is None else p_voxel
        col[:] = (col & ~np.uint32(abi.VOXEL_NO_COLLISION)) | np.where(
            rng.random(col.shape[0]) < p, abi.VOXEL_NO_COLLISION, 0).astype(np.uint32)
        blocks.append(c)
    return Space(space.lower, space.block_ids, blocks, light=space.light, sky_colors=space.sky_colors,
                 light_max_distance=space.light_max_distance)


def voxel_space(seed=5, n=12):
    """Voxel blocks of resolution 2 to 16 with partial bounds and wide palettes, among single blocks."""
    blocks = [Block.air(), Block(color=(0.8, 0.2, 0.1, 1.0)), Block(color=(0.0, 0.0, 0.0, 0.0)),
              Block(color=(0.2, 0.5, 0.9, 0.5))]
    for k, res in enumerate((2, 4, 8, 16, 4, 8)):
        blocks.append(scenes.make_voxel_block(seed + k, resolution=res, palette_size=(16, 300)[k % 2],
                                              partial_bounds=bool(k % 3)))
    h = scenes.grid_hash(seed, (n, n, n))
    ids = np.where((h & np.uint64(3)) != 0, (h >> np.uint64(8)) % np.uint64(len(blocks)), 0).astype(np.uint16)
    ids[:, n - 3:, :] = 0   # open space above
    return Space((-4, 0, 3), ids, blocks)


def random_bodies(space, n, seed):
    rng = np.random.default_rng(seed)
    lo = np.array(space.lower, dtype=np.float64)
    size = np.array(space.size, dtype=np.float64)
    pos = lo - 2.0 + rng.random((n, 3)) * (size + 4.0)   # some outside the bounds
    half = np.where(rng.random((n, 1)) < 0.15, rng.uniform(3.0, 3.6, (n, 3)), rng.uniform(0.2, 0.9, (n, 3)))
    half[:, 1] *= np.where(rng.random(n) < 0.5, 2.0, 1.0)
    box = np.concatenate([-half, half * rng.uniform(0.8, 1.0, (n, 3))], axis=1)
    vel = rng.normal(0.0, 6.0, (n, 3))
    vel[rng.random(n) < 0.1] = 0.0
    b = aicb200.bodies(n, position=pos, collision_box=box, velocity=vel, flying=rng.random(n) < 0.2,
                       noclip=rng.random(n) < 0.05)
    crushed = rng.random(n) < 0.2   # occupying shrunk around the position
    for i in np.nonzero(crushed)[0]:
        f = rng.uniform(0.3, 1.0, 6)
        b["occupying"][i, :3] = pos[i] + box[i, :3] * f[:3]
        b["occupying"][i, 3:] = pos[i] + box[i, 3:] * f[3:]
    return b


def check(got, want, what):
    assert want is not None, f"{what}: the oracle rejected the bodies"
    gb, gi, gc = got
    wb, wi, wc = want
    assert bodyorc.same_bits(gb, wb), f"{what}: bodies differ at {np.nonzero(gb.view(np.uint8).reshape(len(gb), -1) != wb.view(np.uint8).reshape(len(wb), -1))[0][:5]}"
    assert np.array_equal(gi["n_contacts"], wi["n_contacts"]), what
    assert bodyorc.same_bits(gi, wi), f"{what}: step info differs"
    m = gc.shape[1]
    for k in range(len(gb)):
        n = min(int(wi["n_contacts"][k]), m)
        assert sorted(map(bodyorc.contact_tuple, gc[k, :n])) == sorted(map(bodyorc.contact_tuple, wc[k, :n])), what


def host_view(t, dtype, shape):
    return t.cpu().numpy().view(dtype).reshape(shape)


def test_random_batches_match_the_oracle(target):
    space = with_collision(voxel_space(), seed=3)
    orc = bodyorc.BodyScene(space)
    lit = Lit(target, space)
    b = random_bodies(space, 1500, seed=1)
    edv = np.random.default_rng(2).normal(0.0, 1.0, (len(b), 3))
    stats = np.zeros(4)
    for tick in range(6):
        mc = 1 if tick % 3 == 2 else 8   # one contact stored: the rest are counted by re-casting earlier segments
        want = orc.step_bodies(b, 0.05, GRAVITY, edv if tick % 2 else None, max_contacts=mc)
        got = lit.scene.step_bodies(b, 0.05, GRAVITY, edv if tick % 2 else None, max_contacts=mc)
        check(got, want, f"tick {tick}")
        wi = want[1]
        ms = wi["move_segments"]
        recast = (wi["status"] & abi.BODY_CONTACTS_TRUNCATED != 0) & (ms["stopped_by"]["kind"][:, 0] != 0) & (
            np.any(ms["delta_position"][:, 1] != 0.0, axis=1) | (ms["stopped_by"]["kind"][:, 1] != 0))
        stats += [(ms["stopped_by"]["kind"] == abi.CONTACT_VOXEL).sum(), wi["has_push_out"].sum(),
                  (wi["uncrush"] == abi.UNCRUSH_PARTIAL).sum(), recast.sum()]
        b = want[0]
    # voxel stops, push-outs, partial uncrushes, and truncated sets of bodies with a second segment
    assert (stats > 0).all(), stats
    lit.close()


def used_agree(space, used_collide):
    """The Space with each recursive block's used palette entries colliding as `used_collide` and its unused entries
    the other way: the palette disagrees, the entries in use agree."""
    blocks = []
    for b in space.blocks:
        c = copy.copy(b)
        if b.indices is not None:
            c.palette = np.array(b.palette, dtype=np.float32, copy=True)
            used = np.zeros(c.palette.shape[0], dtype=bool)
            used[np.unique(b.indices)] = True
            assert not used.all(), "a block without unused entries"
            none = ~used if used_collide else used
            col = c.palette.view(np.uint32)[:, 7]
            col[:] = (col & ~np.uint32(abi.VOXEL_NO_COLLISION)) | np.where(none, abi.VOXEL_NO_COLLISION, 0).astype(
                np.uint32)
        blocks.append(c)
    return Space(space.lower, space.block_ids, blocks)


def unused_space(seed):
    """voxel_space's layout with recursive blocks whose palettes have unused entries."""
    s = voxel_space(seed=seed)
    for k, res in enumerate((2, 4, 8, 4, 2, 8)):
        s.blocks[4 + k] = scenes.make_voxel_block(seed + k, resolution=res, palette_size=(600, 300)[k % 2],
                                                  partial_bounds=bool(k % 3))
    return s


@pytest.mark.parametrize("palette", ["hard", "none", "used_hard", "used_none"])
def test_uniform_palettes_with_partial_bounds(target, palette):
    """Blocks whose palettes agree, or whose palettes disagree while the entries in use agree, with and without the
    implicit air of smaller voxel bounds, placed from host arrays and from device memory (update_blocks with
    DeviceBlocks): the same bits as the oracle's derivation."""
    if palette.startswith("used"):
        space = used_agree(unused_space(seed=11), used_collide=palette == "used_hard")
    else:
        p_voxel = 0.0 if palette == "hard" else 1.0
        space = with_collision(voxel_space(seed=11), seed=5, p_block=p_voxel, p_voxel=p_voxel)
    lit = Lit(target, space)
    b = random_bodies(space, 800, seed=6)
    want = bodyorc.BodyScene(space).step_bodies(b, 0.05, GRAVITY, max_contacts=8)
    check(lit.scene.step_bodies(b, 0.05, GRAVITY, max_contacts=8), want, "host placement")
    ids = np.arange(4, len(space.blocks), dtype=np.uint16)
    lit.scene.update_blocks(ids, [on_device(space.blocks[i]) for i in ids])
    torch.cuda.synchronize()
    check(lit.scene.step_bodies(b, 0.05, GRAVITY, max_contacts=8), want, "device placement")
    lit.close()


def test_device_form_on_a_side_stream(target):
    space = with_collision(voxel_space(seed=7), seed=4)
    orc = bodyorc.BodyScene(space)
    lit = Lit(target, space)
    b = random_bodies(space, 700, seed=5)
    want = orc.step_bodies(b, 0.1, GRAVITY, max_contacts=4)
    side = torch.cuda.Stream(DEV)
    base = torch.from_numpy(b.view(np.uint8).reshape(len(b), -1).copy()).to(DEV)
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)                 # the bodies are written late on the stream the call is issued on
        db = base + 0
        db, info, contacts = lit.scene.step_bodies(db, 0.1, GRAVITY, max_contacts=4, device=True)
        out = (db.clone(), info.clone(), contacts.clone())
    side.synchronize()
    got = (host_view(out[0], abi.BODY_DTYPE, (-1,)), host_view(out[1], abi.BODY_STEP_INFO_DTYPE, (-1,)),
           host_view(out[2], abi.CONTACT_DTYPE, (len(b), 4)))
    check(got, want, "device form")
    lit.close()


def test_after_changes(target):
    """After a device cube update and a block redefinition, without a rebuild of the id mirror."""
    space = with_collision(voxel_space(seed=9), seed=6)
    lit = Lit(target, space)
    s = lit.scene
    b = random_bodies(space, 500, seed=8)
    cubes = np.array([[x, y, z] for x in range(-4, 4) for y in range(0, 3) for z in range(3, 8)], dtype=np.int32)
    ids = np.full(len(cubes), 4, dtype=np.uint16)
    s.update_cubes(cubes, ids)
    space.block_ids[cubes[:, 0] + 4, cubes[:, 1], cubes[:, 2] - 3] = 4
    nb = scenes.make_voxel_block(77, resolution=8, palette_size=12)
    nb = with_collision(Space((0, 0, 0), np.zeros((1, 1, 1), np.uint16), [nb]), seed=11).blocks[0]
    s.update_blocks(np.array([5], np.uint16), [nb])
    space.blocks[5] = nb
    want = bodyorc.BodyScene(space).step_bodies(b, 0.05, GRAVITY, max_contacts=8)
    check(s.step_bodies(b, 0.05, GRAVITY, max_contacts=8), want, "after changes")
    lit.close()


def test_rejections(target):
    space = voxel_space()
    lit = Lit(target, space)
    good = aicb200.bodies(4, position=(0.0, 20.0, 5.0))
    dgood = torch.from_numpy(good.view(np.uint8).reshape(4, -1).copy()).to(DEV)
    for device, bodies in ((False, good), (True, dgood)):
        for bad_dt in (0.0, -1.0, 1.5, float("nan"), float("inf")):
            with pytest.raises(aicb200.AicbError) as e:
                lit.scene.step_bodies(bodies, bad_dt, GRAVITY, device=device)
            assert e.value.status == abi.ERR_INVALID and "dt" in str(e.value)
        for bad_g in ((0.0, float("inf"), 0.0), (float("nan"), 0.0, 0.0)):
            with pytest.raises(aicb200.AicbError) as e:
                lit.scene.step_bodies(bodies, 0.1, bad_g, device=device)
            assert e.value.status == abi.ERR_INVALID and "gravity" in str(e.value)
    torch.cuda.synchronize()
    assert bodyorc.same_bits(host_view(dgood, abi.BODY_DTYPE, (-1,)), good)   # a rejected call writes nothing
    bad = good.copy()
    bad["position"][2, 0] = float("nan")
    with pytest.raises(aicb200.AicbError):
        lit.scene.step_bodies(bad, 0.1, GRAVITY)
    dbad = torch.from_numpy(bad.view(np.uint8).reshape(4, -1).copy()).to(DEV)
    db, info, _ = lit.scene.step_bodies(dbad, 0.1, GRAVITY, device=True)
    torch.cuda.synchronize()
    info = host_view(info, abi.BODY_STEP_INFO_DTYPE, (-1,))
    assert info["status"].tolist() == [0, 0, abi.BODY_INVALID, 0]
    assert bodyorc.same_bits(host_view(db, abi.BODY_DTYPE, (-1,))[2], bad[2])
    lit.close()


@pytest.mark.parametrize("set_bits", [False, True])
def test_collision_bits_change_no_other_output(set_bits):
    """A frame, the cursor and light are the same with collision bits set as with them clear."""
    space = scenes.config_c1(n=16, seed=2, n_voxel_blocks=4, with_light=True)
    flagged = with_collision(space, seed=1, p_block=0.5 if set_bits else 0.0, p_voxel=0.5 if set_bits else 0.0)
    cam = aicb200.Camera(OPTS, aicb200.Viewport.with_scale(1.0, (64, 48)))
    cam.look_at_y_up((20.0, 22.0, 24.0), (8.0, 8.0, 8.0))
    ref, new = aicb200.SpaceRaytracer(space, OPTS), aicb200.SpaceRaytracer(flagged, OPTS)
    assert_same(every_output(new, OPTS, cam), every_output(ref, OPTS, cam), "collision bits")
    rays = np.random.default_rng(3).normal(0.0, 1.0, (500, 6)) + np.array([8, 8, 8, 0, 0, 0])
    assert cursororc.same_bits(new.cursor_raycast(rays), ref.cursor_raycast(rays))
    assert np.array_equal(new.light_download(), ref.light_download())
