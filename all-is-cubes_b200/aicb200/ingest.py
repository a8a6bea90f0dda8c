"""Scene ingestion from the reference's native save format (SURVEY §8(f) N3): `.alliscubesjson` universes and
`SpaceV1` values (all-is-cubes/src/save/schema.rs:467-498) -> `aicb200.Space`, without Rust.

What is read:
  * `SpaceV1`: `bounds` {lower, upper}; `physics.sky` (`UniformV1` / `OctantsV1`, schema.rs:508-513) and
    `physics.light` (`NoneV1` / `RaysV1{maximum_distance}`, :516-521); `contents` and `light` as `GzSerde`
    (save/compress.rs:20-130: `{"Base64Gzip": "<standard base64 without padding of a gzip stream>"}`; contents are
    little-endian u16 block indices in Z-major order, light is `LightSerV1` = r, g, b, status with the status byte
    0 Uninitialized / 1 NoRays / 2 Opaque / 3 Visible, schema.rs:486-498 — NOT the PackedLight texel's status byte);
  * `blocks`: `BlockV1` with the primitives `AirV1`, `AtomV1{color, light_emission, collision}` and `RecurV1{space, offset,
    resolution}` (schema.rs:84-98) whose voxel Space consists of `AirV1` / `AtomV1` blocks — the cases whose evaluation
    is a table lookup (block/eval: an atom's Evoxel is its colour and emission; a Recur block's Evoxels are its
    Space's blocks over `offset .. offset + resolution`, clipped to the Space's bounds).
  * `SelectableV1{selectable}` sets the block's BlockAttributes::selectable (attributes.rs:389), and through
    Evoxel::from_block (voxel_storage.rs:76-100) the selectable of each voxel a `RecurV1` block takes from it; an
    `AirV1` block, and so an `AirV1` voxel, is never selectable (AIR_ATTRIBUTES);
  * `AtomV1.collision` (`HardV1`, the default, or `NoneV1`; schema.rs:86-114) is the atom's voxel's collision, and a
    `RecurV1` voxel takes its block's uniform collision (Evoxel::from_block: `uniform_collision().unwrap_or(Hard)`);
    an `AirV1` block and an empty `RecurV1` region collide as BlockCollision::None;
  * modifiers that do not change what is drawn or picked (`DisplayNameV1`, `TagV1`, `QuoteV1`, inventory / action
    attributes) are ignored; `RotateV1`, `CompositeV1`, `ZoomV1`, `Move`, `IndirectV1` and `TextPrimitiveV1` need the
    reference's block evaluator (out of scope, SURVEY §2) and raise `UnsupportedBlock`.
  * universes: `UniverseV1{members: [{name, member_type, value}]}` (schema.rs:548-600).

The harness of the reference exports its shared test scenes with `--dump-test-universes DIR`
(test-renderers/runner/src/harness.rs:71-76,177-189): one run on a machine with Rust gives loadable golden scenes.
"""
from __future__ import annotations

import base64
import gzip
import json

import numpy as np

from . import Block, Space

# LightStatusSerV1 (schema.rs:491-498) -> the status byte of PackedLight::as_texel (light/data.rs:31-46, 162)
_STATUS_TEXEL = {0: 0, 1: 1, 2: 128, 3: 255}
_TEXEL_STATUS = {t: s for s, t in _STATUS_TEXEL.items()}
_IGNORED_MODIFIERS = {"DisplayNameV1", "TagV1", "QuoteV1", "BlockInventoryV1", "InventoryConfigV1",
                      "RotationRuleV1", "PlacementActionV1", "TickActionV1", "ActivationActionV1", "AnimationHintV1"}


class UnsupportedBlock(ValueError):
    pass


def gz_decode(value) -> bytes:
    """GzSerde (save/compress.rs): {"Base64Gzip": str} in human-readable formats, {"Gzip": [bytes]} otherwise."""
    if isinstance(value, dict) and "Base64Gzip" in value:
        s = value["Base64Gzip"]
        return gzip.decompress(base64.b64decode(s + "=" * (-len(s) % 4)))
    if isinstance(value, dict) and "Gzip" in value:
        return gzip.decompress(bytes(value["Gzip"]))
    raise ValueError("not a GzSerde value")


def gz_encode(data: bytes):
    """The human-readable GzSerde form (for tests and for writing scenes back)."""
    return {"Base64Gzip": base64.b64encode(gzip.compress(data, compresslevel=1)).decode("ascii").rstrip("=")}


def name_key(name) -> str:
    """universe::Name as serialized (schema.rs:601-605): {"Specific": s} | {"Anonym": n} | {"Builtin": ..}."""
    return json.dumps(name, sort_keys=True)


def _atom(prim):
    c = [float(v) for v in prim["color"]]
    e = [float(v) for v in prim.get("light_emission", (0.0, 0.0, 0.0))]
    coll = prim.get("collision", "HardV1")
    if isinstance(coll, dict):
        coll = coll.get("type")
    if coll not in ("HardV1", "NoneV1"):
        raise UnsupportedBlock(f"collision {coll!r}")
    return c, e, coll == "HardV1"


def _collides(block):
    """Evoxel::from_block's collision for a voxel Space's block: an air block's is None, an atom's its own."""
    if block.is_air:
        return False
    mask = block.voxel_no_collision
    return mask is None or not bool(mask[0])


def _block_of(block_ser, resolve_space):
    if block_ser.get("type") != "BlockV1":
        raise UnsupportedBlock(f"block type {block_ser.get('type')}")
    selectable = True
    for m in block_ser.get("modifiers", []):
        if m.get("type") == "SelectableV1":
            selectable = bool(m["selectable"])
        elif m.get("type") not in _IGNORED_MODIFIERS:
            raise UnsupportedBlock(f"modifier {m.get('type')} needs the reference's block evaluator")
    prim = block_ser["primitive"]
    kind = prim["type"]
    if kind == "AirV1":
        return Block.air()
    if kind == "AtomV1":
        c, e, hard = _atom(prim)
        return Block(color=tuple(c), emission=tuple(e), selectable=selectable, collision=hard)
    if kind == "RecurV1":
        if resolve_space is None:
            raise UnsupportedBlock("RecurV1 needs the universe the Space handle points into")
        res = int(prim["resolution"])
        off = [int(v) for v in prim.get("offset", (0, 0, 0))]
        vs = resolve_space(prim["space"])
        # Evoxels of a Recur block: the voxel Space's cubes offset .. offset + resolution, clipped to its bounds
        lo = [max(off[a], vs.lower[a]) for a in range(3)]
        hi = [min(off[a] + res, vs.lower[a] + vs.size[a]) for a in range(3)]
        if any(hi[a] <= lo[a] for a in range(3)):
            return Block(color=(0.0, 0.0, 0.0, 0.0), selectable=selectable, collision=False)
        sl = tuple(slice(lo[a] - vs.lower[a], hi[a] - vs.lower[a]) for a in range(3))
        ids = vs.block_ids[sl]
        pal = np.zeros((len(vs.blocks), 8), dtype=np.float32)
        for i, b in enumerate(vs.blocks):
            if b.indices is not None:
                raise UnsupportedBlock("a voxel Space made of recursive blocks needs the reference's block evaluator")
            pal[i] = b.palette[0]
        return Block(resolution=res, voxel_lower=[lo[a] - off[a] for a in range(3)], indices=ids.astype(np.uint16),
                     palette=pal, selectable=selectable, voxel_selectable=[b.selectable for b in vs.blocks],
                     voxel_collision=[_collides(b) for b in vs.blocks])
    raise UnsupportedBlock(f"primitive {kind} needs the reference's block evaluator")


def light_from_value(value, size) -> np.ndarray:
    """A `GzSerde` `LightSerV1` volume -> PackedLight texels shaped `size + (4,)`."""
    raw = np.frombuffer(gz_decode(value), dtype=np.uint8).reshape(-1, 4)
    if raw.shape[0] != size[0] * size[1] * size[2]:
        raise ValueError("light volume size mismatch")
    light = raw.copy()
    light[:, 3] = np.vectorize(_STATUS_TEXEL.__getitem__, otypes=[np.uint8])(raw[:, 3])
    return light.reshape(tuple(size) + (4,))


def light_to_value(texels, queue=None):
    """PackedLight texels (and the light update queue: one priority per cube, 0 = not queued, as
    light_download_queue returns it) -> the `GzSerde` `LightSerV1` value of a `SpaceV1`, the inverse of what
    space_from_value reads.  As Serialize for space::Read writes it (save/conversion.rs:773-785), a queued cube's status
    is Uninitialized and its r, g, b are kept, so a Space loaded from it resumes the queued work
    (SpaceRaytracer.light_queue_uninitialized)."""
    t = np.ascontiguousarray(texels, dtype=np.uint8).reshape(-1, 4)
    status = t[:, 3]
    known = np.isin(status, list(_TEXEL_STATUS))
    if not known.all():
        raise ValueError(f"texel status byte {int(status[~known][0])} has no LightStatusSerV1")
    out = t.copy()
    lut = np.zeros(256, dtype=np.uint8)
    lut[list(_TEXEL_STATUS)] = list(_TEXEL_STATUS.values())
    out[:, 3] = lut[status]
    if queue is not None:
        q = np.asarray(queue, dtype=np.uint8).reshape(-1)
        if q.size != t.shape[0]:
            raise ValueError("queue size mismatch")
        out[q > 0, 3] = 0
    return gz_encode(out.tobytes())


def space_from_value(v, resolve_space=None, ctx=None) -> Space:
    """A `SpaceV1` value (the parsed JSON object) -> Space.  With a Context `ctx`, the light data of its recursive
    blocks is compute_derived's, computed on that context's device (Context.derive_block_light), instead of the
    numpy restatement Block computes."""
    if v.get("type") != "SpaceV1":
        raise ValueError(f"not a SpaceV1 value: {v.get('type')}")
    lower = [int(c) for c in v["bounds"]["lower"]]
    upper = [int(c) for c in v["bounds"]["upper"]]
    size = tuple(upper[a] - lower[a] for a in range(3))
    n = size[0] * size[1] * size[2]
    ids = np.frombuffer(gz_decode(v["contents"]), dtype="<u2")
    if ids.size != n:
        raise ValueError(f"contents hold {ids.size} block indices, the bounds {n} cubes")
    blocks = [_block_of(b, resolve_space) for b in v["blocks"]]
    if ids.size and int(ids.max()) >= len(blocks):
        raise ValueError("block index out of range")   # (save/tests.rs:749-785 space_de_invalid_index)
    if ctx is not None:
        recursive = [b for b in blocks if b.indices is not None]
        for b, bl in zip(recursive, ctx.derive_block_light(recursive)):
            b.set_light_data(bl)
    physics = v["physics"]
    sky = physics["sky"]
    if sky["type"] == "UniformV1":
        sky_colors = [tuple(float(c) for c in sky["color"])]
    elif sky["type"] == "OctantsV1":
        sky_colors = [tuple(float(c) for c in col) for col in sky["colors"]]
    else:
        raise ValueError(f"sky {sky['type']}")
    lp = physics["light"]
    max_distance = int(lp["maximum_distance"]) if lp["type"] == "RaysV1" else 0
    light = None
    if v.get("light") is not None and max_distance:
        light = light_from_value(v["light"], size)
    return Space(tuple(lower), ids.astype(np.uint16).reshape(size), blocks, light=light, sky_colors=sky_colors,
                 light_max_distance=max_distance)


def spaces_from_universe(u, ctx=None) -> dict:
    """A `UniverseV1` value -> {name key: Space} for every Space member that can be ingested (voxel Spaces first);
    `ctx` as space_from_value takes it."""
    if u.get("type") != "UniverseV1":
        raise ValueError(f"not a UniverseV1 value: {u.get('type')}")
    raw = {name_key(m["name"]): m["value"] for m in u["members"] if m.get("member_type") == "Space"}
    done, in_progress = {}, set()

    def resolve(handle):
        key = name_key({k: v for k, v in handle.items() if k != "type"})
        if key in done:
            return done[key]
        if key in in_progress or key not in raw:
            raise UnsupportedBlock(f"Space {key} is missing or refers to itself")
        in_progress.add(key)
        done[key] = space_from_value(raw[key], resolve, ctx)
        in_progress.discard(key)
        return done[key]

    out = {}
    for key in raw:
        try:
            out[key] = resolve({"type": "HandleV1", **json.loads(key)})
        except UnsupportedBlock:
            continue
    return out


def load_universe(path, ctx=None) -> dict:
    with open(path, "rb") as f:
        data = f.read()
    if data[:2] == b"\x1f\x8b":
        data = gzip.decompress(data)
    return spaces_from_universe(json.loads(data), ctx)
