"""The host calls' outputs at their edges, on one context and on a two-context group of one device: an output the
caller leaves NULL, shards that reassemble the frame, destinations in pageable, pinned and registered host memory, an
empty texture batch, and one output set drawn right after a larger call of another set on the same context."""
import ctypes as C

import numpy as np
import pytest

import aicb200
from aicb200 import DeviceGroup, GraphicsOptions, RtRenderer, abi, scenes

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W, H = 40, 33
N = W * H
NO_WORLD = (0.74, 0.74, 0.74, 1.0)
KINDS = ("pageable", "pinned", "registered")


@pytest.fixture(scope="module")
def setup():
    space = scenes.small_mixed_scene(n=12, seed=7)
    opts = GraphicsOptions(view_distance=40.0, exposure=1.5)
    cam = scenes.standard_camera(space, opts, W, H)
    r = RtRenderer(cam)
    r.update(space)
    g = DeviceGroup([0, 0])
    g.update(space)
    rng = np.random.default_rng(3)
    lo, size = np.array(space.lower, np.float64), np.array(space.size, np.float64)
    rays = np.ascontiguousarray(np.hstack([lo + rng.uniform(-0.5, 1.5, (1000, 3)) * size, rng.normal(size=(1000, 3))]))
    yield {"space": space, "opts": opts, "cam": cam, "ctx": r.rt.handle, "group": g.scene.handle, "rays": rays,
           "depth_transform": np.ascontiguousarray(cam.depth_transform(), dtype=np.float64).reshape(16)}
    g.close()
    r.rt.close()


class Dest:
    """Host buffers of one kind: numpy arrays over pageable, torch-pinned or cudaHostRegister'ed memory."""

    def __init__(self, kind):
        self.kind, self.keep, self.registered = kind, [], []

    def zeros(self, shape, dtype):
        nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        if self.kind == "pinned":
            t = torch.zeros(max(nbytes, 1), dtype=torch.uint8, pin_memory=True)
            self.keep.append(t)
            raw = t.numpy()
        else:
            raw = np.zeros(max(nbytes, 1), dtype=np.uint8)
            if self.kind == "registered":
                assert int(torch.cuda.cudart().cudaHostRegister(raw.ctypes.data, raw.nbytes, 1)) == 0   # portable
                self.registered.append(raw)
        return raw[:nbytes].view(dtype).reshape(shape)

    def close(self):
        for raw in self.registered:
            torch.cuda.cudart().cudaHostUnregister(raw.ctypes.data)
        self.registered = []


def ptr(a):
    return None if a is None else a.ctypes.data


def lib():
    return aicb200.load_library()


def layer(s, group):
    o = s["opts"].to_abi(True)
    s.setdefault("_keep", []).append(o)
    cls = abi.GroupLayer if group else abi.Layer
    return cls(s["group"] if group else s["ctx"], C.pointer(s["cam"].data), C.pointer(o))


def call(s, name, group, d, shard=None, want=("colorbuf", "depth", "hit", "steps"), pixels=None):
    """One host call into buffers of `d`; returns (status, {output: array}, info)."""
    L, info, o = lib(), abi.RenderInfo(), s["opts"].to_abi(True)
    cam, h = C.byref(s["cam"].data), s["group"] if group else s["ctx"]
    g = "aicb_group_" if group else "aicb_"
    n = N if shard is None else L.aicb_shard_pixel_count(cam, C.byref(shard))
    out = {}
    if name == "srgb8":
        out["srgb8"] = d.zeros((n, 4), np.uint8)
        args = (cam, C.byref(o)) + (() if group else (shard and C.byref(shard),)) + (ptr(out["srgb8"]), n)
        st = getattr(L, g + "render_srgb8")(h, *args, C.byref(info))
    elif name == "rgba16f":
        out["rgba16f"] = d.zeros((n, 4), np.uint16)
        args = (cam, C.byref(o)) + (() if group else (shard and C.byref(shard),)) + (ptr(out["rgba16f"]), n)
        st = getattr(L, g + "render_rgba16f")(h, *args, C.byref(info))
    elif name == "text":
        out["text"] = d.zeros(n, np.int32)
        st = getattr(L, g + "render_text")(h, cam, C.byref(o), ptr(out["text"]), n, C.byref(info))
    elif name in ("colorbuf", "rays"):
        m = n if name == "colorbuf" else len(s["rays"])
        shapes = {"colorbuf": ((m, 4), np.float32), "depth": (m, np.float64), "hit": ((m, 8), np.int32),
                  "steps": (m, np.uint32)}
        out = {k: d.zeros(*shapes[k]) if k in want else None for k in shapes}
        bufs = [ptr(out[k]) for k in ("colorbuf", "depth", "hit", "steps")]
        if name == "colorbuf":
            args = (cam, C.byref(o)) + (() if group else (shard and C.byref(shard),))
            st = getattr(L, g + "render_colorbuf")(h, *args, *bufs, m, C.byref(info))
        else:
            st = getattr(L, g + "trace_rays")(h, s["rays"].ctypes.data, m, C.byref(o), *bufs, C.byref(info))
        out = {k: v for k, v in out.items() if v is not None}
    elif name == "layers_srgb8":
        out["srgb8"] = d.zeros((N, 4), np.uint8)
        st = getattr(L, g + "render_layers_srgb8")(C.byref(layer(s, group)), None, None,
                                                   (C.c_float * 4)(*NO_WORLD), ptr(out["srgb8"]), N, C.byref(info))
    elif name == "terminal":
        out["terminal"] = d.zeros((N, 6), np.int32)
        st = getattr(L, g + "render_layers_terminal")(C.byref(layer(s, group)), None, None,
                                                      (C.c_float * 4)(*NO_WORLD), ptr(out["terminal"]), N,
                                                      C.byref(info))
    elif name == "texture":
        plist = np.arange(N, dtype=np.uint32)[::-3].copy() if pixels is None else pixels
        out["texel_rgba16f"] = d.zeros((len(plist), 4), np.uint16)
        out["texel_depth"] = d.zeros(len(plist), np.float32)
        st = getattr(L, g + "render_layers_texture")(
            C.byref(layer(s, group)), None, None, (C.c_float * 4)(*NO_WORLD),
            s["depth_transform"].ctypes.data_as(C.POINTER(C.c_double)), plist.ctypes.data if len(plist) else None,
            len(plist), ptr(out["texel_rgba16f"]), ptr(out["texel_depth"]), C.byref(info))
    elif name == "ortho":
        w, hh = C.c_uint32(), C.c_uint32()
        assert getattr(L, g + "ortho_image_size")(h, 4, C.byref(w), C.byref(hh)) == abi.OK
        out["ortho"] = d.zeros((w.value * hh.value, 4), np.uint8)
        st = getattr(L, g + "render_orthographic")(h, 4, ptr(out["ortho"]), w.value * hh.value, C.byref(info))
    return st, {k: np.array(v) for k, v in out.items()}, info


def counts(info):
    return (info.cubes_traced, info.rays, tuple(info.counters), info.algorithmic_bytes)


CALLS = ("srgb8", "rgba16f", "text", "colorbuf", "rays", "layers_srgb8", "terminal", "texture", "ortho")


@pytest.mark.parametrize("group", [False, True], ids=["context", "group"])
def test_every_kind_of_destination_takes_the_same_bytes(setup, group):
    for name in CALLS:
        got = {}
        for kind in KINDS:
            d = Dest(kind)
            st, out, info = call(setup, name, group, d)
            d.close()
            assert st == abi.OK, (name, kind)
            got[kind] = (out, counts(info))
        ref_out, ref_counts = got["pageable"]
        assert any(v.any() for v in ref_out.values()), name
        for kind in KINDS[1:]:
            out, c = got[kind]
            assert c == ref_counts, (name, kind)
            for k in ref_out:
                assert out[k].tobytes() == ref_out[k].tobytes(), (name, kind, k)


@pytest.mark.parametrize("name", ["colorbuf", "rays"])
def test_a_null_colorbuf(setup, name):
    _, full, full_info = call(setup, name, False, Dest("pageable"))
    # one context: the companions asked for are delivered without colorbuf
    st, some, info = call(setup, name, False, Dest("pageable"), want=("depth", "hit", "steps"))
    assert st == abi.OK and set(some) == {"depth", "hit", "steps"}
    for k in some:
        assert some[k].tobytes() == full[k].tobytes(), k
    assert counts(info) == counts(full_info)
    # every output NULL: the call still traces and fills info
    st, none, info = call(setup, name, False, Dest("pageable"), want=())
    assert st == abi.OK and not none and counts(info) == counts(full_info)
    # a group rejects a NULL colorbuf
    for want in (("depth", "hit", "steps"), ()):
        st, _, _ = call(setup, name, True, Dest("pageable"), want=want)
        assert st == abi.ERR_INVALID, want


@pytest.mark.parametrize("name", ["srgb8", "rgba16f", "colorbuf"])
def test_shards_reassemble_the_frame(setup, name):
    _, full, _ = call(setup, name, False, Dest("pageable"))
    strip, count = 4, 3
    rows = np.arange(H)
    got = {k: np.zeros_like(v) for k, v in full.items()}
    for index in range(count):
        shard = abi.Shard()
        shard.strip_rows, shard.index, shard.count = strip, index, count
        st, part, _ = call(setup, name, False, Dest("pinned"), shard=shard)
        assert st == abi.OK
        mine = rows[(rows // strip) % count == index]
        for k, v in part.items():
            frame = got[k].reshape(H, W, -1)
            frame[mine] = v.reshape(len(mine), W, -1)
    for k in full:
        assert got[k].tobytes() == full[k].tobytes(), k


@pytest.mark.parametrize("group", [False, True], ids=["context", "group"])
def test_an_empty_texture_batch_is_ok_and_zeroes_info(setup, group):
    info = abi.RenderInfo()
    C.memset(C.byref(info), 0xA5, C.sizeof(info))
    o = setup["opts"].to_abi(True)
    lay = abi.GroupLayer if group else abi.Layer
    lyr = lay(setup["group"] if group else setup["ctx"], C.pointer(setup["cam"].data), C.pointer(o))
    fn = lib().aicb_group_render_layers_texture if group else lib().aicb_render_layers_texture
    pixels = np.zeros(1, dtype=np.uint32)
    st = fn(C.byref(lyr), None, None, (C.c_float * 4)(*NO_WORLD),
            setup["depth_transform"].ctypes.data_as(C.POINTER(C.c_double)), pixels.ctypes.data, 0, None, None,
            C.byref(info))
    assert st == abi.OK
    assert bytes(info) == bytes(C.sizeof(info))


@pytest.mark.parametrize("group", [False, True], ids=["context", "group"])
def test_each_set_after_a_larger_call_of_another_set(setup, group):
    # every call after the one before it in CALLS, then each right after the largest staging layout (ColorBuf with
    # every companion), and that one again after it: a stale layout of the staging buffer would misplace an output
    alone = {name: call(setup, name, group, Dest("pageable")) for name in CALLS}
    for name in CALLS:
        big = call(setup, "colorbuf", group, Dest("pageable"))
        assert big[0] == abi.OK
        st, out, info = call(setup, name, group, Dest("pageable"))
        assert st == abi.OK and counts(info) == counts(alone[name][2]), name
        for k in out:
            assert out[k].tobytes() == alone[name][1][k].tobytes(), (name, k)
        st, again, _ = call(setup, "colorbuf", group, Dest("pageable"))
        for k in again:
            assert again[k].tobytes() == big[1][k].tobytes(), (name, k)
