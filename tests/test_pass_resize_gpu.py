"""Pass resize on the device: a resized pass matches one created at the new size (also when it had a row range, which the resize
returns to the whole frame), a failed resize changes nothing, a resize forgets the cost map, and zero sizes are refused. Cornell box at small sizes; outputs are compared byte for byte."""
import ctypes as C

import numpy as np
import pytest
import torch

A, B = (64, 48), (96, 40)
HUGE = 1 << 20                  # 2^20 x 2^20 pixels: no plane of that size fits on any device
ZR_ERR_INVALID_ARG, ZR_ERR_OUT_OF_MEMORY = 1, 5
KINDS = ["direct", "indirect", "gi", "pathtracer", "compositing", "taa", "svgf"]
# AutoExposure's planes do not grow with the image, so no size makes its resize fail
RESIZE_KINDS = KINDS + ["auto_exposure", "display"]


class _World:
    """Scene, per-size G-buffers and frame sequences, and per-frame input signals shared by every pass under test."""

    def __init__(self):
        from zetaray_b200.passes import Scene, GBufferRT
        from tests import scene_util
        self.scene = Scene(scene_util.cornell())
        self.scene.prelighting()
        self.gpass = GBufferRT()
        self.sizes = {}

    def frame(self, size):
        """Renders the next G-buffer at `size`; returns the frame inputs and two deterministic RGBA32F signals."""
        from zetaray_b200 import _lib
        from zetaray_b200.passes import GBuffers
        from tests import rpt_util
        if size not in self.sizes:
            self.sizes[size] = (GBuffers(*size), rpt_util.FrameSequence(*size))
        gb, seq = self.sizes[size]
        fc = seq.next()
        fc.dt = 1 / 60                  # AutoExposure's time step
        gb.flip()
        fi = _lib.FrameInputs()
        fi.frame = fc
        gb.fill_inputs(fi)
        fi.scene = self.scene.handle
        self.gpass.Render(fi)
        g = torch.Generator(device="cpu").manual_seed(fc.FrameNum * 7919 + size[0] * 31 + size[1])
        sig = [torch.rand(size[0] * size[1] * 4, generator=g).cuda() for _ in range(2)]
        torch.cuda.synchronize()
        return fi, sig

    def close(self):
        for gb, _ in self.sizes.values():
            gb.close()
        self.scene.close()


class _Pass:
    """One pass of `kind` behind the same four verbs: render, resize (returns the status), outputs, size."""

    def __init__(self, kind, size):
        from zetaray_b200 import lib
        from zetaray_b200 import passes as P
        self.kind = kind
        cls = {"direct": P.DirectLighting, "indirect": P.IndirectLighting, "gi": P.IndirectLightingGI, "pathtracer": P.IndirectLightingGI,
               "compositing": P.Compositing, "taa": P.TAA, "svgf": P.SVGF, "auto_exposure": P.AutoExposure, "display": P.Display}[kind]
        self.p = cls(*size)
        if kind == "pathtracer":
            self.p.SetMethod(0)     # ZR_INTEGRATOR_PATH_TRACING
        if kind == "display":
            from tests.test_display_oracle import load_lut
            self.p.SetLUT(load_lut())
        self.prefix = self.p.prefix
        self.ids = {"direct": [0, 1, 2], "indirect": [0, 1, 2, 3, 4, 6], "gi": [0, 1, 2], "pathtracer": [0, 1, 2],
                    "compositing": [None], "taa": [None], "svgf": [0, 1, 2, 3], "auto_exposure": [None], "display": [None]}[kind]
        self.lib = lib

    def render(self, world, size):
        from zetaray_b200 import lib, check
        fi, sig = world.frame(size)
        self.feed(fi, sig)
        check(lib.zr_stream_synchronize(None))

    def feed(self, fi, sig):
        if self.kind == "compositing":
            self.p.Render(fi, sig[0].data_ptr(), sig[1].data_ptr())
        elif self.kind in ("taa", "svgf", "auto_exposure"):
            self.p.Render(fi, sig[0].data_ptr())
        elif self.kind == "display":
            self.p.Render(fi, sig[0].data_ptr(), sig[1].data_ptr())     # signal read as half4, exposure as float2
        else:
            self.p.Render(fi)

    def resize(self, w, h):
        return getattr(self.lib, self.prefix + "_resize")(self.p.handle, w, h)

    def images(self):
        return [self.p.GetOutput() if i is None else self.p.GetOutput(i) for i in self.ids]

    def size(self):
        img = self.images()[0]
        return img.width, img.height

    def outputs(self):
        """(id, width, height, pitch, bytes) of every exported image."""
        from zetaray_b200 import lib, check
        out = []
        for i, img in zip(self.ids, self.images()):
            raw = np.zeros(img.height * img.pitch_bytes, dtype=np.uint8)
            check(lib.zr_memcpy_d2h(C.c_void_p(raw.ctypes.data), C.c_void_p(img.d_ptr), C.c_size_t(raw.nbytes), None))
            check(lib.zr_stream_synchronize(None))
            out.append((i, img.width, img.height, img.pitch_bytes, raw.tobytes()))
        return out


def _render_both(world, size, a, b, n):
    """Feeds the same n frames at `size` to passes a and b."""
    from zetaray_b200 import lib, check
    for _ in range(n):
        fi, sig = world.frame(size)
        a.feed(fi, sig)
        b.feed(fi, sig)
        check(lib.zr_stream_synchronize(None))


def _assert_same(a, b, what):
    for (i, w, h, pitch, ra), (_, w2, h2, pitch2, rb) in zip(a.outputs(), b.outputs()):
        assert (w, h, pitch) == (w2, h2, pitch2), "%s output %s: %dx%d pitch %d vs %dx%d pitch %d" % (what, i, w, h, pitch, w2, h2, pitch2)
        assert ra == rb, "%s output %s differs in %d of %d bytes" % (
            what, i, int((np.frombuffer(ra, np.uint8) != np.frombuffer(rb, np.uint8)).sum()), len(ra))


@pytest.fixture(scope="module")
def world():
    w = _World()
    yield w
    w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", RESIZE_KINDS)
def test_resize_equals_fresh(world, kind):
    from zetaray_b200 import check
    p = _Pass(kind, A)
    for _ in range(3):
        p.render(world, A)
    p.p.SetRows(16, 32)                 # the first resize returns the pass to the whole frame; the second one starts there
    for size in (B, A):
        check(p.resize(*size))
        assert p.size() == (size if kind != "auto_exposure" else (1, 1))        # AutoExposure's output is its 1 x 1 state
        fresh = _Pass(kind, size)
        _render_both(world, size, p, fresh, 3)
        _assert_same(p, fresh, "%s resized to %dx%d" % ((kind,) + size))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_failed_resize_changes_nothing(world, kind):
    from zetaray_b200 import lib
    p, twin = _Pass(kind, A), _Pass(kind, A)
    _render_both(world, A, p, twin, 2)
    st = p.resize(HUGE, HUGE)
    assert st == ZR_ERR_OUT_OF_MEMORY, (st, lib.zr_last_error())
    assert p.prefix.encode() in lib.zr_last_error(), lib.zr_last_error()
    assert p.size() == A
    # only now that the pass is known to be whole does anything launch on it
    _assert_same(p, twin, "%s after the failed resize" % kind)
    _render_both(world, A, p, twin, 2)
    _assert_same(p, twin, "%s rendering after the failed resize" % kind)


@pytest.mark.gpu
def test_failed_gbuffer_alloc_frees_and_zeroes():
    from zetaray_b200 import lib, _lib
    g = _lib.GBuffer()
    st = lib.zr_gbuffer_alloc(HUGE, HUGE, 1, C.byref(g))
    assert st == ZR_ERR_OUT_OF_MEMORY, (st, lib.zr_last_error())
    assert b"zr_gbuffer_alloc" in lib.zr_last_error()
    assert bytes(g) == bytes(C.sizeof(g))
    # the failed allocation is not left behind as the runtime's last error
    g2 = _lib.GBuffer()
    assert lib.zr_gbuffer_alloc(A[0], A[1], 1, C.byref(g2)) == 0
    lib.zr_gbuffer_free(C.byref(g2))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["direct", "indirect"])
def test_resize_forgets_cost_map(world, kind):
    from zetaray_b200 import check
    p = _Pass(kind, A)
    tiles = ((A[0] + 31) // 32) * ((A[1] + 31) // 32)
    cost = torch.zeros(tiles, dtype=torch.int64, device="cuda")
    p.p.SetCostMap(cost.data_ptr())
    small = (A[0] // 2, A[1] // 2)
    check(p.resize(*small))
    p.render(world, small)
    torch.cuda.synchronize()
    assert int(cost.count_nonzero()) == 0, cost.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["direct", "indirect", "gi", "compositing", "taa", "svgf"])
def test_zero_size_resize_is_refused(kind):
    p = _Pass(kind, A)
    assert p.resize(0, A[1]) == ZR_ERR_INVALID_ARG
    assert p.resize(A[0], 0) == ZR_ERR_INVALID_ARG
    assert p.size() == A
