"""Pixel picking (csrc/gbuffer.cu), the Display pass's G-buffer debug views and the outline of picked instances (csrc/display.cu)
against the CPU oracle (oracle/orc_display_views.cpp), bit for bit; an independent check of the pick mask against the G-buffer's
own hits; strip-sharded frames through the thread-transport harness; refusals, resize and launch counts."""
import ctypes as C

import numpy as np
import pytest

from tests.orc import ptr

pytestmark = pytest.mark.gpu

W, H = 96, 64
SHORT_BOX, TALL_BOX = 8, 9          # instance indices in the Cornell fixture


def _scene():
    """Cornell with a coated back wall, a metal short box, a glass tall box and the emissive ceiling light"""
    from tests import scene_util
    from zetaray_b200 import scene as zscene
    s = scene_util.glossy_cornell()
    m = s.materials.copy()
    m[8] = zscene.make_material(base_color=(0.6, 0.85, 0.7, 1), roughness=0.3, ior=1.33, transmission=1.0, double_sided=True)
    s.materials = m
    return s


def _fc(w=W, h=H, cam=(0.0, 1.2, -4.043), jitter=(0.0, 0.0), dof=False):
    from zetaray_b200.camera import look_at_frame_constants
    fc = look_at_frame_constants(w, h, jitter=jitter, cam=cam)
    if dof:
        fc.DoF, fc.LensRadius, fc.FocusDepth = 1, 0.05, 4.0
    return fc


class Frame:
    """A device G-buffer of one frame and the oracle scene beside it."""

    def __init__(self, flat, w=W, h=H):
        from zetaray_b200.passes import Scene, GBuffers, GBufferRT
        from tests.scene_util import OracleScene
        self.flat, self.w, self.h = flat, w, h
        self.scene = Scene(flat)
        self.scene.prelighting()
        self.gb, self.gpass = GBuffers(w, h), GBufferRT()
        self.orc = OracleScene(flat)
        self.o = self.orc.o
        self.o.orc_gbuffer_pick.restype = C.c_uint32

    def render(self, fc):
        from zetaray_b200 import _lib, lib, check
        fi = _lib.FrameInputs()
        fi.frame = fc
        self.gb.fill_inputs(fi)
        fi.scene = self.scene.handle
        self.gpass.Render(fi)
        check(lib.zr_stream_synchronize(None))
        self.fi = fi
        return fi

    def orc_pick(self, fc, x, y):
        return self.o.orc_gbuffer_pick(self.orc.h, C.byref(fc), x, y)

    def orc_display(self, fc, view, picks, base=None, th=1.0, y0=0, y1=None):
        """the oracle's display image: `base` (the DEFAULT image) or the view, then the outline of `picks`"""
        y1 = self.h if y1 is None else y1
        n = self.w * self.h
        out = np.zeros(n, dtype=np.uint32) if base is None else base.copy()
        if view:
            core, _, me, coat, _ = self.gb.download()
            self.o.orc_display_view(ptr(core), ptr(me), ptr(coat), self.w, y0, y1, view, C.c_float(th), C.c_float(fc.CameraNear), ptr(out))
        if len(picks):
            mask = self.mask(fc, picks)
            self.o.orc_outline(ptr(mask), self.w, self.h, y0, y1, ptr(out))
        return out

    def mask(self, fc, picks):
        mask = np.zeros(self.w * self.h, dtype=np.uint32)
        inst = np.asarray(picks, dtype=np.uint32)
        self.o.orc_pick_mask(self.orc.h, C.byref(fc), ptr(inst), len(inst), 0, self.h, ptr(mask))
        return mask


def _display(frame, fc, view, picks, th=1.0, signal=None):
    """the device display image: DEFAULT with tone mapper NONE over `signal`, or a view (no signal, exposure or LUT)"""
    from zetaray_b200.passes import Display, download_image
    d = Display(frame.w, frame.h)
    d.SetParams(tonemapper=Display.NONE, auto_exposure=0)
    d.SetView(view, th)
    d.SetPicked(picks)
    d.Render(frame.fi, signal, None)
    return d, download_image(d.GetOutput(), np.uint32, 1).ravel()


def _taa(w, h, seed):
    from tests.test_display_gpu import _taa_image
    from tests.gpu_util import dev
    img = _taa_image(w, h, seed)
    return img, dev(img)


def _oracle_default(frame, img):
    from zetaray_b200 import _lib
    p = _lib.DisplayParams(0, 0, 1.0, 1.0)
    out = np.zeros(frame.w * frame.h, dtype=np.uint32)
    frame.o.orc_display(ptr(img), frame.w, 0, frame.h, C.byref(p), None, None, ptr(out))
    return out


@pytest.fixture(scope="module")
def frame():
    return Frame(_scene())


@pytest.mark.parametrize("view", range(1, 10))
def test_views_match_oracle(frame, view):
    fc = _fc()
    frame.render(fc)
    core = frame.gb.download()[0]
    flags = core[:, 3] & 0xff
    for bit in (1, 2, 32, 128):             # transmissive, emissive, coated, metal pixels are all on screen
        assert ((flags & bit) != 0).any(), bit
    for th in (0.25, 1.0):
        _, got = _display(frame, fc, view, [], th)
        want = frame.orc_display(fc, view, [], th=th)
        assert np.array_equal(got, want), (view, th, np.flatnonzero(got != want)[:10])


def test_pick_matches_oracle_with_dof_and_jitter(frame):
    from zetaray_b200.passes import GBufferRT
    fc = _fc(jitter=(0.3125, -0.1875), dof=True)
    rng = np.random.default_rng(3)
    seen = set()
    for x, y in zip(rng.integers(0, W, 64), rng.integers(0, H, 64)):
        frame.gpass.Pick(int(x), int(y))
        frame.render(fc)
        got = frame.gpass.GetPick()
        assert got == frame.orc_pick(fc, int(x), int(y)), (x, y)
        seen.add(got)
    assert len(seen) >= 4
    depth = frame.gb.download()[1]
    bg = int(np.flatnonzero(depth == np.float32(3.402823466e38))[0])
    frame.gpass.Pick(bg % W, bg // W)
    frame.render(fc)
    assert frame.gpass.GetPick() == GBufferRT.NO_PICK
    frame.gpass.Pick(W // 2, H // 2)
    frame.render(fc)
    hit = frame.gpass.GetPick()
    assert hit != GBufferRT.NO_PICK
    frame.gpass.Pick(W + 3, 1)              # outside the frame
    frame.render(fc)
    assert frame.gpass.GetPick() == GBufferRT.NO_PICK
    frame.gpass.Pick(W // 2, H // 2)
    frame.render(fc)
    frame.render(fc)                        # a pick is one-shot: the second render leaves the word alone
    frame.gpass.SetRows(0, H // 2)
    frame.render(fc)
    assert frame.gpass.GetPick() == hit
    frame.gpass.Pick(W // 2, H // 2 + 1)    # a row this pass does not render
    frame.render(fc)
    assert frame.gpass.GetPick() == GBufferRT.NO_PICK
    frame.gpass.SetRows(0, H)


@pytest.mark.parametrize("picks,cam,jitter,view", [
    ([SHORT_BOX], (0.0, 1.2, -4.043), (0.0, 0.0), 0),
    ([SHORT_BOX, TALL_BOX], (0.0, 1.2, -4.043), (0.3125, -0.4375), 0),
    (list(range(10)) * 3 + [0, 9], (0.0, 1.2, -4.043), (0.0, 0.0), 2),
    ([0, SHORT_BOX, TALL_BOX], (0.1, 1.6, -0.85), (0.0, 0.0), 0),          # inside the room: walls cross the near plane
    ([0, 3, TALL_BOX], (0.1, 1.6, -0.85), (-0.25, 0.125), 7),
], ids=["one", "two-jitter", "32-normal-view", "inside-room", "inside-room-jitter-emissive-view"])
def test_outline_matches_oracle(frame, picks, cam, jitter, view):
    fc = _fc(cam=cam, jitter=jitter)
    frame.render(fc)
    img, d_img = _taa(W, H, 5)
    base = _oracle_default(frame, img) if view == 0 else None
    _, got = _display(frame, fc, view, picks, signal=d_img.data_ptr() if view == 0 else None)
    want = frame.orc_display(fc, view, picks, base=base)
    assert (want != (base if base is not None else frame.orc_display(fc, view, []))).any(), "no outline drawn"
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]


def test_mask_is_the_silhouette_of_an_unoccluded_instance(frame):
    fc = _fc()
    ids = np.array([frame.orc_pick(fc, x, y) for y in range(H) for x in range(W)], dtype=np.int64).reshape(H, W)
    mask = (frame.mask(fc, [SHORT_BOX]) & 1).reshape(H, W).astype(bool)
    hit = ids == SHORT_BOX
    pad = np.pad(hit, 1, constant_values=False)
    nb = [pad[1 + dy:H + 1 + dy, 1 + dx:W + 1 + dx] for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
    mixed = np.any(nb, 0) & ~np.all(nb, 0)
    assert hit.sum() > 100
    assert np.array_equal(mask[~mixed], hit[~mixed])


@pytest.mark.parametrize("view,bounds", [(2, [0, 64, 128]), (0, [0, 32, 64, 128])], ids=["normal-view", "default-3-ranks"])
def test_sharded_display_and_pick(view, bounds):
    W, H = 96, 128          # strip bounds are multiples of 32 rows; these cut through both boxes
    import torch
    from zetaray_b200.passes import Scene, Renderer, GBufferRT
    from tests.sharded_util import ThreadTransport, host_rows, run_threads
    from tests.test_display_oracle import load_lut
    flat, lut = _scene(), load_lut()
    picks, px = [SHORT_BOX, TALL_BOX, 3], (W // 2 - 7, 64)        # on a strip boundary, inside the box
    fcs = [_fc(W, H) for _ in range(3)]
    for f, fc in enumerate(fcs):
        fc.FrameNum, fc.dt = f + 1, 1 / 60

    def setup(R):
        R.SetDisplay(True, lut=lut)
        R.display.SetView(view)
        R.display.SetPicked(picks)

    ref = Renderer(Scene(flat), W, H, two_streams=False)
    setup(ref)
    for f, fc in enumerate(fcs):
        if f == len(fcs) - 1:
            ref.Pick(*px)
        ref.Render(fc)
        torch.cuda.synchronize()
    want, want_pick = host_rows(ref.GetDisplayOutput()), ref.GetPick()
    assert want_pick != GBufferRT.NO_PICK

    world = len(bounds) - 1
    ranks = [Renderer(Scene(flat), W, H, two_streams=False) for _ in range(world)]
    transports = ThreadTransport.group(world)
    comms = [t.comm() for t in transports]
    got, picked = [None] * world, [None] * world

    def rank_main(rank):
        R = ranks[rank]
        st = torch.cuda.Stream()
        setup(R)
        for f, fc in enumerate(fcs):
            if f == 1:
                R.SetShard(comms[rank], bounds, gather_output=True)
            if f == len(fcs) - 1:
                R.Pick(*px)
            R.Render(fc, C.c_void_p(st.cuda_stream))
            torch.cuda.synchronize()
        got[rank] = host_rows(R.GetDisplayOutput())
        picked[rank] = R.GetPick()

    run_threads(transports, rank_main)
    assert np.array_equal(got[0], want)
    assert min(picked) == want_pick
    # the rank that owns the row reports it; a rank whose G-buffer rows reach it as a halo reports the same instance
    owner = [r for r in range(world) if bounds[r] <= px[1] < bounds[r + 1]][0]
    assert picked[owner] == want_pick and all(p in (want_pick, GBufferRT.NO_PICK) for p in picked), picked


def test_refusals_resize_and_launch_counts(frame):
    from zetaray_b200 import lib
    from zetaray_b200._lib import ZRError
    from zetaray_b200.passes import Display
    fc = _fc()
    frame.render(fc)
    img, d_img = _taa(W, H, 9)
    d = Display(W, H)
    d.SetParams(tonemapper=Display.NONE, auto_exposure=0)
    for bad in (lambda: d.SetView(10), lambda: d.SetView(1, float("nan")), lambda: d.SetView(6, float("inf")),
                lambda: d.SetPicked(list(range(33)))):
        with pytest.raises(ZRError):
            bad()
    assert lib.zr_display_pass_set_picked(d.handle, None, 2) != 0
    # DEFAULT with nothing picked launches k_display alone
    n0 = lib.zr_kernel_launch_count()
    d.Render(frame.fi, d_img.data_ptr(), None)
    assert lib.zr_kernel_launch_count() - n0 == 1
    d.SetPicked([len(frame.flat.instances)])
    n0 = lib.zr_kernel_launch_count()
    with pytest.raises(ZRError, match="picked instance %d" % len(frame.flat.instances)):
        d.Render(frame.fi, d_img.data_ptr(), None)
    assert lib.zr_kernel_launch_count() == n0
    d.SetView(Display.VIEW_NORMAL)
    d.SetPicked([SHORT_BOX])
    n0 = lib.zr_kernel_launch_count()
    d.Render(frame.fi, None, None)
    assert lib.zr_kernel_launch_count() - n0 == 3         # view, mask, outline
    d.SetPicked([])
    n0 = lib.zr_kernel_launch_count()
    d.Render(frame.fi, None, None)
    assert lib.zr_kernel_launch_count() - n0 == 1
    # a resize keeps the view and the picks and resizes the mask
    from zetaray_b200.passes import download_image
    w2, h2 = 120, 72
    f2 = Frame(frame.flat, w2, h2)
    fc2 = _fc(w2, h2)
    f2.render(fc2)
    d.SetPicked([SHORT_BOX, TALL_BOX])
    d.OnWindowResized(w2, h2)
    d.Render(f2.fi, None, None)
    got = download_image(d.GetOutput(), np.uint32, 1).ravel()
    assert np.array_equal(got, f2.orc_display(fc2, Display.VIEW_NORMAL, [SHORT_BOX, TALL_BOX]))
