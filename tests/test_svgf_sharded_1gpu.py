"""The SVGF denoiser in strip-sharded frames, on ONE GPU.

A lone pass with a row range computes only those rows and calls the halo hook once after its temporal stage and once after every
a-trous pass; fed the bands of a whole-frame pass there, its rows are byte-identical to that pass's. The renderer with the stage
in strip-sharded frames is tested with the rest of the frame in tests/test_sharded_1gpu.py."""
import numpy as np
import pytest

from tests.sharded_util import check_set_rows, device_rows, host_rows

pytestmark = pytest.mark.gpu

HALO = 32
ZR_SVGF_DENOISED, ZR_SVGF_ACCUMULATED, ZR_SVGF_GUIDE, ZR_SVGF_HISTORY = range(4)


def _svgf_rows(p):
    return {name: host_rows(p.GetOutput(i)) for name, i in (("denoised", ZR_SVGF_DENOISED), ("guide", ZR_SVGF_GUIDE), ("history", ZR_SVGF_HISTORY))}


def _gbuffer_frame(which, w, h, nframes):
    """(DeviceFrame, [frame constants]) of a slowly moving camera; DeviceFrame.render(fc) renders the G-buffer only."""
    from tests import scene_util
    from tests.parity import DeviceFrame
    from zetaray_b200.camera import FrameSequence
    seq = FrameSequence(w, h, cam_path=lambda f: (0.02 * f, 1.2, -4.043))
    return DeviceFrame(scene_util.SCENES[which](), w, h, ()), [seq.next() for _ in range(nframes)]


def _signal(w, h, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    s = torch.rand((h, w, 4), device="cuda", generator=g) * torch.tensor([1.0, 30.0, 0.1], device="cuda")[
        torch.randint(0, 3, (h, w, 1), device="cuda", generator=g)]
    return s.contiguous()


class HookLog:
    """A halo hook that records every call: [(d_ptr, width, height, pitch_bytes, texel_bytes) per plane]. `then` runs after."""

    def __init__(self, then=None):
        from zetaray_b200 import _lib
        self.calls, self.errors, self.then = [], [], then
        self.fn = _lib.HALO_EXCHANGE_FN(self._hook)

    def _hook(self, user, planes, n, stream):
        try:
            self.calls.append([(planes[i].d_ptr or 0, planes[i].width, planes[i].height, planes[i].pitch_bytes, planes[i].texel_bytes)
                               for i in range(n)])
            if self.then:
                self.then(len(self.calls) - 1, [planes[i] for i in range(n)])
        except BaseException as e:      # noqa: BLE001  (nothing propagates out of a ctypes callback)
            self.errors.append(e)


def test_svgf_set_rows_refuses_empty_ranges():
    from zetaray_b200.passes import SVGF
    check_set_rows(SVGF(96, 70), 70)


def test_svgf_hook_calls_and_planes():
    """num_passes + 1 hook calls per render, each with the planes the next stage reads beyond the strip and their real pitches."""
    import torch
    from zetaray_b200.passes import SVGF
    W, H = 96, 70
    dev, fcs = _gbuffer_frame("cornell", W, H, 1)
    fi = dev.render(fcs[0])
    sig = _signal(W, H, 1)
    p = SVGF(W, H)
    log = HookLog()
    p.SetHaloExchange(log.fn)
    for n in range(1, 6):
        p.SetParams(num_passes=n)
        log.calls.clear()
        p.Render(fi, sig.data_ptr())
        torch.cuda.synchronize()
        assert not log.errors, log.errors[0]
        assert len(log.calls) == n + 1, (n, len(log.calls))
        guide, hist, cv0, out = p.GetOutput(ZR_SVGF_GUIDE), p.GetOutput(ZR_SVGF_HISTORY), p.GetOutput(ZR_SVGF_ACCUMULATED), p.GetOutput(ZR_SVGF_DENOISED)
        pitch = guide.pitch_bytes // 8
        assert pitch > W and hist.pitch_bytes == pitch * 16        # padded planes: the hook must see their pitch, not width * texel
        assert log.calls[0] == [(cv0.d_ptr, W, H, pitch * 8, 8), (guide.d_ptr, W, H, pitch * 8, 8), (hist.d_ptr, W, H, pitch * 16, 16)]
        cv1 = None
        for k in range(1, n):           # pass k - 1 wrote colour + variance plane k % 2 (pass 0 reads plane 0)
            (plane,) = log.calls[k]
            assert plane[1:] == (W, H, pitch * 8, 8), (n, k, plane)
            if k % 2 == 0:
                assert plane[0] == cv0.d_ptr, (n, k)
            else:
                cv1 = cv1 or plane[0]
                assert plane[0] == cv1 and cv1 != cv0.d_ptr, (n, k)
        assert log.calls[n] == [(out.d_ptr, W, H, W * 16, 16)]
    dev.close()


def test_svgf_resize_returns_to_the_whole_frame_and_keeps_the_hook():
    import torch
    from zetaray_b200.passes import SVGF
    W, H = 160, 96
    a = SVGF(96, 70)
    log = HookLog()
    a.SetRows(32, 64)
    a.SetHaloExchange(log.fn)
    a.OnWindowResized(W, H)
    b = SVGF(W, H)
    dev, fcs = _gbuffer_frame("glossy", W, H, 2)
    for f, fc in enumerate(fcs):
        fi = dev.render(fc)
        sig = _signal(W, H, 10 + f)
        a.Render(fi, sig.data_ptr())
        b.Render(fi, sig.data_ptr())
        torch.cuda.synchronize()
        got, want = _svgf_rows(a), _svgf_rows(b)
        for k in want:
            assert np.array_equal(got[k], want[k]), "frame %d: %s differs after the resize" % (f, k)
    assert not log.errors and len(log.calls) == 2 * 6, (log.errors, len(log.calls))
    dev.close()


@pytest.mark.parametrize("W,H,y0,y1,radius,passes", [
    (288, 200, 96, 256, 2, 5),      # the last strip, rows past the image clipped; every pass reaches the full 32 rows
    (320, 300, 248, 300, 2, 5),     # unaligned start: the y-phases of a lattice pass start in different tile rows
    (333, 187, 5, 37, 1, 3),        # odd size, a 32-row strip near the top
    (256, 144, 131, 132, 2, 4),     # one row: most y-phases of the coarse passes hold none of it
], ids=["last-strip-clipped", "unaligned", "odd-r1", "one-row"])
def test_svgf_strip_rows_equal_whole_frame(W, H, y0, y1, radius, passes):
    """A pass with rows [y0, y1) whose hook fills the 32-row bands either side with what a whole-frame pass had at the same stage,
    and fills every row beyond them with random bytes: its own rows equal the whole-frame pass's, its temporal stage writes no
    other row of the guide and the history, and its last pass writes no other row of the denoised image."""
    import torch
    from zetaray_b200.passes import SVGF
    y1 = min(y1, H)
    nframes = 3                         # the guide / history plane written in frame f is written again in frame f + 2
    dev, fcs = _gbuffer_frame("glass", W, H, nframes)
    whole, strip = SVGF(W, H), SVGF(W, H)
    for p in (whole, strip):
        p.SetParams(radius=radius, num_passes=passes)
    strip.SetRows(y0, y1)
    gen = torch.Generator(device="cuda").manual_seed(5)
    stages, left, problems = [], {}, []
    SENTINEL = 0xAB

    def snapshot(call, planes):
        torch.cuda.synchronize()
        stages.append([device_rows(pl).clone() for pl in planes])

    def bands(call, planes):
        torch.cuda.synchronize()
        lo, hi = max(0, y0 - HALO), min(H, y1 + HALO)
        for j, pl in enumerate(planes):
            rows = device_rows(pl)
            outside = torch.ones(H, dtype=torch.bool, device="cuda")
            outside[y0:y1] = False
            if call == 0 and j > 0 and pl.d_ptr in left:
                if not torch.equal(rows[outside], left[pl.d_ptr][outside]):
                    problems.append("temporal stage wrote rows outside the strip of plane %d" % j)
            if call == passes and not bool((rows[outside] == SENTINEL).all()):
                problems.append("last pass wrote rows of the denoised image outside the strip")
            rows[lo:y0].copy_(stages[call][j][lo:y0])
            rows[y1:hi].copy_(stages[call][j][y1:hi])
            for a, b in ((0, lo), (hi, H)):
                if b > a:
                    rows[a:b].copy_(torch.randint(0, 256, rows[a:b].shape, dtype=torch.uint8, device="cuda", generator=gen))
            if call == 0 and j > 0:
                left[pl.d_ptr] = rows.clone()
        torch.cuda.synchronize()

    hw, hs = HookLog(snapshot), HookLog(bands)
    whole.SetHaloExchange(hw.fn)
    strip.SetHaloExchange(hs.fn)
    for f, fc in enumerate(fcs):
        fi = dev.render(fc)
        sig = _signal(W, H, 100 + f)
        stages.clear(); hw.calls.clear(); hs.calls.clear()     # a hook call's index is its stage in this frame
        whole.Render(fi, sig.data_ptr())
        torch.cuda.synchronize()
        device_rows(strip.GetOutput(ZR_SVGF_DENOISED)).fill_(SENTINEL)
        strip.Render(fi, sig.data_ptr())
        torch.cuda.synchronize()
        assert not hw.errors and not hs.errors, (hw.errors + hs.errors)[0]
        assert len(stages) == passes + 1
        assert not problems, "frame %d: %s" % (f, problems[0])
        got, want = _svgf_rows(strip), _svgf_rows(whole)
        for k in want:
            bad = np.argwhere(got[k][y0:y1] != want[k][y0:y1])
            assert not bad.size, "frame %d: %s differs, first at (row, byte) %s of strip [%d, %d)" % (f, k, (bad[0] + [y0, 0]).tolist(), y0, y1)
    dev.close()
