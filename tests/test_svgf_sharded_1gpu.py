"""The SVGF denoiser in strip-sharded frames, on ONE GPU.

A lone pass with a row range computes only those rows and calls the halo hook once after its temporal stage and once after every
a-trous pass; fed the bands of a whole-frame pass there, its rows are byte-identical to that pass's. The renderer runs the stage
sharded with host threads as ranks over a caller-supplied transport (ThreadTransport, tests/test_sharded_1gpu.py): every rank's
rows of the denoised image, the SVGF history and guide, TAA and the display image are byte-identical to the unsharded frame."""
import ctypes as C
import threading

import numpy as np
import pytest

from tests.test_sharded_1gpu import ThreadTransport, _device_rows

pytestmark = pytest.mark.gpu

HALO = 32
ZR_SVGF_DENOISED, ZR_SVGF_ACCUMULATED, ZR_SVGF_GUIDE, ZR_SVGF_HISTORY = range(4)


def _rows(img):
    """uint8 [height, width * texel] host copy of a (possibly padded) zr_image2d."""
    from zetaray_b200.passes import download_image_pitched
    return download_image_pitched(img, np.uint8, img.texel_bytes).reshape(img.height, -1)


def _svgf_rows(p):
    return {name: _rows(p.GetOutput(i)) for name, i in (("denoised", ZR_SVGF_DENOISED), ("guide", ZR_SVGF_GUIDE), ("history", ZR_SVGF_HISTORY))}


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
    from zetaray_b200 import lib
    from zetaray_b200.passes import SVGF
    W, H = 96, 70
    p = SVGF(W, H)
    for y0, y1 in ((0, 0), (40, 20), (H, H + 32), (H + 5, H + 40)):
        assert lib.zr_svgf_pass_set_rows(p.handle, y0, y1) == 1, (y0, y1)      # ZR_ERR_INVALID_ARG
        assert lib.zr_last_error() == b"zr_svgf_pass_set_rows: empty row range"
    assert lib.zr_svgf_pass_set_rows(None, 0, H) == 1
    assert lib.zr_svgf_pass_set_halo_exchange(None, None, None) == 1
    p.SetRows(32, H + 100)              # rows past the image are clipped when the pass renders
    p.SetHaloExchange(None)


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
        stages.append([_device_rows(pl).clone() for pl in planes])

    def bands(call, planes):
        torch.cuda.synchronize()
        lo, hi = max(0, y0 - HALO), min(H, y1 + HALO)
        for j, pl in enumerate(planes):
            rows = _device_rows(pl)
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
        _device_rows(strip.GetOutput(ZR_SVGF_DENOISED)).fill_(SENTINEL)
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


# ---- the renderer: host threads as ranks ---------------------------------------------------------------------------------------

W, H = 288, 200


def _frame_constants(n):
    from zetaray_b200.camera import FrameSequence
    seq = FrameSequence(W, H, cam_path=lambda f: (0.02 * f, 1.2, -4.043))
    fcs = [seq.next() for _ in range(n)]
    for fc in fcs:
        fc.dt = 1 / 60
    return fcs


def _renderer(flat, integrator, two_streams, display, lut):
    from zetaray_b200.passes import Scene, Renderer
    R = Renderer(Scene(flat), W, H, two_streams=two_streams)       # every renderer has its own scene (prelighting runs on it)
    if integrator == "gi":
        R.SetMethod(Renderer.RESTIR_GI)
    if display:
        R.SetDisplay(True, lut=lut)
    return R


def _denoise(R, svgf):
    R.SetDenoiser(True)
    R.svgf.SetParams(radius=svgf[0], num_passes=svgf[1])


def _outputs(R, display):
    out = {"composited": _rows(R.compositing.GetOutput()), "taa": _rows(R.GetOutput())}
    if R.svgf is not None:
        out.update(("svgf " + k, v) for k, v in _svgf_rows(R.svgf).items())
    if display:
        out["display"] = _rows(R.GetDisplayOutput())
    return out


def _frame_inputs(R, fc):
    """The FrameInputs the renderer's passes saw in its last frame."""
    from zetaray_b200 import lib, check, _lib
    fi = _lib.FrameInputs()
    fi.frame = fc
    check(lib.zr_renderer_get_gbuffer(R.handle, 0, C.byref(fi.curr)))
    check(lib.zr_renderer_get_gbuffer(R.handle, 1, C.byref(fi.prev)))
    fi.scene = R.scene.handle
    return fi


def _run_threads(which, integrator, bounds, two_streams, svgf, display=False, warm=2, frames=4, svgf_from=0, unshard_after=0,
                 compare=True):
    """Renders warm unsharded frames, then `frames` sharded frames on len(bounds) - 1 thread ranks (and, with unshard_after,
    that many more after SetShard(None)). The denoiser (radius, num_passes), when given, is enabled before frame svgf_from.
    With `compare`, every sharded frame is held to an unsharded renderer. Returns each rank's (bytes, calls) of its comm over
    the sharded frames."""
    import torch
    from zetaray_b200.passes import SVGF
    from zetaray_b200.sharding import StripPlan
    from tests import scene_util
    from tests.test_display_oracle import load_lut
    world = len(bounds) - 1
    plan = StripPlan(H, bounds)
    flat = scene_util.SCENES[which]()
    lut = load_lut() if display else None
    fcs = _frame_constants(warm + frames + unshard_after)

    want = []
    if compare:
        ref = _renderer(flat, integrator, False, display, lut)
        s0 = torch.cuda.Stream()
        for f, fc in enumerate(fcs[:warm + frames]):
            if svgf and f == svgf_from:
                _denoise(ref, svgf)
            ref.Render(fc, C.c_void_p(s0.cuda_stream))
            torch.cuda.synchronize()
            want.append(_outputs(ref, display))

    ranks = [_renderer(flat, integrator, two_streams, display, lut) for _ in range(world)]
    shared, sums, barrier, errors = {}, {}, threading.Barrier(world), []
    transports = [ThreadTransport(r, world, shared, sums, barrier, errors) for r in range(world)]
    comms = [t.comm() for t in transports]
    traffic = [None] * world

    def rank_main(rank):
        R = ranks[rank]
        try:
            torch.cuda.set_device(0)
            st = torch.cuda.Stream()
            y0, y1 = plan.rows(rank)
            lone = None
            for f, fc in enumerate(fcs):
                if f == warm:       # unsharded warm-up frames (every rank has the full history), then cut
                    torch.cuda.synchronize()
                    R.SetShard(comms[rank], plan.bounds, gather_output=True)
                    start = comms[rank].stats()
                if svgf and f == svgf_from:
                    _denoise(R, svgf)
                if f == warm + frames:
                    end = comms[rank].stats()
                    traffic[rank] = (end[0] - start[0], end[1] - start[1])
                    # whole frames again: with its history reset, the denoiser equals a whole-frame pass fed the same frames
                    R.SetShard(None, None)
                    R.svgf.ResetTemporal()
                    lone = SVGF(W, H)
                    lone.SetParams(radius=svgf[0], num_passes=svgf[1])
                R.Render(fc, C.c_void_p(st.cuda_stream))
                torch.cuda.synchronize()
                if lone is not None:
                    lone.Render(_frame_inputs(R, fc), R.compositing.GetOutput().d_ptr)
                    torch.cuda.synchronize()
                    got, exp = _svgf_rows(R.svgf), _svgf_rows(lone)
                    for k in exp:
                        if not np.array_equal(got[k], exp[k]):
                            raise AssertionError("rank %d frame %d after SetShard(None): svgf %s is not the whole-frame pass's" % (rank, f, k))
                    continue
                if f < warm or not compare:
                    continue
                got = _outputs(R, display)
                assert got.keys() == want[f].keys(), (got.keys(), want[f].keys())
                for k in got:
                    bad = np.argwhere(got[k][y0:y1] != want[f][k][y0:y1])
                    if bad.size:
                        raise AssertionError("rank %d frame %d: %s differs, first at (row, byte) %s of strip [%d, %d)" % (
                            rank, f, k, (bad[0] + [y0, 0]).tolist(), y0, y1))
                for k in ("taa", "display") if rank == 0 else ():
                    if k in got and not np.array_equal(got[k], want[f][k]):
                        raise AssertionError("frame %d: %s image gathered on rank 0 differs" % (f, k))
            if traffic[rank] is None:
                end = comms[rank].stats()
                traffic[rank] = (end[0] - start[0], end[1] - start[1])
            elif comms[rank].stats()[1] != start[1] + traffic[rank][1]:
                raise AssertionError("rank %d: the comm was used after SetShard(None)" % rank)
        except BaseException as e:      # noqa: BLE001
            errors.append(e)
            barrier.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[0]
    return traffic


@pytest.mark.parametrize("which,integrator,bounds,two_streams,svgf,display", [
    ("glossy", "pt", [0, 96, 200], True, (2, 5), False),          # ReSTIR PT, 5x5 taps, 5 passes: the stage reaches 62 rows
    ("glossy", "pt", [0, 32, 128, 200], False, (1, 3), False),    # 3x3 taps, 3 passes; a one-band strip: its top and bottom bands coincide
    ("cornell", "gi", [0, 96, 200], False, (2, 5), True),         # ReSTIR GI; AutoExposure histograms the denoised strip
], ids=["pt-r2-5-passes", "pt-r1-one-band-strip", "gi-display"])
def test_svgf_sharded_threads_equal_unsharded(which, integrator, bounds, two_streams, svgf, display):
    _run_threads(which, integrator, bounds, two_streams, svgf, display)


def test_svgf_enabled_after_set_shard_then_unsharded():
    """zr_renderer_set_denoiser after zr_renderer_set_shard: the new pass takes the renderer's strip and hook, so the frames equal an
    unsharded renderer that enables the denoiser at the same frame; after SetShard(None) it denoises whole frames without the hook."""
    _run_threads("glossy", "pt", [0, 96, 200], False, (2, 5), svgf_from=3, unshard_after=2)


def test_svgf_band_traffic():
    """The comm's bytes per frame with the denoiser minus those without it are the SVGF bands: min(32, strip rows) rows per band,
    colour + variance, guide (8 B/px each) and history (16 B/px) at the padded pitch after the temporal stage, colour + variance after
    every a-trous pass but the last, the denoised image (16 B/px, unpadded) after the last."""
    from zetaray_b200.passes import SVGF
    bounds, frames, (radius, passes) = [0, 32, 128, 200], 3, (2, 5)
    plain = _run_threads("cornell", "pt", bounds, False, None, frames=frames, compare=False)
    denoised = _run_threads("cornell", "pt", bounds, False, (radius, passes), frames=frames, compare=False)
    pitch = SVGF(W, H).GetOutput(ZR_SVGF_GUIDE).pitch_bytes // 8
    per_row = pitch * (8 + 8 + 16) + (passes - 1) * pitch * 8 + W * 16
    for r in range(len(bounds) - 1):
        n_bands = (r > 0) + (r < len(bounds) - 2)
        rows = min(HALO, bounds[r + 1] - bounds[r])
        assert denoised[r][0] - plain[r][0] == frames * n_bands * rows * per_row, (r, plain[r], denoised[r])
        assert denoised[r][1] - plain[r][1] == frames * (passes + 1), (r, plain[r], denoised[r])
