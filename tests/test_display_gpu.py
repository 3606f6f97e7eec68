"""AutoExposure and Display (csrc/display.cu) against the CPU oracle (oracle/orc_display.cpp), bit for bit: the luminance
histogram, the exposure state over a frame sequence, the RGBA8 display image for every tone mapper; the renderer's optional
display stage; error paths; and a lone AutoExposure + Display pair in strip-sharded frames (threads on one GPU; the renderer's
display stage in sharded frames is tested with the rest of the frame in tests/test_sharded_1gpu.py and tests/test_sharded_gpu.py)."""
import ctypes as C

import numpy as np
import pytest

from tests.orc import ptr
from tests.sharded_util import ThreadTransport, compare_strip, host_rows, run_threads
from tests.test_display_oracle import load_lut, ae_params

pytestmark = pytest.mark.gpu

SIZES = [(7, 3), (64, 40), (257, 131), (1920, 1080), (2560, 1440), (3840, 2160)]


def _fi(w, h, dt=1 / 60):
    from zetaray_b200 import _lib
    from zetaray_b200.camera import look_at_frame_constants
    fi = _lib.FrameInputs()
    fi.frame = look_at_frame_constants(w, h)
    fi.frame.dt = dt
    return fi


def _signal(w, h, seed):
    """RGBA32F like the composited image: HDR colour, fireflies, black pixels (bin 0) and a few NaN / negative / huge ones."""
    from tests import synth
    rng = np.random.default_rng(seed)
    s = synth.synth_hdr(w, h, seed)
    n = w * h
    s[rng.integers(0, n, size=max(1, n // 20)), :3] = 0.0
    s[rng.integers(0, n, size=max(1, n // 97)), :3] *= np.float32(1e-3)
    s[rng.integers(0, n, size=max(1, n // 1000)), 0] = np.nan
    s[rng.integers(0, n, size=max(1, n // 1000)), 1] = -3.0
    s[rng.integers(0, n, size=max(1, n // 5000)), 2] = 1e6
    return s


def _taa_image(w, h, seed):
    """half4 like the TAA output, over the whole tone-mapping range, with a few inf / NaN / negative texels."""
    rng = np.random.default_rng(seed)
    n = w * h
    rgb = np.exp(rng.uniform(np.log(1e-4), np.log(300.0), size=(n, 3)))
    rgb[rng.integers(0, n, size=max(1, n // 50))] = 0.0
    img = np.zeros((n, 4), dtype=np.float16)
    img[:, :3] = rgb.astype(np.float16)
    img[rng.integers(0, n, size=max(1, n // 3000)), 0] = np.inf
    img[rng.integers(0, n, size=max(1, n // 3000)), 1] = np.nan
    img[rng.integers(0, n, size=max(1, n // 3000)), 2] = -0.5
    return img.view(np.uint16)


def _download(d_ptr, arr, stream=None):
    from zetaray_b200 import lib, check
    check(lib.zr_memcpy_d2h(ptr(arr), C.c_void_p(d_ptr), C.c_size_t(arr.nbytes), stream))
    check(lib.zr_stream_synchronize(stream))
    return arr


class BinTap:
    """Reduce hook that copies the histogram out between the two kernels and leaves it as it is."""

    def __init__(self, ae):
        from zetaray_b200 import _lib
        self.bins = None
        self.fn = _lib.REDUCE_U32_FN(self._hook)
        ae.SetReduce(self.fn)

    def _hook(self, user, d_values, n, stream):
        self.bins = _download(d_values, np.zeros(n, dtype=np.uint32), C.c_void_p(stream))


@pytest.mark.parametrize("w,h", SIZES)
def test_histogram_and_exposure_match_oracle(oracle, w, h):
    from zetaray_b200.passes import AutoExposure
    from tests.gpu_util import dev, stream
    ae = AutoExposure(w, h)
    tap = BinTap(ae)
    sig = _signal(w, h, 3)
    d_sig = dev(sig)
    p = ae_params()
    ae.Render(_fi(w, h), d_sig.data_ptr(), stream())
    got = _download(ae.GetOutput().d_ptr, np.zeros(2, dtype=np.float32))
    hist = np.zeros(256, dtype=np.uint32)
    oracle.orc_lum_histogram(ptr(sig), w, 0, h, C.byref(p), ptr(hist))
    assert hist.sum() == w * h and hist[0] > 0 and hist[1] > 0
    assert np.array_equal(tap.bins, hist)
    state = np.zeros(2, dtype=np.float32)
    oracle.orc_exposure(ptr(hist), w * h, C.byref(p), 1 / 60, ptr(state))
    assert got.tobytes() == state.tobytes(), (got, state)
    assert np.isfinite(state).all() and state[0] > 0


@pytest.mark.parametrize("w,h", [(257, 131), (1920, 1080)])
def test_exposure_sequence_and_reset(oracle, w, h):
    from zetaray_b200 import lib
    from zetaray_b200.passes import AutoExposure
    from tests.gpu_util import dev, stream
    ae = AutoExposure(w, h)
    tap = BinTap(ae)
    state = np.zeros(2, dtype=np.float32)
    steps = [(1 / 60, {}), (1 / 30, {}), (0.0, {}), (0.25, dict(min_lum=0.02, max_lum=9.0)), (1 / 144, dict(lum_map_exp=0.8, adaptation_rate=0.4))]
    for f, (dt, prm) in enumerate(steps):
        if prm:
            ae.SetParams(**prm)
        sig = _signal(w, h, 40 + f)
        ae.Render(_fi(w, h, dt), dev(sig).data_ptr(), stream())
        got = _download(ae.GetOutput().d_ptr, np.zeros(2, dtype=np.float32))
        hist = np.zeros(256, dtype=np.uint32)
        oracle.orc_lum_histogram(ptr(sig), w, 0, h, C.byref(ae.params), ptr(hist))
        assert np.array_equal(tap.bins, hist), "frame %d" % f
        oracle.orc_exposure(ptr(hist), w * h, C.byref(ae.params), dt, ptr(state))
        assert got.tobytes() == state.tobytes(), "frame %d: %s vs %s" % (f, got, state)
    ae.ResetTemporal()
    assert not _download(ae.GetOutput().d_ptr, np.zeros(2, dtype=np.float32)).any()
    sig = _signal(w, h, 60)
    d_sig = dev(sig)
    assert lib.zr_auto_exposure_pass_render(ae.handle, C.byref(_fi(w, h, 0.0)), C.c_void_p(d_sig.data_ptr()), stream()) == 1
    ae.Render(_fi(w, h, 0.5), d_sig.data_ptr(), stream())
    state = np.zeros(2, dtype=np.float32)
    hist = np.zeros(256, dtype=np.uint32)
    oracle.orc_lum_histogram(ptr(sig), w, 0, h, C.byref(ae.params), ptr(hist))
    oracle.orc_exposure(ptr(hist), w * h, C.byref(ae.params), 0.5, ptr(state))
    assert _download(ae.GetOutput().d_ptr, np.zeros(2, dtype=np.float32)).tobytes() == state.tobytes()


@pytest.mark.parametrize("w,h", SIZES)
def test_display_matches_oracle_every_tonemapper(oracle, w, h):
    from zetaray_b200.passes import Display
    from tests.gpu_util import dev, stream
    lut = load_lut()
    disp = Display(w, h)
    disp.SetLUT(lut)
    taa = _taa_image(w, h, 7)
    exposure = np.array([0.37, 1.0], dtype=np.float32)
    d_taa, d_exp = dev(taa), dev(exposure)
    fi = _fi(w, h)
    out = np.zeros(w * h, dtype=np.uint32)
    ref = np.zeros(w * h, dtype=np.uint32)
    for tm in range(6):
        for auto in (1, 0):
            sat, agx_exp = (1.25, 0.8) if tm in (Display.NEUTRAL, Display.AGX_CUSTOM) else (1.0, 1.0)
            disp.SetParams(tonemapper=tm, auto_exposure=auto, saturation=sat, agx_exp=agx_exp)
            disp.Render(fi, d_taa.data_ptr(), d_exp.data_ptr(), stream())
            img = disp.GetOutput()
            assert (img.width, img.height, img.pitch_bytes, img.texel_bytes) == (w, h, 4 * w, 4)
            _download(img.d_ptr, out)
            oracle.orc_display(ptr(taa), w, 0, h, C.byref(disp.params), ptr(exposure), ptr(lut), ptr(ref))
            bad = np.flatnonzero(out != ref)
            assert bad.size == 0, "tonemapper %d auto %d: pixel %d is %08x, oracle %08x" % (tm, auto, bad[0], out[bad[0]], ref[bad[0]])
            assert (out >> 24 == 255).all()
            assert len(np.unique(out & 0xff)) > min(50, w * h // 4)


def test_renderer_display_stage_on_cornell(oracle):
    """Enabling the stage leaves the TAA output byte-identical, and the display image is the oracle applied to the frame's own
    TAA input (exposure) and output (display), frame after frame."""
    from zetaray_b200 import lib, check, _lib
    from zetaray_b200.passes import Scene, Renderer
    from tests import scene_util, rpt_util
    w, h = 320, 180
    lut = load_lut()
    flat = scene_util.SCENES["cornell"]()
    plain = Renderer(Scene(flat), w, h, two_streams=False)
    R = Renderer(Scene(flat), w, h, two_streams=False)
    assert lib.zr_renderer_get_display_output(R.handle, C.byref(_lib.Image2D())) == 3
    R.SetDisplay(True, lut=lut)
    seq = rpt_util.FrameSequence(w, h, cam_path=lambda f: (0.02 * f, 1.2, -4.043))
    state = np.zeros(2, dtype=np.float32)
    for fr in range(4):
        fc = seq.next()
        fc.dt = 1 / 60 if fr != 2 else 0.0
        plain.Render(fc)
        R.Render(fc)
        check(lib.zr_stream_synchronize(None))
        taa = host_rows(R.GetOutput())
        assert taa.tobytes() == host_rows(plain.GetOutput()).tobytes(), "frame %d: TAA output changed" % fr
        comp = host_rows(R.compositing.GetOutput())
        hist = np.zeros(256, dtype=np.uint32)
        oracle.orc_lum_histogram(ptr(comp), w, 0, h, C.byref(R.auto_exposure.params), ptr(hist))
        oracle.orc_exposure(ptr(hist), w * h, C.byref(R.auto_exposure.params), fc.dt, ptr(state))
        got_state = _download(R.auto_exposure.GetOutput().d_ptr, np.zeros(2, dtype=np.float32))
        assert got_state.tobytes() == state.tobytes(), "frame %d: %s vs %s" % (fr, got_state, state)
        ref = np.zeros(w * h, dtype=np.uint32)
        oracle.orc_display(ptr(taa), w, 0, h, C.byref(R.display.params), ptr(state), ptr(lut), ptr(ref))
        got = host_rows(R.GetDisplayOutput()).view(np.uint32).reshape(-1)
        assert got.tobytes() == ref.tobytes(), "frame %d: display image differs from the oracle" % fr
    assert len(np.unique(got & 0xffffff)) > 100
    R.SetDisplay(False)
    assert lib.zr_renderer_get_display_output(R.handle, C.byref(_lib.Image2D())) == 3
    R.close()
    plain.close()


def test_errors_and_resize():
    from zetaray_b200 import lib, _lib
    from zetaray_b200.passes import AutoExposure, Display
    from tests.gpu_util import dev, stream
    w, h = 96, 64
    ae = AutoExposure(w, h)
    d_sig = dev(_signal(w, h, 1))
    sig = C.c_void_p(d_sig.data_ptr())

    def ae_render(dt, fi=None):
        return lib.zr_auto_exposure_pass_render(ae.handle, C.byref(fi or _fi(w, h, dt)), sig, stream())

    for dt in (float("nan"), float("inf"), -1e-3, 0.0):
        assert ae_render(dt) == 1, dt
        assert b"dt" in lib.zr_last_error()
    assert ae_render(1 / 60) == 0
    assert ae_render(0.0) == 0              # adaptation freezes after the first frame
    assert ae_render(-1.0) == 1
    assert ae_render(1 / 60, _fi(w + 1, h)) == 1                    # frame size differs from the pass
    for bad in (dict(min_lum=-1.0), dict(max_lum=5e-3), dict(max_lum=1e-3), dict(lum_map_exp=0.0), dict(lum_map_exp=-1.0),
                dict(lum_map_exp=float("nan")), dict(max_lum=float("inf")), dict(adaptation_rate=float("nan"))):
        p = _lib.AutoExposureParams.from_buffer_copy(ae.params)
        for k, v in bad.items():
            setattr(p, k, v)
        assert lib.zr_auto_exposure_pass_set_params(ae.handle, C.byref(p)) == 1, bad
    # resize: new size, state back to {0, 0}, dt == 0 rejected again
    ae.OnWindowResized(2 * w, h)
    assert not _download(ae.GetOutput().d_ptr, np.zeros(2, dtype=np.float32)).any()
    d_big = dev(_signal(2 * w, h, 2))
    assert lib.zr_auto_exposure_pass_render(ae.handle, C.byref(_fi(2 * w, h, 0.0)), C.c_void_p(d_big.data_ptr()), stream()) == 1
    assert lib.zr_auto_exposure_pass_render(ae.handle, C.byref(_fi(2 * w, h)), C.c_void_p(d_big.data_ptr()), stream()) == 0

    disp = Display(w, h)
    d_taa = dev(_taa_image(w, h, 3))
    d_exp = dev(np.array([1.0, 1.0], dtype=np.float32))

    def disp_render(fi=None, exposure=d_exp):
        return lib.zr_display_pass_render(disp.handle, C.byref(fi or _fi(w, h)), C.c_void_p(d_taa.data_ptr()),
                                          C.c_void_p(exposure.data_ptr() if exposure is not None else None), stream())

    assert disp.params.tonemapper == Display.NEUTRAL and disp.params.auto_exposure == 1
    assert disp_render() == 1 and b"LUT" in lib.zr_last_error()          # NEUTRAL without the LUT
    lut = load_lut()
    assert lib.zr_display_pass_set_lut(disp.handle, ptr(lut), C.c_uint32(47)) == 1
    assert lib.zr_display_pass_set_lut(disp.handle, None, C.c_uint32(48)) == 1
    disp.SetLUT(lut)
    assert disp_render() == 0
    assert disp_render(exposure=None) == 1                                # auto exposure on, no state
    fi = _fi(w, h)
    fi.frame.DisplayWidth = 2 * w
    assert disp_render(fi) == 1 and b"display size" in lib.zr_last_error()
    assert disp_render(_fi(w, h + 1)) == 1
    for bad in (dict(tonemapper=6), dict(saturation=float("nan")), dict(agx_exp=float("inf"))):
        p = _lib.DisplayParams.from_buffer_copy(disp.params)
        for k, v in bad.items():
            setattr(p, k, v)
        assert lib.zr_display_pass_set_params(disp.handle, C.byref(p)) == 1, bad
    disp.SetParams(auto_exposure=0)
    assert disp_render(exposure=None) == 0
    disp.OnWindowResized(w // 2, h)
    img = disp.GetOutput()
    assert (img.width, img.height, img.pitch_bytes) == (w // 2, h, 2 * w)
    assert disp_render(_fi(w // 2, h)) == 0                               # the LUT survives a resize


@pytest.mark.parametrize("bounds", [[0, 96, 200], [0, 64, 128, 200]])
def test_sharded_threads_equal_unsharded(bounds):
    """AutoExposure and Display over each rank's rows, the histogram summed over the ranks: every rank's exposure and its rows of
    the display image equal the whole-frame passes'."""
    import torch
    from zetaray_b200.passes import AutoExposure, Display
    from tests.gpu_util import dev
    W, H = 288, 200
    world = len(bounds) - 1
    lut = load_lut()
    sigs = [_signal(W, H, 70 + f) for f in range(3)]
    taas = [_taa_image(W, H, 80 + f) for f in range(3)]
    d_sigs, d_taas = [dev(s) for s in sigs], [dev(t) for t in taas]

    def passes():
        ae, disp = AutoExposure(W, H), Display(W, H)
        disp.SetLUT(lut)
        return ae, disp

    def render(ae, disp, f, stream):
        fi = _fi(W, H, 1 / 60 + f * 0.01)
        ae.Render(fi, d_sigs[f].data_ptr(), C.c_void_p(stream.cuda_stream))
        disp.Render(fi, d_taas[f].data_ptr(), ae.GetOutput().d_ptr, C.c_void_p(stream.cuda_stream))
        torch.cuda.synchronize()
        return {"exposure": host_rows(ae.GetOutput()), "display": host_rows(disp.GetOutput())}

    ae, disp = passes()
    s0 = torch.cuda.Stream()
    want = [render(ae, disp, f, s0) for f in range(3)]
    transports = ThreadTransport.group(world)

    def rank_main(rank):
        ae, disp = passes()
        y0, y1 = bounds[rank], bounds[rank + 1]
        ae.SetRows(y0, y1)
        disp.SetRows(y0, y1)
        ae.SetReduce(transports[rank].reduce_fn())
        st = torch.cuda.Stream()
        for f in range(3):
            compare_strip(render(ae, disp, f, st), want[f], y0, y1, "rank %d frame %d" % (rank, f))
        assert transports[rank].reductions == 3

    run_threads(transports, rank_main)
