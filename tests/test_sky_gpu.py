"""The sky on the device, byte for byte against the oracle (oracle/sky): the LUT under several suns, atmospheres and sizes; the
background compositing writes in frames that do not accumulate (firefly filter on and off, emissive_di on and off, the sun in view,
a moving camera); the background DirectLighting accumulates (jittered silhouettes over 8 frames); whole renderer frames with SVGF
and the display stage on one and two streams; strip-sharded frames; and a sky that is off: its refusals, launches and outputs."""
import ctypes as C

import numpy as np
import pytest

from tests import orc, scene_util, sky_util
from tests.orc import ptr
from tests.parity import DeviceFrame, rgba32f_bits
from tests.sky_util import frame, oracle, oracle_lut
from zetaray_b200 import _lib, check, lib
from zetaray_b200.camera import FrameSequence
from zetaray_b200.passes import Compositing, DirectLighting, Renderer, Scene, SkyPass, download_image

pytestmark = pytest.mark.gpu

W, H = 192, 108
SUN_IN_VIEW = (0.0, -0.3, -1.0)
MOVING = lambda f: (0.03 * f, 1.2 + 0.02 * f, -4.043 + 0.05 * f)


def _sync():
    check(lib.zr_stream_synchronize(None))


def _inputs(fc):
    fi = _lib.FrameInputs()
    fi.frame = fc
    return fi


def device_lut(fc, w=sky_util.LUT_W, h=sky_util.LUT_H):
    p = SkyPass(w, h)
    p.Render(_inputs(fc))
    _sync()
    return download_image(p.GetOutput(), np.uint32, 1).reshape(-1)


LUT_CASES = {
    "default": dict(),
    "sun-ahead": dict(sun=SUN_IN_VIEW),
    "sun-overhead": dict(sun=(0.1, -1.0, 0.2)),
    "sun-below-horizon": dict(sun=(0.3, 0.2, 0.9)),
    "haze": dict(sun=(0.5, -0.6, 0.4), g=0.6, MieSigmaS=0.02, MieSigmaA=0.01, RayleighSigmaSScale=0.05,
                 RayleighSigmaSColor=(0.2, 0.5, 0.84)),
}


@pytest.mark.parametrize("case", list(LUT_CASES))
def test_lut_matches_oracle(case):
    fc = frame(16, 16, **LUT_CASES[case])
    assert np.array_equal(device_lut(fc), oracle_lut(fc))


@pytest.mark.parametrize("size", [(64, 32), (255, 127)])
def test_lut_sizes_match_oracle(size):
    fc = frame(16, 16, sun=SUN_IN_VIEW)
    assert np.array_equal(device_lut(fc, *size), oracle_lut(fc, *size))


def test_refusals():
    with pytest.raises(Exception):
        SkyPass(0, 128)
    with pytest.raises(Exception):
        SkyPass(256, 0)
    assert lib.zr_sky_pass_create(256, 128, None) != 0
    assert lib.zr_sky_pass_render(None, None, None) != 0
    p = SkyPass(32, 16)
    assert lib.zr_sky_pass_render(p.handle, None, None) != 0
    for field, v in (("PlanetRadius", 0.0), ("PlanetRadius", -1.0), ("AtmosphereAltitude", 0.0), ("g", float("nan")),
                     ("SunIlluminance", float("inf")), ("MieSigmaS", float("nan"))):
        fc = frame(16, 16, **{field: v})
        assert lib.zr_sky_pass_render(p.handle, C.byref(_inputs(fc)), None) == 1, field
    good = p.GetOutput()
    bad = [_lib.Image2D(None, 32, 16, 128, 4), _lib.Image2D(good.d_ptr, 0, 16, 0, 4), _lib.Image2D(good.d_ptr, 32, 0, 128, 4),
           _lib.Image2D(good.d_ptr, 32, 16, 128, 8), _lib.Image2D(good.d_ptr, 32, 16, 256, 4)]
    comp, di = Compositing(16, 16), DirectLighting(16, 16)
    for img in bad:
        assert lib.zr_compositing_pass_set_sky(comp.handle, C.byref(img)) == 1
        assert lib.zr_direct_pass_set_sky(di.handle, C.byref(img)) == 1
    assert lib.zr_compositing_pass_set_sky(None, C.byref(good)) == 1 and lib.zr_direct_pass_set_sky(None, C.byref(good)) == 1
    comp.SetSky(good); di.SetSky(good); comp.SetSky(None); di.SetSky(None)
    assert lib.zr_renderer_set_sky(None, 1, None) == 1
    out = (C.c_int32 * 2)()
    n = C.c_int()
    check(lib.zr_sky_pass_describe_io(p.handle, out, C.byref(n)))
    assert n.value == 1 and list(out) == [9, 1]


def _composite_oracle(fc, core, di, pt, lut, emissive_di, firefly):
    o = orc.load()
    n = fc.RenderWidth * fc.RenderHeight
    comp = np.zeros((n, 4), dtype=np.float32)
    o.orc_compositing(C.byref(fc), ptr(core), ptr(di) if emissive_di else None, ptr(pt), ptr(comp))
    oracle().sky_composite(C.byref(fc), ptr(core), ptr(lut), sky_util.LUT_W, sky_util.LUT_H, emissive_di, ptr(comp))
    if not firefly:
        return comp
    out = np.zeros_like(comp)
    o.orc_firefly(C.byref(fc), ptr(core), ptr(comp), ptr(out))
    return out


@pytest.mark.parametrize("firefly", [1, 0])
@pytest.mark.parametrize("emissive_di", [1, 0])
@pytest.mark.parametrize("sun,cam_path", [(None, None), (SUN_IN_VIEW, None), (SUN_IN_VIEW, MOVING)], ids=["default", "sun", "moving"])
def test_compositing_matches_oracle(firefly, emissive_di, sun, cam_path):
    f = DeviceFrame(scene_util.SCENES["cornell"](), W, H, ("rdi", "rpt", "post"))
    sky = SkyPass(sky_util.LUT_W, sky_util.LUT_H)
    f.comp.SetParams(emissive_di=emissive_di, indirect=1, firefly_filter=firefly)
    f.comp.SetSky(sky.GetOutput())
    seq = FrameSequence(W, H, cam_path=cam_path)
    invalid_seen = sun_seen = 0
    try:
        for _ in range(3):
            fc = seq.next()
            if sun is not None:
                s = np.asarray(sun) / np.linalg.norm(sun)
                fc.SunDir[0], fc.SunDir[1], fc.SunDir[2] = (float(v) for v in s.astype(np.float32))
                fc.SunCosAngularRadius, fc.SunSinAngularRadius = float(np.float32(np.cos(0.05))), float(np.float32(np.sin(0.05)))
            sky.Render(_inputs(fc))
            fi = f.render(fc)
            lut = download_image(sky.GetOutput(), np.uint32, 1).reshape(-1)
            core = rgba32f_bits(_lib.Image2D(fi.curr.d_core, W, H, W * 16, 16))
            di, pt = rgba32f_bits(f.di.GetOutput(0)), rgba32f_bits(f.rpt.GetOutput(0))
            want = _composite_oracle(fc, core, di, pt, lut, emissive_di, firefly)
            got = rgba32f_bits(f.comp.GetOutput())
            assert np.array_equal(got, want.view(np.uint32)), "frame %d: %d pixels differ" % (fc.FrameNum, (got != want.view(np.uint32)).any(axis=1).sum())
            invalid = (core[:, 3] & 4) != 0
            invalid_seen = max(invalid_seen, int(invalid.sum()))
            _, sunmask = sky_util.oracle_background(fc, lut)
            sun_seen = max(sun_seen, int((sunmask & invalid).sum()))
    finally:
        f.close()
    assert invalid_seen > 0
    assert sun is None or sun_seen > 0


def _copy_final(src, dst):
    """DirectLighting dst's FINAL := src's (device to device through the host)."""
    a, b = src.GetOutput(0), dst.GetOutput(0)
    host = rgba32f_bits(a)
    check(lib.zr_memcpy_h2d(b.d_ptr, host.ctypes.data_as(C.c_void_p), host.nbytes, None))
    _sync()


@pytest.mark.parametrize("scene", ["glossy", "cornell"])
def test_accumulating_frames_match_oracle(scene):
    """8 accumulating jittered frames. The sky-on pass's FINAL equals, at pixels with geometry, a sky-off pass that starts each frame
    from the sky-on pass's FINAL (so silhouette pixels that were sky last frame are covered), and at pixels without geometry the
    oracle's write from the FINAL before the frame."""
    f = DeviceFrame(scene_util.SCENES[scene](), W, H, ("rdi",))
    twin = DirectLighting(W, H)
    sky = SkyPass(sky_util.LUT_W, sky_util.LUT_H)
    f.di.SetSky(sky.GetOutput())
    seq = FrameSequence(W, H, accumulate=True)
    flips = np.zeros(W * H, dtype=bool)
    last_invalid = None
    try:
        for _ in range(8):
            fc = seq.next()
            before = rgba32f_bits(f.di.GetOutput(0)).copy()
            _copy_final(f.di, twin)
            sky.Render(_inputs(fc))
            fi = f.render(fc)
            twin.Render(fi)
            _sync()
            core = rgba32f_bits(_lib.Image2D(fi.curr.d_core, W, H, W * 16, 16))
            invalid = (core[:, 3] & 4) != 0
            got, other = rgba32f_bits(f.di.GetOutput(0)), rgba32f_bits(twin.GetOutput(0))
            assert np.array_equal(got[~invalid], other[~invalid]), "frame %d: pixels with geometry differ" % fc.FrameNum
            lut = download_image(sky.GetOutput(), np.uint32, 1).reshape(-1)
            want = other.view(np.float32).copy()
            oracle().sky_di_accumulate(C.byref(fc), ptr(core), ptr(lut), sky_util.LUT_W, sky_util.LUT_H, ptr(before), ptr(want))
            assert np.array_equal(got, want.view(np.uint32)), "frame %d: sky pixels differ" % fc.FrameNum
            if last_invalid is not None:
                flips |= invalid != last_invalid
            last_invalid = invalid
    finally:
        f.close()
    assert last_invalid.sum() > 0 and flips.sum() > 0, "no sky pixels or no silhouette pixels under jitter"


def _renderer_frames(two_streams, sky_schedule, n=4, setup=None):
    """Renders n frames of the Cornell scene with SVGF and the display stage on; sky_schedule[i] is the SetSky value before frame i
    (None: no call), setup(R) runs before the first frame. Returns per frame (fc, composited bits, TAA bits, display bits,
    launches) and the renderer."""
    from tests.test_display_oracle import load_lut
    R = Renderer(Scene(scene_util.SCENES["cornell"]()), W, H, two_streams=two_streams)
    R.SetDenoiser(True)
    R.SetDisplay(True, lut=load_lut())
    if setup:
        setup(R)
    seq = FrameSequence(W, H)
    out = []
    for i in range(n):
        if sky_schedule[i] is not None:
            R.SetSky(sky_schedule[i])
        fc = seq.next()
        fc.dt = 1 / 60
        _sync()
        l0 = lib.zr_kernel_launch_count()
        R.Render(fc)
        _sync()
        launches = lib.zr_kernel_launch_count() - l0
        out.append((fc, rgba32f_bits(R.compositing.GetOutput()).copy(), download_image(R.GetOutput(), np.uint32, 2).copy(),
                    download_image(R.GetDisplayOutput(), np.uint32, 1).copy(), launches))
    return out, R


def test_renderer_sky_off_is_unchanged_and_can_be_turned_off_again():
    plain, _ = _renderer_frames(True, [None] * 4)
    # on for one frame: one more launch (k_sky_view_lut) in that frame only
    toggled, R = _renderer_frames(True, [True, False, None, None])
    assert [b[4] - a[4] for a, b in zip(plain, toggled)] == [1, 0, 0, 0]
    assert R.sky is None and lib.zr_renderer_set_sky(R.handle, 0, None) == 0
    # enabled and disabled before the first frame: the frames of a renderer that never enabled it, byte for byte
    def on_off(R):
        R.SetSky(True)
        assert R.sky is not None
        R.SetSky(False)
    again, _ = _renderer_frames(True, [None] * 4, setup=on_off)
    for a, b in zip(plain, again):
        assert a[4] == b[4] and all(np.array_equal(x, y) for x, y in zip(a[1:4], b[1:4]))


@pytest.mark.parametrize("two_streams", [0, 1])
def test_renderer_frames_match_oracle(two_streams):
    frames, R = _renderer_frames(two_streams, [True, None, None, None])
    _sync()
    for fc, comp, taa, shown, _ in frames[-1:]:
        lut = download_image(R.sky.GetOutput(), np.uint32, 1).reshape(-1)
        assert np.array_equal(lut, oracle_lut(fc))
        fi = _lib.FrameInputs()
        check(lib.zr_renderer_get_gbuffer(R.handle, 0, C.byref(fi.curr)))
        core = rgba32f_bits(_lib.Image2D(fi.curr.d_core, W, H, W * 16, 16))
        di, pt = rgba32f_bits(R.direct.GetOutput(0)), rgba32f_bits(R.indirect.GetOutput(0))
        want = _composite_oracle(fc, core, di, pt, lut, 1, 1)
        assert np.array_equal(comp, want.view(np.uint32))
        invalid = (core[:, 3] & 4) != 0
        print("sky pixels in the %d x %d frame: %d" % (W, H, int(invalid.sum())))
        assert invalid.sum() > 0 and (comp.view(np.float32)[invalid, :3] > 0).any()
    other, _ = _renderer_frames(1 - two_streams, [True, None, None, None])
    for a, b in zip(frames, other):
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])


def test_default_view_background_pixel_count_at_1080p():
    """How much of the benchmark's 1080p Cornell frame shows the background (the pixels the sky changes)."""
    R = Renderer(Scene(scene_util.SCENES["cornell"]()), 1920, 1080, two_streams=True)
    R.SetSky(True)
    fc = FrameSequence(1920, 1080).next()
    R.Render(fc)
    _sync()
    fi = _lib.FrameInputs()
    check(lib.zr_renderer_get_gbuffer(R.handle, 0, C.byref(fi.curr)))
    core = rgba32f_bits(_lib.Image2D(fi.curr.d_core, 1920, 1080, 1920 * 16, 16))
    n = int(((core[:, 3] & 4) != 0).sum())
    print("invalid pixels in the default 1080p Cornell view: %d of %d" % (n, 1920 * 1080))
    comp = rgba32f_bits(R.compositing.GetOutput()).view(np.float32)
    assert (comp[(core[:, 3] & 4) != 0, :3] > 0).all() if n else True


def test_sharded_threads_equal_unsharded():
    import torch
    from tests.sharded_util import ThreadTransport, compare_strip, renderer_planes, run_threads
    from zetaray_b200.sharding import StripPlan
    w, h, bounds = 128, 200, [0, 96, 200]
    flat = scene_util.SCENES["glossy"]()
    seq = FrameSequence(w, h, cam_path=lambda f: (0.02 * f, 1.2, -4.043))
    fcs = [seq.next() for _ in range(5)]
    ref = Renderer(Scene(flat), w, h, two_streams=False)
    ref.SetSky(True)
    want = []
    for fc in fcs:
        ref.Render(fc)
        torch.cuda.synchronize()
        want.append(renderer_planes(ref, "pt"))
    plan = StripPlan(h, bounds)
    ranks = [Renderer(Scene(flat), w, h, two_streams=True) for _ in range(2)]
    transports = ThreadTransport.group(2)
    comms = [t.comm() for t in transports]

    def rank_main(rank):
        R = ranks[rank]
        R.SetSky(True)
        st = torch.cuda.Stream()
        y0, y1 = plan.rows(rank)
        for f, fc in enumerate(fcs):
            if f == 2:
                torch.cuda.synchronize()
                R.SetShard(comms[rank], plan.bounds, gather_output=True)
            R.Render(fc, C.c_void_p(st.cuda_stream))
            torch.cuda.synchronize()
            if f >= 2:
                compare_strip(renderer_planes(R, "pt"), want[f], y0, y1, "rank %d frame %d" % (rank, f), gathered=rank == 0)
        # every rank computes the whole LUT
        assert np.array_equal(download_image(R.sky.GetOutput(), np.uint32, 1), download_image(ref.sky.GetOutput(), np.uint32, 1))

    run_threads(transports, rank_main)
