"""SVGF on the device vs its oracle (oracle/orc_svgf.cpp), byte for byte: denoised image, history (colour, moments, history length),
guide planes -- 3x3 and 5x5 taps, every a-trous step incl. the strided-lattice TMA passes, odd resolutions, a moving camera (temporal
reprojection + rejection), and the bench resolution. The signal is the oracle's composited frame of the same sequence."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _run(which, w, h, nframes, radius=2, num_passes=5, cam_path=None, synthetic=False):
    import torch
    from zetaray_b200 import lib, check
    from zetaray_b200.passes import SVGF, download_image, download_image_pitched
    from tests import scene_util, rpt_util
    from tests.parity import DeviceFrame
    from tests.svgf_util import OracleSVGF
    flat = scene_util.SCENES[which]()
    R = rpt_util.OracleRenderer(flat, w, h)
    dev = DeviceFrame(flat, w, h, ())
    svgf = SVGF(w, h)
    svgf.SetParams(radius=radius, num_passes=num_passes)
    osv = OracleSVGF(w, h, radius=radius, num_passes=num_passes)
    seq = rpt_util.FrameSequence(w, h, cam_path=cam_path)
    rng = np.random.default_rng(11)
    taa_prev = np.zeros((w * h, 2), dtype=np.uint32)
    problems = []
    for fr in range(nframes):
        fc = seq.next()
        R.gbuffer(fc)
        if synthetic:
            signal = np.zeros((w * h, 4), dtype=np.float32)
            signal[:, :3] = (rng.random((w * h, 3)) * rng.choice([0.1, 1.0, 30.0], (w * h, 1))).astype(np.float32)
        else:
            R.rdi(fc); R.rpt(fc)
            signal, taa_prev = R.post(fc, taa_prev, fr > 0)
            signal = np.ascontiguousarray(signal, dtype=np.float32)
        core, _, me, _ = R.gb[R.cur][:4]
        want, want_acc = osv.render(fc, core, me, signal)
        fi = dev.render(fc)
        d_signal = torch.from_numpy(signal).cuda()
        torch.cuda.synchronize()
        svgf.Render(fi, d_signal.data_ptr())
        check(lib.zr_stream_synchronize(None))
        got = download_image(svgf.GetOutput(0), np.float32, 4)
        checks = [("denoised", got.view(np.uint32), want.view(np.uint32)),
                  ("guide", download_image_pitched(svgf.GetOutput(2), np.uint32, 2), osv.guide[osv.cur]),
                  ("history", download_image_pitched(svgf.GetOutput(3), np.uint32, 4), osv.hist[osv.cur])]
        if num_passes == 1:
            checks.append(("accumulated", download_image_pitched(svgf.GetOutput(1), np.uint32, 2), want_acc))
        for name, a, b in checks:
            if a.tobytes() != b.tobytes():
                d = np.nonzero((a != b).any(axis=1))[0]
                problems.append("frame %d: %s differs at %d/%d pixels; first %d (x %d, y %d) got %s want %s" %
                                (fc.FrameNum, name, len(d), len(a), d[0], d[0] % w, d[0] // w, a[d[0]], b[d[0]]))
        if problems:
            break
    dev.close()
    return problems


@pytest.mark.parametrize("radius", [1, 2])
def test_svgf_frames(radius):
    problems = _run("cornell", 320, 180, 3, radius=radius)
    assert not problems, "\n".join(problems)


def test_svgf_temporal_stage_and_single_steps():
    # one pass: the accumulated plane survives and is compared; 2..4 passes end on every lattice step as the LAST pass
    for n in (1, 2, 3, 4):
        problems = _run("glossy", 256, 144, 2, num_passes=n)
        assert not problems, "passes=%d\n%s" % (n, "\n".join(problems))


def test_svgf_odd_resolution_moving_camera_synthetic_signal():
    path = lambda f: (0.04 * f, 1.2 + 0.01 * f, -4.043 + 0.03 * f)
    problems = _run("glass", 333, 187, 4, cam_path=path, synthetic=True)
    assert not problems, "\n".join(problems)
    problems = _run("glossy", 333, 187, 3, radius=1, cam_path=path)
    assert not problems, "\n".join(problems)


def test_svgf_1080p():
    problems = _run("cornell", 1920, 1080, 2, synthetic=True)
    assert not problems, "\n".join(problems)


def test_svgf_rejects_bad_calls():
    import ctypes as C
    from zetaray_b200 import lib, _lib
    from zetaray_b200.passes import SVGF
    s = SVGF(64, 64)
    fi = _lib.FrameInputs()
    assert lib.zr_svgf_pass_render(s.handle, C.byref(fi), None, None) != 0
    p = _lib.SvgfParams()
    lib.zr_svgf_pass_default_params(C.byref(p))
    assert p.radius == 2 and p.num_passes == 5
    p.radius = 3
    assert lib.zr_svgf_pass_set_params(s.handle, C.byref(p)) != 0
