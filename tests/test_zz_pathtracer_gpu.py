"""The plain path tracer (IndirectLighting, INTEGRATOR::PATH_TRACING; PathTracer/PathTracer.hlsl with PathTracer/Params.hlsli:
MIS next-event estimation at every bounce, exact shadow rays, Beer's law in translucent media) on the device vs the CPU
oracle, frame by frame, byte for byte -- stand-alone through zr_gi_pass_set_method and inside the native frame driver."""
import numpy as np
import pytest

from tests.parity import diff_report, frame_parity, rgba32f_bits, uint32x2

pytestmark = pytest.mark.gpu


def _run(which, w, h, nframes, **kw):
    return frame_parity(which, w, h, nframes, ("pt",), **kw)


@pytest.mark.parametrize("which", ["cornell", "glossy", "glass"])
def test_path_tracer_frames(which):
    problems, R = _run(which, 320, 180, 3)
    assert not problems, "\n".join(problems)
    assert (R.gi_final[:, :3].sum(axis=1) > 0).sum() > 5000


def test_path_tracer_variants():
    # translating camera, 6 bounces (the wave-wide Russian roulette runs), transmissive scene (Beer's law, exact shadow rays
    # through glass), accumulation mode, presampled sets
    path = lambda f: (0.03 * f, 1.2 + 0.01 * f, -4.043 + 0.04 * f)
    problems, _ = _run("glass", 256, 144, 3, gi_params=dict(max_non_tr_bounces=6, max_glossy_tr_bounces=6), cam_path=path)
    assert not problems, "\n".join(problems)
    problems, _ = _run("glossy", 256, 144, 3, accumulate=True, presample=(16, 64))
    assert not problems, "\n".join(problems)
    problems, _ = _run("tunnel", 160, 90, 2)
    assert not problems, "\n".join(problems)


def test_path_tracer_through_the_renderer_and_method_switch():
    from zetaray_b200 import lib, check
    from zetaray_b200.passes import Scene, Renderer
    from tests import scene_util, rpt_util
    w, h = 192, 108
    flat = scene_util.glossy_cornell()
    R = rpt_util.OracleRenderer(flat, w, h)
    sc = Scene(flat)
    rd = Renderer(sc, w, h)
    rd.SetMethod(Renderer.PATH_TRACING)
    seq = rpt_util.FrameSequence(w, h)
    taa_prev = np.zeros((w * h, 2), dtype=np.uint32)
    for fr in range(3):
        fc = seq.next()
        R.gbuffer(fc); R.rdi(fc); R.pt(fc)
        R.final = R.gi_final
        _, taa_prev = R.post(fc, taa_prev, fr > 0)
        rd.Render(fc)
        check(lib.zr_stream_synchronize(None))
        msg = diff_report("pt final", rgba32f_bits(rd.gi.GetOutput(0)), R.gi_final.view(np.uint32))
        assert not msg, "frame %d: %s" % (fr + 1, msg)
        msg = diff_report("taa", uint32x2(rd.GetOutput()), taa_prev)
        assert not msg, "frame %d: %s" % (fr + 1, msg)
    # switching to ReSTIR GI drops the history: its first frame equals the oracle's first GI frame on this G-buffer sequence
    rd.SetMethod(Renderer.RESTIR_GI)
    fc = seq.next()
    R.gbuffer(fc); R.rdi(fc); R.rgi(fc)
    rd.Render(fc)
    check(lib.zr_stream_synchronize(None))
    msg = diff_report("gi final after the switch", rgba32f_bits(rd.gi.GetOutput(0)), R.gi_final.view(np.uint32))
    assert not msg, msg
    assert lib.zr_gi_pass_set_method(rd.gi.handle, 2) != 0      # ReSTIR PT is a different pass object
