"""ReSTIR DI (emissive) and the whole reference-shaped frame on the device vs the CPU oracle (bit-exact)."""
import ctypes as C
import pytest

from tests.parity import WHOLE_FRAME, frame_parity


def _frame_loop(which, w, h, nframes, full=False, **kw):
    return frame_parity(which, w, h, nframes, WHOLE_FRAME if full else ("rdi",), **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["cornell", "glossy"])
def test_rdi_frames(which):
    problems, R = _frame_loop(which, 320, 180, 4)
    assert not problems, "\n".join(problems)
    assert (R.di_curr_reservoirs()["lightIdx"] != 0xffffffff).sum() > 1000


@pytest.mark.gpu
def test_rdi_variants():
    problems, _ = _frame_loop("glossy", 256, 144, 3, di_params=dict(spatial_resample=0))
    assert not problems, "\n".join(problems)
    problems, _ = _frame_loop("glossy", 256, 144, 3, di_params=dict(stochastic_spatial=0, extra_disocclusion_sampling=0, M_max=8))
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
@pytest.mark.parametrize("which,w,h", [("cornell", 480, 270), ("glossy", 333, 187)])
def test_full_frame_pipeline(which, w, h):
    # G-buffer -> pre-lighting -> ReSTIR DI -> ReSTIR PT -> compositing + firefly -> TAA, 4 frames
    problems, R = _frame_loop(which, w, h, 4, full=True)
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
def test_full_frame_pipeline_glass_moving_camera():
    # transmissive scene + translating camera through the whole frame (DI disocclusion vote, TAA history reprojection)
    path = lambda f: (0.04 * f, 1.2, -4.043 + 0.03 * f)
    problems, _ = _frame_loop("glass", 320, 180, 5, full=True, cam_path=path)
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
def test_full_frame_pipeline_accumulate():
    problems, _ = _frame_loop("glossy", 256, 144, 4, full=True, accumulate=True)
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
def test_presampled_sets_di_and_full_frame():
    problems, _ = _frame_loop("glossy", 320, 180, 4, presample=(16, 64))
    assert not problems, "\n".join(problems)
    problems, _ = _frame_loop("cornell", 333, 187, 4, full=True, presample=(128, 512))
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
def test_presampling_needs_the_presample_pass():
    from zetaray_b200 import lib, _lib
    from zetaray_b200.passes import Scene, GBuffers, GBufferRT, DirectLighting
    from tests import scene_util, rpt_util
    sc = Scene(scene_util.cornell())
    sc.prelighting()
    sc.set_presampling(4, 32)
    gb, g, di = GBuffers(64, 64), GBufferRT(), DirectLighting(64, 64)
    fi = _lib.FrameInputs()
    fi.scene = sc.handle
    fi.frame = rpt_util.FrameSequence(64, 64).next()
    gb.flip(); gb.fill_inputs(fi)
    g.Render(fi)
    assert lib.zr_direct_pass_render(di.handle, C.byref(fi), None) != 0      # presample pass has not run
    assert b"zr_presample_emissives" in lib.zr_last_error()
    sc.presample(1)
    di.Render(fi)
    assert lib.zr_scene_set_presampling(sc.handle, 4, 0) != 0
