"""ReSTIR GI (IndirectLighting, INTEGRATOR::ReSTIR_GI, emissive NEE) on the device vs the CPU oracle, frame by frame:
48-byte reservoirs and the final image byte for byte. Covers the path-traced initial candidate (MIS NEE at the first
indirect vertex, light-sampled NEE after it), temporal reuse with one and two candidates, the reconnection Jacobian,
outlier suppression, the wave-wide Russian roulette (5+ bounces), presampled sets, a translating camera and DoF."""
import pytest

from tests.parity import frame_parity

pytestmark = pytest.mark.gpu


def _run(which, w, h, nframes, **kw):
    return frame_parity(which, w, h, nframes, ("rgi",), **kw)


@pytest.mark.parametrize("which", ["cornell", "glossy", "glass"])
def test_rgi_frames(which):
    problems, R = _run(which, 320, 180, 4)
    assert not problems, "\n".join(problems)
    res = R.gi_curr_reservoirs()
    assert (res["ID"] != 0xffffffff).sum() > 5000


def test_rgi_moving_camera_and_variants():
    path = lambda f: (0.03 * f, 1.2 + 0.01 * f, -4.043 + 0.04 * f)
    problems, _ = _run("glossy", 320, 180, 5, cam_path=path)
    assert not problems, "\n".join(problems)
    # deterministic bounce count, 6 bounces so the wave-wide Russian roulette runs, no outlier suppression
    problems, _ = _run("glass", 256, 144, 4, gi_params=dict(stochastic_multi_bounce=0, max_non_tr_bounces=6, max_glossy_tr_bounces=6,
                                                             boiling_suppression=0), cam_path=path)
    assert not problems, "\n".join(problems)
    problems, _ = _run("cornell", 256, 144, 3, gi_params=dict(temporal_resample=0, M_max=4))
    assert not problems, "\n".join(problems)


def test_rgi_presampled_sets_dof_accumulate():
    problems, _ = _run("glossy", 256, 144, 4, presample=(16, 64))
    assert not problems, "\n".join(problems)
    problems, _ = _run("glossy", 256, 144, 3, dof=True)
    assert not problems, "\n".join(problems)
    problems, _ = _run("cornell", 256, 144, 3, accumulate=True)
    assert not problems, "\n".join(problems)


def test_rgi_light_voxel_grid():
    # ReSTIR_GI_LVG: the NEE light sample after the first indirect vertex comes from the camera-centred voxel grid, with the
    # presampled set as fallback outside it. A small grid so that both branches run; then the reference's own dimensions.
    path = lambda f: (0.03 * f, 1.2, -4.043 + 0.04 * f)
    problems, _ = _run("glossy", 320, 180, 4, presample=(32, 128), lvg=((8, 4, 8), (0.6, 0.45, 0.6), 0.1), cam_path=path,
                       gi_params=dict(stochastic_multi_bounce=0))
    assert not problems, "\n".join(problems)
    problems, _ = _run("glass", 256, 144, 3, presample=(128, 512), lvg=((32, 8, 40), (0.6, 0.45, 0.6), 0.0))
    assert not problems, "\n".join(problems)


def test_rgi_rejects_bad_calls():
    from zetaray_b200 import lib, _lib
    from zetaray_b200.passes import IndirectLightingGI
    gi = IndirectLightingGI(64, 64)
    fi = _lib.FrameInputs()
    import ctypes as C
    assert lib.zr_gi_pass_render(gi.handle, C.byref(fi), None) != 0
    bad = _lib.GIParams(0, 4, 1, 1, 1, 10, 1)
    assert lib.zr_gi_pass_set_params(gi.handle, C.byref(bad)) != 0
