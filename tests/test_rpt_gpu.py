"""ReSTIR PT on the device vs the CPU oracle, frame by frame (bit-exact integer state AND radiance).

Covers: initial path generation (frame 1), temporal reuse (frame 2+), spatial search, the StC thread map,
CtS+StC spatial reuse with boiling suppression, ping-pong bookkeeping over several frames, on the
Cornell box (k == 2 everywhere) and on the glossy variant (k > 2 replay, case 3, metals, coat)."""
import ctypes as C
import pytest

from tests.parity import frame_parity


def _run(which, w, h, nframes, **kw):
    return frame_parity(which, w, h, nframes, ("rpt",), **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["cornell", "glossy"])
def test_rpt_pathtrace_only(which):
    problems, _ = _run(which, 320, 180, 2, rpt_params=dict(temporal_resample=0, num_spatial_passes=0))
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["cornell", "glossy"])
def test_rpt_temporal_only(which):
    problems, _ = _run(which, 320, 180, 3, rpt_params=dict(num_spatial_passes=0))
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
@pytest.mark.parametrize("which,w,h", [("cornell", 320, 180), ("glossy", 320, 180), ("glossy", 333, 187)])
def test_rpt_full_frames(which, w, h):
    problems, R = _run(which, w, h, 4)
    assert not problems, "\n".join(problems)
    res = R.curr_reservoirs()
    k = res["meta"] & 0xf
    assert (k == 0).sum() > 0
    if which == "glossy":
        assert ((k > 0) & (k < 15)).sum() > 0, "glossy scene must exercise k > 2 replay"


@pytest.mark.gpu
def test_rpt_variants():
    # no sorting, no boiling suppression, 5 bounces with Russian roulette, DoF camera
    problems, _ = _run("glossy", 320, 180, 3, rpt_params=dict(sort_spatial=0, boiling_suppression=0, max_non_tr_bounces=5))
    assert not problems, "\n".join(problems)
    problems, _ = _run("glossy", 256, 144, 3, dof=True)
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
def test_rpt_glass_scene():
    # specular + rough transmission, in-medium extinction, thin-walled translucency; 4 transmissive bounces so the
    # wave-wide Russian roulette (bounce >= 3) runs; then the same with 5/6 bounces and two spatial passes
    problems, R = _run("glass", 320, 180, 4)
    assert not problems, "\n".join(problems)
    k = R.curr_reservoirs()["meta"] & 0xf
    assert ((k > 0) & (k < 15)).sum() > 0, "glass scene must exercise k > 2 replay"
    problems, _ = _run("glass", 256, 144, 4, rpt_params=dict(max_non_tr_bounces=5, max_glossy_tr_bounces=6, num_spatial_passes=2))
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
@pytest.mark.parametrize("which,w,h,nframes,params", [
    pytest.param("glossy", 320, 180, 5, None, id="glossy"),
    pytest.param("glass", 320, 180, 5, None, id="glass"),
    # odd size: partial 16x8 groups and 32x32 sort tiles at the right and bottom edges
    pytest.param("glossy", 333, 187, 3, None, id="glossy-333-187"),
    # 6 bounces so that the wave-wide Russian roulette runs on long transmissive paths, two spatial passes
    pytest.param("glass", 256, 144, 4, dict(max_non_tr_bounces=5, max_glossy_tr_bounces=6, num_spatial_passes=2), id="glass-6-bounces"),
])
def test_rpt_moving_camera(which, w, h, nframes, params):
    # a translating camera: non-zero motion vectors, reprojection into other pixels, disocclusions at the box edges
    path = lambda f: (0.03 * f, 1.2 + 0.02 * f, -4.043 + 0.05 * f)
    problems, _ = _run(which, w, h, nframes, rpt_params=params, cam_path=path)
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
def test_rpt_accumulate_and_two_spatial_passes():
    problems, _ = _run("glossy", 256, 144, 4, accumulate=True)
    assert not problems, "\n".join(problems)
    problems, _ = _run("cornell", 256, 144, 4, rpt_params=dict(num_spatial_passes=2))
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
def test_rpt_presampled_sets():
    # the *_WPS shader variants: lights come from per-group presampled sets (PresampleEmissives.hlsl); small sets so that
    # several groups share a set and a set holds repeated lights
    problems, _ = _run("glossy", 320, 180, 4, presample=(16, 64))
    assert not problems, "\n".join(problems)
    problems, _ = _run("glass", 256, 144, 3, presample=(128, 512))
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
def test_indirect_rejects_bad_calls():
    from zetaray_b200 import lib, _lib
    from zetaray_b200.passes import IndirectLighting
    ind = IndirectLighting(64, 64)
    fi = _lib.FrameInputs()
    assert lib.zr_indirect_pass_render(ind.handle, C.byref(fi), None) != 0
    p = _lib.IndirectParams()
    lib.zr_indirect_pass_default_params(C.byref(p))
    assert p.max_non_tr_bounces == 3 and p.M_max_temporal == 10 and p.M_max_spatial == 8
    p.M_max_temporal = 99
    assert lib.zr_indirect_pass_set_params(ind.handle, C.byref(p)) != 0
