"""ReSTIR PT on the device vs the CPU oracle, frame by frame (bit-exact integer state AND radiance).

Covers: initial path generation (frame 1), temporal reuse (frame 2+), spatial search, the StC thread map,
CtS+StC spatial reuse with boiling suppression, ping-pong bookkeeping over several frames, on the
Cornell box (k == 2 everywhere) and on the glossy variant (k > 2 replay, case 3, metals, coat)."""
import ctypes as C
import numpy as np
import pytest

from tests.orc import ptr


def _diff_report(name, a, b, fields=None):
    if a.tobytes() == b.tobytes():
        return None
    av = a.reshape(len(a), -1) if a.dtype.fields is None else a
    if a.dtype.fields is not None:
        bad = {}
        for fld in a.dtype.names:
            n = int((a[fld] != b[fld]).sum())
            if n:
                bad[fld] = n
        first = int(np.nonzero(a != b)[0][0])
        return "%s differs: per-field mismatches %s; first idx %d got %s want %s" % (name, bad, first, a[first], b[first])
    d = np.nonzero((a.reshape(len(a), -1) != b.reshape(len(b), -1)).any(axis=1))[0]
    return "%s differs at %d/%d entries; first idx %d got %s want %s" % (name, len(d), len(a), d[0], a[d[0]], b[d[0]])


def _run(which, w, h, nframes, params=None, jitter=True, dof=False, dump=None, cam_path=None, accumulate=False, presample=None):
    import torch
    from zetaray_b200 import lib, check, _lib
    from zetaray_b200.passes import Scene, GBuffers, GBufferRT, IndirectLighting, download_image
    from tests import scene_util, rpt_util
    flat = scene_util.SCENES[which]()
    R = rpt_util.OracleRenderer(flat, w, h)
    sc = Scene(flat)
    sc.prelighting()
    if presample:
        R.osc.set_presampling(*presample)
        sc.set_presampling(*presample)
    gb = GBuffers(w, h)
    gpass = GBufferRT()
    ind = IndirectLighting(w, h)
    if params:
        for k, v in params.items():
            setattr(R.params, k, v)
        ind.SetParams(**params)
    seq = rpt_util.FrameSequence(w, h, jitter=jitter, cam_path=cam_path, accumulate=accumulate)
    problems = []
    for fr in range(nframes):
        fc = seq.next()
        if dof:
            fc.DoF, fc.FocusDepth, fc.LensRadius = 1, 4.0, 0.02
        R.gbuffer(fc)
        R.rpt(fc)
        gb.flip()
        fi = _lib.FrameInputs()
        fi.frame = fc
        gb.fill_inputs(fi)
        fi.scene = sc.handle
        gpass.Render(fi)
        sc.presample(fc.FrameNum)
        ind.Render(fi)
        check(lib.zr_stream_synchronize(None))
        if presample and fr == 0:
            assert sc.sample_sets().tobytes() == R.osc.sample_sets[:presample[0] * presample[1] * 10].tobytes(), "presampled sets differ"
        got_res = download_image(ind.GetOutput(1), np.uint8, 64).view(rpt_util.RES).reshape(-1)
        got_final = download_image(ind.GetOutput(0), np.float32, 4)
        checks = [("reservoir", got_res, R.curr_reservoirs()), ("final", got_final.view(np.uint32), R.final.view(np.uint32))]
        if fr >= 1 and R.params.num_spatial_passes > 0 and R.params.temporal_resample:
            checks.append(("neighbor", download_image(ind.GetOutput(4), np.uint16, 1).reshape(-1), R.neighbor))
            if R.params.sort_spatial:
                checks.append(("threadmap_ntc", download_image(ind.GetOutput(6), np.uint16, 1).reshape(-1), R.tmNtC))
        if fr >= 1 and R.params.temporal_resample:
            checks.append(("target", download_image(ind.GetOutput(3), np.float32, 4).view(np.uint32), R.target.view(np.uint32)))
        for name, a, b in checks:
            msg = _diff_report(name, a, b)
            if msg:
                problems.append("frame %d: %s" % (fc.FrameNum, msg))
        if problems:
            break
    gb.close()
    return problems, R


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["cornell", "glossy"])
def test_rpt_pathtrace_only(which):
    problems, _ = _run(which, 320, 180, 2, params=dict(temporal_resample=0, num_spatial_passes=0))
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["cornell", "glossy"])
def test_rpt_temporal_only(which):
    problems, _ = _run(which, 320, 180, 3, params=dict(num_spatial_passes=0))
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
    problems, _ = _run("glossy", 320, 180, 3, params=dict(sort_spatial=0, boiling_suppression=0, max_non_tr_bounces=5))
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
    problems, _ = _run("glass", 256, 144, 4, params=dict(max_non_tr_bounces=5, max_glossy_tr_bounces=6, num_spatial_passes=2))
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
    problems, _ = _run(which, w, h, nframes, params=params, cam_path=path)
    assert not problems, "\n".join(problems)


@pytest.mark.gpu
def test_rpt_accumulate_and_two_spatial_passes():
    problems, _ = _run("glossy", 256, 144, 4, accumulate=True)
    assert not problems, "\n".join(problems)
    problems, _ = _run("cornell", 256, 144, 4, params=dict(num_spatial_passes=2))
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
