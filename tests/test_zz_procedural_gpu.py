"""The procedural stand-ins for BASELINE.json's configs C4 ("Sponza-class" atrium: ReSTIR GI + light voxel grid, >= 13107
emissive triangles) and C5 ("Subway-class" tunnel: ReSTIR PT, 5 bounces, glass + glossy metal) on the device vs the CPU oracle,
bit for bit, at sizes the oracle's brute-force ray queries finish in seconds -- and, at the benchmark's full sizes
(3 x 10^5 / 10^6 triangles), the product's BVH kernels against the oracle's brute force on sampled rays.

Unlike the Cornell variants these scenes have hundreds of mesh instances with rotations and non-uniform scales, shared
vertex ranges (instancing), 19-25 materials, curved geometry with interpolated normals, and thousands of lights."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.parity import GBUFFER_CHECKS, WHOLE_FRAME, diff_report, frame_parity, gi_reservoirs, rgba32f_bits, uint32x2

pytestmark = pytest.mark.gpu
NTHREADS = min(os.cpu_count() or 8, 64)


def _setup(which, w, h):
    from zetaray_b200.passes import Scene
    from tests import scene_util, rpt_util
    flat = scene_util.SCENES[which]()
    R = rpt_util.OracleRenderer(flat, w, h, nthreads=NTHREADS)
    sc = Scene(flat)
    cam = scene_util.CAMERAS[which]
    return flat, R, sc, cam


def _frames(which, w, h, nframes, **kw):
    """Whole frame, pass by pass: G-buffer, ReSTIR DI, ReSTIR PT, compositing + firefly, TAA."""
    checks = GBUFFER_CHECKS + ("di_reservoir", "di_final", "pt_reservoir", "pt_final", "composited", "taa")
    return frame_parity(which, w, h, nframes, WHOLE_FRAME, checks, nthreads=NTHREADS, **kw)


def test_atrium_whole_frame():
    problems, R = _frames("atrium", 240, 135, 3)
    assert not problems, "\n".join(problems)
    res = R.curr_reservoirs()
    k = res["meta"] & 0xf
    assert (k == 0).sum() > 0 and ((k > 0) & (k < 15)).sum() > 0       # coated floor / metals: k > 2 reconnections occur
    assert (R.di_curr_reservoirs()["lightIdx"] != 0xffffffff).sum() > 2000
    assert len(np.unique(R.di_curr_reservoirs()["lightIdx"])) > 50      # many different lights win, not one quad


def test_tunnel_five_bounces_two_spatial_passes_moving_camera():
    """Config C5's parameters: 5 non-transmissive bounces (the wave-wide Russian roulette runs), 2 spatial passes; the
    camera walks down the platform so temporal reprojection and the TAA history taps move."""
    path = lambda f: (-1.6 + 0.01 * f, 1.7, -4.0 + 0.05 * f)
    problems, R = _frames("tunnel", 192, 108, 4, rpt_params=dict(max_non_tr_bounces=5, max_glossy_tr_bounces=5, num_spatial_passes=2),
                          cam_path=path)
    assert not problems, "\n".join(problems)


def test_atrium_many_lights_gi_lvg_through_the_renderer():
    """Config C4's path through the native frame driver: the scene has >= 13107 emissive triangles, so the renderer makes the
    reference's host decision (presampled sets 128 x 512; light voxel grid 32 x 8 x 40 because it was asked for), the
    integrator is ReSTIR GI (LVG NEE variant), DirectLighting reads the presampled sets. Compared with the oracle running
    the same configuration pass by pass."""
    from zetaray_b200 import lib, check
    from zetaray_b200.passes import Renderer
    from tests import rpt_util
    w, h = 128, 72
    flat, R, sc, cam = _setup("atrium_lights", w, h)
    assert len(flat.emissives) >= 13107
    rd = Renderer(sc, w, h, two_streams=True)
    assert rd.ApplySceneSettings(use_lvg=True) == (True, True)
    rd.SetMethod(Renderer.RESTIR_GI)
    R.osc.set_presampling(128, 512)
    R.osc.set_light_voxel_grid((32, 8, 40), (0.6, 0.45, 0.6), 0.1)
    seq = rpt_util.FrameSequence(w, h, cam_path=lambda f: cam)
    taa_prev = np.zeros((w * h, 2), dtype=np.uint32)
    problems = []
    for fr in range(3):
        fc = seq.next()
        R.gbuffer(fc)
        R.rdi(fc)
        R.rgi(fc)
        R.final = R.gi_final           # compositing reads the indirect integrator's output
        ref_comp, ref_taa = R.post(fc, taa_prev, fr > 0)
        taa_prev = ref_taa
        rd.Render(fc)
        check(lib.zr_stream_synchronize(None))
        if fr == 0:
            assert sc.sample_sets().tobytes() == R.osc.sample_sets[:128 * 512 * 10].tobytes(), "presampled sets differ"
            n = 32 * 8 * 40 * 64 * 8
            msg = diff_report("light voxel grid", sc.light_voxel_grid().reshape(-1, 8), R.osc.lvg[:n].reshape(-1, 8))
            assert not msg, msg
        checks = [("gi reservoir", gi_reservoirs(rd.gi.GetOutput(1)), R.gi_curr_reservoirs()),
                  ("gi final", rgba32f_bits(rd.gi.GetOutput(0)), R.gi_final.view(np.uint32)),
                  ("di_final", rgba32f_bits(rd.direct.GetOutput(0)), R.di_final.view(np.uint32)),
                  ("taa", uint32x2(rd.GetOutput()), ref_taa)]
        for name, a, b in checks:
            msg = diff_report(name, a, b)
            if msg:
                problems.append("frame %d: %s" % (fc.FrameNum, msg))
        if problems:
            break
    assert not problems, "\n".join(problems)
    # few lights -> the same call decides against presampling and therefore against the grid
    flat2, _, sc2, _ = _setup("atrium", 64, 36)
    rd2 = Renderer(sc2, 64, 36)
    assert rd2.ApplySceneSettings(use_lvg=True) == (False, False)
    assert lib.zr_renderer_set_integrator(rd2.handle, 7) != 0
    assert b"integrator" in lib.zr_last_error()


@pytest.mark.parametrize("which,detail,nrays", [("atrium", 1.0, 500), ("tunnel", 1.0, 250)])
def test_full_size_scene_bvh_kernels_against_brute_force(which, detail, nrays):
    """The benchmark-size scenes (C4 ~ 3 x 10^5, C5 ~ 10^6 triangles): scene upload + host BVH build + the product traversal
    kernels vs the oracle's brute force, closest hits bit for bit and any-hit flags, on camera rays and random segments."""
    import torch
    from zetaray_b200 import lib, check, procedural
    from zetaray_b200.passes import Scene
    from tests import scene_util
    from tests.orc import ptr
    from tests.test_bvh_host import make_rays
    make, cam = procedural.SCENES[which]
    flat = make(detail)
    osc = scene_util.OracleScene(flat)
    n = osc.o.orc_scene_num_tris(osc.h)
    assert n == flat.num_triangles and n > 250000
    wt = np.zeros((n, 9), dtype=np.float32)
    osc.o.orc_scene_get_tris(osc.h, ptr(wt))
    sc = Scene(flat)
    stats = sc.bvh_stats()
    assert stats["tris"] == n and stats["nodes"] > 1000
    rays = make_rays(wt, nrays, 5, np.array(cam, dtype=np.float32))
    ref = np.zeros((nrays, 4), dtype=np.float32)
    osc.o.orc_trace_closest(osc.h, ptr(rays), nrays, ptr(ref))
    ref_any = np.zeros(nrays, dtype=np.uint32)
    d_rays = torch.from_numpy(rays).cuda()
    d_hits = torch.zeros((nrays, 4), dtype=torch.float32, device="cuda")
    d_flags = torch.zeros(nrays, dtype=torch.int32, device="cuda")
    check(lib.zr_scene_trace_closest(sc.handle, C.c_void_p(d_rays.data_ptr()), nrays, C.c_void_p(d_hits.data_ptr()), None))
    check(lib.zr_scene_trace_any(sc.handle, C.c_void_p(d_rays.data_ptr()), nrays, C.c_void_p(d_flags.data_ptr()), None))
    torch.cuda.synchronize()
    got = d_hits.cpu().numpy()
    assert got.tobytes() == ref.tobytes(), int((got.view(np.uint32) != ref.view(np.uint32)).any(axis=1).sum())
    assert np.array_equal(d_flags.cpu().numpy() != 0, ref[:, 0] < 3.0e38)
    assert (ref[:, 0] < 3.0e38).mean() > 0.2
