"""ReSTIR PT debug views on the device: bit-exact against the oracle's restatement at the reference's write points under every
reuse setting, with accumulation, a moving camera and the glass scene's full material build; the reservoir planes and launches
of frames without a view untouched; the refusals; the view across resize and reset; strip-sharded frames."""
import ctypes as C

import numpy as np
import pytest

from tests import scene_util
from tests.parity import CHECKS, DeviceFrame, _planes, diff_report, pt_reservoirs, rgba32f_bits, uint16_plane
from tests.rpt_debug_view_util import (NONE, K, CASE, FOUND_CONNECTION, CONNECTION_LOBE_K_MIN_1, CONNECTION_LOBE_K, VIEWS, REUSE,
                                       ViewOracle, debug_color)
from zetaray_b200 import lib
from zetaray_b200.camera import FrameSequence

pytestmark = pytest.mark.gpu

W, H = 256, 144
MOVING = lambda f: (0.03 * f, 1.2 + 0.02 * f, -4.043 + 0.05 * f)


def view_parity(scene, views, rpt_params=None, cam_path=None, accumulate=False, setup=None, w=W, h=H):
    """Frames of `scene` on the oracle and the device, frame i with debug view views[i] on both, every ReSTIR PT plane compared
    byte for byte. setup(DeviceFrame) runs before the first frame. Returns (problems, the device frame's FINAL per frame)."""
    flat = scene_util.SCENES[scene]()
    R = ViewOracle(flat, w, h)
    for k, v in (rpt_params or {}).items():
        setattr(R.params, k, v)
    f = DeviceFrame(flat, w, h, ("rpt",), rpt_params=rpt_params)
    seq = FrameSequence(w, h, cam_path=cam_path, accumulate=accumulate)
    problems, finals = [], []
    try:
        if setup:
            setup(f)
        for fr, view in enumerate(views):
            R.view = view
            if view is not None:
                f.rpt.SetDebugView(view)
            fc = seq.next()
            R.gbuffer(fc)
            R.rpt(fc)
            f.render(fc)
            for name, read, want in _planes(f, R, fr, None):
                msg = diff_report(name, read(), want) if name in CHECKS[("rpt",)] else None
                if msg:
                    problems.append("frame %d (view %s): %s" % (fc.FrameNum, view, msg))
            finals.append(rgba32f_bits(f.rpt.GetOutput(0)).copy())
            if problems:
                break
    finally:
        f.close()
    return problems, finals


@pytest.mark.parametrize("view", VIEWS)
@pytest.mark.parametrize("reuse", list(REUSE))
@pytest.mark.parametrize("scene", ["glossy", "cornell"])
def test_view_matches_oracle(scene, reuse, view):
    problems, finals = view_parity(scene, [view] * 4, REUSE[reuse])
    assert not problems, "\n".join(problems)
    rgb = finals[-1].view(np.float32).reshape(-1, 4)[:, :3]
    assert (rgb != 0).any(axis=1).sum() > 0, "the view is black everywhere"


@pytest.mark.parametrize("reuse", list(REUSE))
def test_view_with_accumulation(reuse):
    problems, _ = view_parity("glossy", [K, K, CONNECTION_LOBE_K, CONNECTION_LOBE_K], REUSE[reuse], accumulate=True)
    assert not problems, "\n".join(problems)


@pytest.mark.parametrize("reuse", list(REUSE))
def test_view_with_moving_camera(reuse):
    problems, _ = view_parity("glossy", [CASE, CASE, K, FOUND_CONNECTION], REUSE[reuse], cam_path=MOVING)
    assert not problems, "\n".join(problems)


@pytest.mark.parametrize("reuse", ["pathtrace", "spatial1"])
def test_glass_scene_lobe_views(reuse):
    """The full material build (transmission): the lobe views show GLOSSY_T and DIFFUSE_T."""
    problems, finals = view_parity("glass", [CONNECTION_LOBE_K_MIN_1] * 2 + [CONNECTION_LOBE_K] * 2, REUSE[reuse])
    assert not problems, "\n".join(problems)
    seen = set()
    for fr, view in ((1, CONNECTION_LOBE_K_MIN_1), (3, CONNECTION_LOBE_K)):
        cols = set(map(tuple, finals[fr].view(np.float32).reshape(-1, 4)[:, :3].tolist()))
        for lobe in (1, 3):     # DIFFUSE_T, GLOSSY_T
            meta = np.array([(lobe | (lobe << 3)) << 8], np.uint32)
            if tuple(debug_color(view, meta, np.zeros((1, 3), np.float32))[0].tolist()) in cols:
                seen.add((view, lobe))
    assert {(CONNECTION_LOBE_K_MIN_1, 3), (CONNECTION_LOBE_K, 3)} <= seen and any(l == 1 for _, l in seen), seen


def test_view_switched_on_and_off_mid_sequence():
    """On the oracle and the device alike, then against a sequence that never had a view: the same FINAL once it is off again."""
    views = [NONE, NONE, K, CASE, NONE, NONE]
    problems, finals = view_parity("glossy", views, REUSE["spatial1"])
    assert not problems, "\n".join(problems)
    problems, plain = view_parity("glossy", [NONE] * len(views), REUSE["spatial1"])
    assert not problems, "\n".join(problems)
    for fr in (0, 1, 4, 5):
        assert finals[fr].tobytes() == plain[fr].tobytes(), fr
    assert finals[2].tobytes() != plain[2].tobytes()


def _device_frames(scene, views, rpt_params):
    """Device frames with the given views: every plane but FINAL and the kernel launches per frame."""
    flat = scene_util.SCENES[scene]()
    f = DeviceFrame(flat, W, H, ("rpt",), rpt_params=rpt_params)
    seq = FrameSequence(W, H)
    out = []
    try:
        for view in views:
            f.rpt.SetDebugView(view)
            fc = seq.next()
            n0 = lib.zr_kernel_launch_count()
            f.render(fc)
            n1 = lib.zr_kernel_launch_count()
            planes = {"reservoir curr": pt_reservoirs(f.rpt.GetOutput(1)).tobytes(),
                      "reservoir prev": pt_reservoirs(f.rpt.GetOutput(2)).tobytes(),
                      "target": rgba32f_bits(f.rpt.GetOutput(3)).tobytes(), "neighbor": uint16_plane(f.rpt.GetOutput(4)).tobytes(),
                      "threadmap": uint16_plane(f.rpt.GetOutput(6)).tobytes()}
            out.append((planes, n1 - n0))
    finally:
        f.close()
    return out


@pytest.mark.parametrize("reuse", list(REUSE))
def test_reservoir_planes_and_launches(reuse):
    """Every plane but FINAL is the same bytes with and without a view. A frame with view NONE -- also right after frames with one
    -- launches what a pass that never had a view launches; a frame with a view launches one more kernel per stage that writes
    FINAL."""
    views = [K, CONNECTION_LOBE_K, NONE, FOUND_CONNECTION, NONE]
    got = _device_frames("glossy", views, REUSE[reuse])
    want = _device_frames("glossy", [NONE] * len(views), REUSE[reuse])
    passes = REUSE[reuse]["num_spatial_passes"]
    for fr, ((gp, gn), (wp, wn)) in enumerate(zip(got, want)):
        for name in wp:
            assert gp[name] == wp[name], "frame %d: %s differs" % (fr, name)
        stages = 0 if views[fr] == NONE else (passes if (passes and fr > 0) else 1)
        assert gn == wn + stages, (fr, gn, wn)


def test_set_debug_view_refuses_bad_calls_and_the_view_survives_resize_and_reset():
    from zetaray_b200.passes import IndirectLighting
    ind = IndirectLighting(64, 64)
    assert lib.zr_indirect_pass_set_debug_view(ind.handle, 6) == 1           # ZR_ERR_INVALID_ARG
    assert b"out of range" in lib.zr_last_error()
    assert lib.zr_indirect_pass_set_debug_view(None, K) == 1
    for v in (NONE,) + VIEWS:
        assert lib.zr_indirect_pass_set_debug_view(ind.handle, v) == 0

    def setup(f):
        f.rpt.OnWindowResized(96, 64)
        f.rpt.SetDebugView(CASE)
        f.rpt.OnWindowResized(W, H)
        f.rpt.ResetTemporal()
    # the device pass is never told the view again; the oracle renders CASE throughout
    views = [CASE, CASE, CASE]
    flat = scene_util.SCENES["glossy"]()
    R = ViewOracle(flat, W, H)
    R.view = CASE
    f = DeviceFrame(flat, W, H, ("rpt",))
    seq = FrameSequence(W, H)
    try:
        setup(f)
        for fr in range(len(views)):
            fc = seq.next()
            R.gbuffer(fc)
            R.rpt(fc)
            f.render(fc)
            msg = diff_report("pt_final", rgba32f_bits(f.rpt.GetOutput(0)), R.final.view(np.uint32))
            assert msg is None, "frame %d: %s" % (fr, msg)
    finally:
        f.close()


def _sharded(bounds, view, frames=3, warm=1):
    import torch
    from zetaray_b200.passes import Scene, Renderer
    from zetaray_b200.sharding import StripPlan
    from tests.sharded_util import ThreadTransport, compare_strip, renderer_planes, run_threads
    SW, SH = 288, 200
    plan = StripPlan(SH, bounds)
    flat = scene_util.SCENES["glossy"]()
    seq = FrameSequence(SW, SH, cam_path=lambda f: (0.02 * f, 1.2, -4.043))
    fcs = [seq.next() for _ in range(warm + frames)]
    for fc in fcs:
        fc.dt = 1 / 60
    ref = Renderer(Scene(flat), SW, SH, two_streams=False)
    ref.indirect.SetDebugView(view)
    s0 = torch.cuda.Stream()
    want = []
    for fc in fcs:
        ref.Render(fc, C.c_void_p(s0.cuda_stream))
        torch.cuda.synchronize()
        want.append(renderer_planes(ref, "pt"))
    world = len(bounds) - 1
    ranks = [Renderer(Scene(flat), SW, SH, two_streams=False) for _ in range(world)]
    for R in ranks:
        R.indirect.SetDebugView(view)               # each rank sets the view on its own pass
    transports = ThreadTransport.group(world)
    comms = [t.comm() for t in transports]

    def rank_main(rank):
        R, comm = ranks[rank], comms[rank]
        st = torch.cuda.Stream()
        y0, y1 = plan.rows(rank)
        for fr, fc in enumerate(fcs):
            if fr == warm:
                torch.cuda.synchronize()
                R.SetShard(comm, plan.bounds, gather_output=True)
            R.Render(fc, C.c_void_p(st.cuda_stream))
            torch.cuda.synchronize()
            if fr >= warm:
                compare_strip(renderer_planes(R, "pt"), want[fr], y0, y1, "rank %d frame %d" % (rank, fr), gathered=rank == 0)

    run_threads(transports, rank_main)


@pytest.mark.parametrize("view", [K, CONNECTION_LOBE_K])
def test_sharded_threads_equal_unsharded(view):
    _sharded([0, 96, 200], view)

