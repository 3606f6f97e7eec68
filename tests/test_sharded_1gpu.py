"""Strip-sharded frames of the native renderer exercised on ONE GPU: every rank is a host thread with its own scene, renderer and
stream on cuda:0, and its zr_comm is built from a caller-supplied transport (zr_comm_create_transport) that copies the halo
bands between the ranks' planes on the device. Everything above the transport is the product path (zr_renderer_set_shard, the
row ranges in every pass, the exchange hooks inside the lighting and SVGF passes, the exchange before Compositing, AutoExposure's
all-reduce, the gather on rank 0), so this checks on a single-GPU box what tests/test_sharded_gpu.py checks with NCCL on several:
every rank's strip of every plane is byte-identical to the unsharded frame. Also: the sized passes' set_rows."""
import ctypes as C

import numpy as np
import pytest

from tests.sharded_util import ThreadTransport, check_set_rows, compare_strip, host_rows, renderer_planes, run_threads

pytestmark = pytest.mark.gpu

W, H = 288, 200
HALO = 32


@pytest.mark.parametrize("pass_cls", ["DirectLighting", "IndirectLighting", "IndirectLightingGI", "Compositing", "TAA", "AutoExposure",
                                      "Display"])
def test_set_rows_refuses_bad_input(pass_cls):
    """check_set_rows for every sized pass but SVGF (tests/test_svgf_sharded_1gpu.py); the lighting passes also refuse a
    schedule-cost array of the wrong tile shape."""
    from zetaray_b200 import lib, passes
    Wp, Hp = 96, 70
    p = getattr(passes, pass_cls)(Wp, Hp)
    check_set_rows(p, Hp)
    if not hasattr(lib, p.prefix + "_set_schedule_costs"):
        return
    set_costs = getattr(lib, p.prefix + "_set_schedule_costs")
    tx, ty = (Wp + 31) // 32, (Hp + 31) // 32
    for bx, by in ((tx - 1, ty), (tx, ty + 1), (Wp // 8, Hp // 8)):
        assert set_costs(p.handle, (C.c_double * (bx * by))(), bx, by) == 1, (bx, by)
        assert lib.zr_last_error() == ("%s_set_schedule_costs: expected %u x %u tiles" % (p.prefix, tx, ty)).encode()
    assert set_costs(p.handle, (C.c_double * (tx * ty))(*range(tx * ty)), tx, ty) == 0
    assert set_costs(p.handle, None, 0, 0) == 0


def _frame_constants(n):
    from zetaray_b200.camera import FrameSequence
    seq = FrameSequence(W, H, cam_path=lambda f: (0.02 * f, 1.2, -4.043))
    fcs = [seq.next() for _ in range(n)]
    for fc in fcs:
        fc.dt = 1 / 60
    return fcs


def _frame_inputs(R, fc):
    """The FrameInputs the renderer's passes saw in its last frame."""
    from zetaray_b200 import lib, check, _lib
    fi = _lib.FrameInputs()
    fi.frame = fc
    check(lib.zr_renderer_get_gbuffer(R.handle, 0, C.byref(fi.curr)))
    check(lib.zr_renderer_get_gbuffer(R.handle, 1, C.byref(fi.prev)))
    fi.scene = R.scene.handle
    return fi


def _svgf_rows(p):
    return {k: host_rows(p.GetOutput(i)) for k, i in (("denoised", 0), ("guide", 2), ("history", 3))}


def _run_threads(which, integrator, bounds, two_streams=False, cost=False, display=False, svgf=None, warm=2, frames=4,
                 integrator_from=0, display_from=0, svgf_from=0, unshard_after=0, compare=True):
    """Renders `warm` unsharded frames, then `frames` sharded frames on len(bounds) - 1 thread ranks (and, with unshard_after,
    that many more after SetShard(None)). ReSTIR GI (integrator "gi"), the display stage and the denoiser (radius, num_passes)
    are switched on before frames integrator_from, display_from and svgf_from. With `cost`, the lighting passes measure their
    cost during the warm-up and run the cost-ordered block schedule after the cut. With `compare`, every sharded frame is held to
    an unsharded renderer that switches the same stages on at the same frames. Returns each rank's (bytes, calls) of its comm over
    the sharded frames."""
    import torch
    from zetaray_b200.passes import Scene, Renderer, SVGF
    from zetaray_b200.sharding import StripPlan
    from tests import scene_util
    from tests.test_display_oracle import load_lut
    world = len(bounds) - 1
    plan = StripPlan(H, bounds)
    flat = scene_util.SCENES[which]()
    lut = load_lut() if display else None
    fcs = _frame_constants(warm + frames + unshard_after)
    tiles_x, tiles_y = (W + 31) // 32, StripPlan.num_units(H)

    def method(f):
        return integrator if f >= integrator_from else "pt"

    def switch_on(R, f):
        if integrator == "gi" and f == integrator_from:
            R.SetMethod(Renderer.RESTIR_GI)
        if display and f == display_from:
            R.SetDisplay(True, lut=lut)
        if svgf and f == svgf_from:
            R.SetDenoiser(True)
            R.svgf.SetParams(radius=svgf[0], num_passes=svgf[1])

    # every renderer has its own scene: the first frame of each runs prelighting on it
    want = []
    if compare:
        ref = Renderer(Scene(flat), W, H, two_streams=False)
        s0 = torch.cuda.Stream()
        for f, fc in enumerate(fcs[:warm + frames]):
            switch_on(ref, f)
            ref.Render(fc, C.c_void_p(s0.cuda_stream))
            torch.cuda.synchronize()
            want.append(renderer_planes(ref, method(f)))

    ranks = [Renderer(Scene(flat), W, H, two_streams=two_streams) for _ in range(world)]
    transports = ThreadTransport.group(world)
    comms = [t.comm() for t in transports]
    traffic = [None] * world

    def rank_main(rank):
        R, comm = ranks[rank], comms[rank]
        st = torch.cuda.Stream()
        d_cost = torch.zeros(tiles_x * tiles_y, dtype=torch.int64, device="cuda")
        if cost:
            R.direct.SetCostMap(d_cost.data_ptr()); R.indirect.SetCostMap(d_cost.data_ptr())
        y0, y1 = plan.rows(rank)
        lone = None
        for f, fc in enumerate(fcs):
            if f == warm:       # unsharded warm-up frames (every rank has the full history), then cut
                torch.cuda.synchronize()
                if cost:
                    R.direct.SetCostMap(0); R.indirect.SetCostMap(0)
                    tiles = [float(v) for v in d_cost.tolist()]
                    assert sum(tiles) > 0, "cost map stayed empty"
                    R.direct.SetScheduleCosts(tiles, tiles_x, tiles_y)
                    R.indirect.SetScheduleCosts(tiles, tiles_x, tiles_y)
                R.SetShard(comm, plan.bounds, gather_output=True)
                start = comm.stats()
            switch_on(R, f)
            if f == warm + frames:
                end = comm.stats()
                traffic[rank] = (end[0] - start[0], end[1] - start[1])
                # whole frames again: with its history reset, the denoiser equals a whole-frame pass fed the same frames
                R.SetShard(None, None)
                R.svgf.ResetTemporal()
                lone = SVGF(W, H)
                lone.SetParams(radius=svgf[0], num_passes=svgf[1])
            R.Render(fc, C.c_void_p(st.cuda_stream))
            torch.cuda.synchronize()
            if lone is not None:
                lone.Render(_frame_inputs(R, fc), R.compositing.GetOutput().d_ptr)
                torch.cuda.synchronize()
                got, exp = _svgf_rows(R.svgf), _svgf_rows(lone)
                for k in exp:
                    if not np.array_equal(got[k], exp[k]):
                        raise AssertionError("rank %d frame %d after SetShard(None): svgf %s is not the whole-frame pass's" % (rank, f, k))
            elif f >= warm and compare:
                compare_strip(renderer_planes(R, method(f)), want[f], y0, y1, "rank %d frame %d" % (rank, f), gathered=rank == 0,
                              empty_reservoirs_dont_care=method(f) == "pt")
        if traffic[rank] is None:
            end = comm.stats()
            traffic[rank] = (end[0] - start[0], end[1] - start[1])
        elif comm.stats()[1] != start[1] + traffic[rank][1]:
            raise AssertionError("rank %d: the comm was used after SetShard(None)" % rank)
        sent, calls = traffic[rank]
        assert calls >= (3 if integrator == "gi" else 4) * frames and sent > 0, (sent, calls)
        # with two streams DirectLighting exchanges its reservoirs on the second comm
        ex = transports[rank].exchanges
        assert (ex[1] >= frames) if two_streams else (ex[1] == 0), ex

    run_threads(transports, rank_main)
    return traffic


@pytest.mark.parametrize("which,integrator,bounds,options", [
    ("glossy", "pt", [0, 96, 200], dict(two_streams=True)),             # the DirectLighting hook runs on the second comm
    ("glass", "pt", [0, 64, 128, 200], dict(cost=True)),                # measured cost map -> block schedule
    ("glossy", "gi", [0, 32, 128, 200], {}),                            # ReSTIR GI; a one-band strip: its top and bottom bands coincide
    ("cornell", "pt", [0, 96, 200], dict(display=True)),                # AutoExposure's all-reduce, the display image gathered
    ("glossy", "pt", [0, 96, 200], dict(two_streams=True, svgf=(2, 5))),    # SVGF 5x5 taps, 5 passes: the stage reaches 62 rows
    ("glossy", "pt", [0, 32, 128, 200], dict(svgf=(1, 3))),             # SVGF 3x3 taps, 3 passes over a one-band strip
    ("cornell", "gi", [0, 96, 200], dict(svgf=(2, 5), display=True)),   # AutoExposure histograms the denoised strip
    ("glossy", "gi", [0, 96, 200], dict(integrator_from=3)),            # the GI pass is created after the cut
    ("cornell", "pt", [0, 96, 200], dict(display=True, display_from=3)),    # the display stage is created after the cut
], ids=["pt-two-streams", "pt-cost-schedule", "gi-one-band-strip", "pt-display", "svgf-pt-r2-5-passes", "svgf-pt-r1-one-band-strip",
        "svgf-gi-display", "gi-after-set-shard", "display-after-set-shard"])
def test_sharded_threads_equal_unsharded(which, integrator, bounds, options):
    _run_threads(which, integrator, bounds, **options)


def test_svgf_enabled_after_set_shard_then_unsharded():
    """zr_renderer_set_denoiser after zr_renderer_set_shard: the new pass takes the renderer's strip and hook, so the frames equal an
    unsharded renderer that enables the denoiser at the same frame; after SetShard(None) it denoises whole frames without the hook."""
    _run_threads("glossy", "pt", [0, 96, 200], svgf=(2, 5), svgf_from=3, unshard_after=2)


def test_svgf_band_traffic():
    """The comm's bytes per frame with the denoiser minus those without it are the SVGF bands: min(32, strip rows) rows per band,
    colour + variance, guide (8 B/px each) and history (16 B/px) at the padded pitch after the temporal stage, colour + variance after
    every a-trous pass but the last, the denoised image (16 B/px, unpadded) after the last."""
    from zetaray_b200.passes import SVGF
    bounds, frames, (radius, passes) = [0, 32, 128, 200], 3, (2, 5)
    plain = _run_threads("cornell", "pt", bounds, frames=frames, compare=False)
    denoised = _run_threads("cornell", "pt", bounds, svgf=(radius, passes), frames=frames, compare=False)
    pitch = SVGF(W, H).GetOutput(2).pitch_bytes // 8        # ZR_SVGF_GUIDE
    per_row = pitch * (8 + 8 + 16) + (passes - 1) * pitch * 8 + W * 16
    for r in range(len(bounds) - 1):
        n_bands = (r > 0) + (r < len(bounds) - 2)
        rows = min(HALO, bounds[r + 1] - bounds[r])
        assert denoised[r][0] - plain[r][0] == frames * n_bands * rows * per_row, (r, plain[r], denoised[r])
        assert denoised[r][1] - plain[r][1] == frames * (passes + 1), (r, plain[r], denoised[r])
