"""Strip-sharded frames exercised on ONE GPU: two ranks run as two host threads with their own streams and full-size
buffers on cuda:0, and the halo "transport" is a device-to-device copy between the two ranks' planes at the points where
the passes call the exchange hook. Everything above the transport is the production code path (row ranges in every pass,
the hook inside zr_direct_pass_render / zr_indirect_pass_render, ShardedFrame), so this checks on a single-GPU box what
tests/test_sharded_gpu.py checks with NCCL on several: every rank's strip is byte-identical to the unsharded frame."""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


class ThreadHalo:
    """Drop-in for sharding.HaloExchanger between host threads of one process."""

    def __init__(self, plan, rank, shared, barrier):
        self.plan, self.rank, self.world = plan, rank, plan.world
        self.shared, self.barrier = shared, barrier
        self.calls = 0

    def _bands(self, r):
        y0, y1 = self.plan.rows(r)
        return (y0, min(y0 + 32, y1)), (max(y1 - 32, y0), y1)

    def exchange(self, planes):
        import torch
        torch.cuda.synchronize()                    # my rows of this stage are complete
        self.shared[self.rank] = planes
        self.barrier.wait()
        r = self.rank
        for i, p in enumerate(planes):
            if r > 0:
                (_, _), (b0, b1) = self._bands(r - 1)
                p[b0:b1].copy_(self.shared[r - 1][i][b0:b1])
            if r < self.world - 1:
                (t0, t1), (_, _) = self._bands(r + 1)
                p[t0:t1].copy_(self.shared[r + 1][i][t0:t1])
        torch.cuda.synchronize()
        self.barrier.wait()                         # nobody overwrites rows a peer is still reading
        self.calls += 1

    def gather_rows(self, plane):
        import torch
        torch.cuda.synchronize()
        self.shared[self.rank] = [plane]
        self.barrier.wait()
        for q in range(self.world):
            if q != self.rank:
                a, b = self.plan.rows(q)
                plane[a:b].copy_(self.shared[q][0][a:b])
        torch.cuda.synchronize()
        self.barrier.wait()


@pytest.mark.parametrize("pass_cls,has_schedule_costs", [("DirectLighting", True), ("IndirectLighting", True), ("IndirectLightingGI", False)])
def test_lighting_pass_strip_setters_refuse_bad_input(pass_cls, has_schedule_costs):
    """The lighting passes refuse an empty or out-of-image row range and a schedule-cost array of the wrong tile shape with
    ZR_ERR_INVALID_ARG, and zr_last_error names the pass and the entry point."""
    from zetaray_b200 import lib, passes
    W, H = 96, 70
    p = getattr(passes, pass_cls)(W, H)
    set_rows = getattr(lib, p.prefix + "_set_rows")
    for y0, y1 in ((0, 0), (40, 20), (H, H + 32), (H + 5, H + 40)):
        assert set_rows(p.handle, y0, y1) == 1, (y0, y1)
        assert lib.zr_last_error() == (p.prefix + "_set_rows: empty row range").encode()
    assert set_rows(p.handle, 32, H + 100) == 0         # rows past the image are clipped when the pass renders
    if not has_schedule_costs:
        return
    set_costs = getattr(lib, p.prefix + "_set_schedule_costs")
    tx, ty = (W + 31) // 32, (H + 31) // 32
    for bx, by in ((tx - 1, ty), (tx, ty + 1), (W // 8, H // 8)):
        assert set_costs(p.handle, (C.c_double * (bx * by))(), bx, by) == 1, (bx, by)
        assert lib.zr_last_error() == ("%s_set_schedule_costs: expected %u x %u tiles" % (p.prefix, tx, ty)).encode()
    assert set_costs(p.handle, (C.c_double * (tx * ty))(*range(tx * ty)), tx, ty) == 0
    assert set_costs(p.handle, None, 0, 0) == 0


@pytest.mark.parametrize("which,bounds", [("glossy", [0, 96, 200]), ("glass", [0, 64, 128, 200])])
def test_sharded_threads_equal_unsharded(which, bounds):
    import torch
    from zetaray_b200 import _lib
    from zetaray_b200.passes import (Scene, GBuffers, GBufferRT, DirectLighting, IndirectLighting, Compositing, TAA, download_image)
    from zetaray_b200.sharding import ShardedFrame, StripPlan
    from zetaray_b200.camera import FrameSequence
    from tests import scene_util
    W, H = 288, 200
    world = len(bounds) - 1
    plan = StripPlan(H, bounds)
    scene = Scene(scene_util.SCENES[which]())
    scene.prelighting()
    torch.cuda.synchronize()
    frames = [FrameSequence(W, H, cam_path=lambda f: (0.02 * f, 1.2, -4.043)) for _ in range(world + 1)]
    fcs = [[seq.next() for _ in range(6)] for seq in frames]

    def pipeline(rank):
        passes = dict(gbuffer=GBufferRT(), direct=DirectLighting(W, H), indirect=IndirectLighting(W, H),
                      compositing=Compositing(W, H), taa=TAA(W, H))
        fi = _lib.FrameInputs()
        fi.scene = scene.handle
        return ShardedFrame(passes, GBuffers(W, H), W, H, rank, world), fi

    # unsharded reference
    ref, fi_ref = pipeline(0)
    ref.world = 1
    s0 = torch.cuda.Stream()
    ref_out = []
    for fc in fcs[world]:
        ref.render(fi_ref, fc, s0)
        torch.cuda.synchronize()
        ref_out.append({k: download_image(img, np.uint8, img.texel_bytes).reshape(H, -1) for k, img in (
            ("direct", ref.p["direct"].GetOutput(0)), ("indirect", ref.p["indirect"].GetOutput(0)),
            ("di_res", ref.p["direct"].GetOutput(1)), ("pt_res", ref.p["indirect"].GetOutput(1)), ("taa", ref.p["taa"].GetOutput()))})

    shared, barrier = {}, threading.Barrier(world)
    errors = []

    def rank_main(rank):
        try:
            torch.cuda.set_device(0)
            stream = torch.cuda.Stream()
            sf, fi = pipeline(rank)
            for f, fc in enumerate(fcs[rank]):
                if f == 2:          # two unsharded warm-up frames (every rank has the full history), then cut
                    sf.shard(plan)
                    sf.halo = ThreadHalo(plan, rank, shared, barrier)
                sf.render(fi, fc, stream)
                torch.cuda.synchronize()
                if f >= 2:
                    y0, y1 = plan.rows(rank)
                    for k, img in (("direct", sf.p["direct"].GetOutput(0)), ("indirect", sf.p["indirect"].GetOutput(0)),
                                   ("di_res", sf.p["direct"].GetOutput(1)), ("pt_res", sf.p["indirect"].GetOutput(1)), ("taa", sf.p["taa"].GetOutput())):
                        got = download_image(img, np.uint8, img.texel_bytes).reshape(H, -1)[y0:y1]
                        want = ref_out[f][k][y0:y1]
                        if k == "pt_res":       # bytes of an EMPTY reservoir beyond its header are don't-care
                            g4, w4 = got.reshape(y1 - y0, W, 64), want.reshape(y1 - y0, W, 64)
                            empty = (w4[..., 0] & 0xf) == 15
                            g4 = np.where(empty[..., None] & (np.arange(64) >= 16)[None, None, :], 0, g4)
                            w4 = np.where(empty[..., None] & (np.arange(64) >= 16)[None, None, :], 0, w4)
                            got, want = g4.reshape(y1 - y0, -1), w4.reshape(y1 - y0, -1)
                        if not np.array_equal(got, want):
                            bad = np.argwhere(got != want)[0]
                            raise AssertionError("rank %d frame %d: %s differs at row %d" % (rank, f, k, y0 + bad[0]))
            sf.gather_output(stream)
            torch.cuda.synchronize()
            full = download_image(sf.p["taa"].GetOutput(), np.uint8, 8).reshape(H, -1)
            if not np.array_equal(full, ref_out[-1]["taa"]):
                raise AssertionError("rank %d: gathered image differs" % rank)
            assert sf.halo.calls >= 3 * 4
        except BaseException as e:      # noqa: BLE001
            errors.append(e)
            barrier.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[0]
