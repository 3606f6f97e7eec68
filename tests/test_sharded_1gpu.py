"""Strip-sharded frames of the native renderer exercised on ONE GPU: every rank is a host thread with its own scene, renderer and
stream on cuda:0, and its zr_comm is built from a caller-supplied transport (zr_comm_create_transport) that copies the halo
bands between the ranks' planes on the device. Everything above the transport is the product path (zr_renderer_set_shard, the
row ranges in every pass, the exchange hooks inside the lighting passes, the exchange before Compositing, the gather on rank 0),
so this checks on a single-GPU box what tests/test_sharded_gpu.py checks with NCCL on several: every rank's strip is
byte-identical to the unsharded frame."""
import ctypes as C
import threading
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ZR_ERR_CUDA = 2


def _device_rows(img):
    """uint8 [H, pitch] torch view of a zr_image2d on cuda:0, without a copy."""
    import torch
    cai = {"shape": (img.height * img.pitch_bytes,), "typestr": "|u1", "data": (int(img.d_ptr), False), "version": 2}
    return torch.as_tensor(types.SimpleNamespace(__cuda_array_interface__=cai), device="cuda").view(img.height, img.pitch_bytes)


class ThreadTransport:
    """zr_comm_transport between ranks that are host threads of one process on one GPU. Each call synchronises the device (the
    rank's rows of this stage are complete), meets the other ranks at a barrier, copies what it needs out of their planes,
    synchronises again and meets them once more (nobody overwrites rows a peer is still reading). An exception is recorded,
    aborts the barrier so no peer waits forever, and becomes an error status the renderer returns."""

    def __init__(self, rank, world, shared, sums, barrier, errors):
        from tests.test_display_gpu import ThreadSum
        self.rank, self.world, self.shared, self.barrier, self.errors = rank, world, shared, barrier, errors
        self.sum = ThreadSum(rank, sums, barrier, errors)
        self.exchanges = [0, 0]         # per which_comm

    def comm(self):
        from zetaray_b200.passes import Comm
        return Comm.from_transport(*(self._guarded(fn) for fn in (self._exchange_halos, self._gather_rows, self._allreduce_u32)),
                                   self.rank, self.world)

    def _guarded(self, fn):
        def call(*args):
            try:
                fn(*args)
                return 0
            except BaseException as e:      # noqa: BLE001  (nothing propagates out of a ctypes callback)
                self.errors.append(e)
                self.barrier.abort()
                return ZR_ERR_CUDA
        return call

    def _publish(self, planes):
        import torch
        torch.cuda.synchronize()                    # my rows of this stage are complete
        self.shared[self.rank] = planes
        self.barrier.wait()

    def _release(self):
        import torch
        torch.cuda.synchronize()
        self.barrier.wait()                         # nobody overwrites rows a peer is still reading

    def _exchange_halos(self, user, which_comm, bounds, halo, planes, n, stream):
        b, r = [bounds[q] for q in range(self.world + 1)], self.rank
        mine = [_device_rows(planes[i]) for i in range(n)]
        self._publish(mine)
        for i, p in enumerate(mine):
            if r > 0:                               # the upper neighbour's bottom band
                y0 = max(b[r] - halo, b[r - 1])
                p[y0:b[r]].copy_(self.shared[r - 1][i][y0:b[r]])
            if r < self.world - 1:                  # the lower neighbour's top band
                y1 = min(b[r + 1] + halo, b[r + 2])
                p[b[r + 1]:y1].copy_(self.shared[r + 1][i][b[r + 1]:y1])
        self._release()
        self.exchanges[which_comm] += 1

    def _gather_rows(self, user, bounds, plane, root, stream):
        mine = _device_rows(plane[0])
        self._publish(mine)
        for q in range(self.world) if self.rank == root else ():
            if q != root:
                mine[bounds[q]:bounds[q + 1]].copy_(self.shared[q][bounds[q]:bounds[q + 1]])
        self._release()

    def _allreduce_u32(self, user, which_comm, d_values, n, stream):
        self.sum.reduce(d_values, n, stream)


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


def _planes(R, integrator, display):
    """(name, image, texel bytes) of every output the sharded frame must reproduce in its strip."""
    ind = R.gi if integrator == "gi" else R.indirect
    out = [("direct final", R.direct.GetOutput(0)), ("direct reservoirs", R.direct.GetOutput(1)),
           ("indirect final", ind.GetOutput(0)), ("indirect reservoirs", ind.GetOutput(1)),
           ("composited", R.compositing.GetOutput()), ("taa", R.GetOutput())]
    if display:
        out.append(("display", R.GetDisplayOutput()))
    return out


def _download(img):
    from zetaray_b200.passes import download_image
    return download_image(img, np.uint8, img.texel_bytes).reshape(img.height, -1)


@pytest.mark.parametrize("which,integrator,bounds,two_streams,cost,display", [
    ("glossy", "pt", [0, 96, 200], True, False, False),        # the DirectLighting hook runs on the second comm
    ("glass", "pt", [0, 64, 128, 200], False, True, False),     # measured cost map -> block schedule
    ("glossy", "gi", [0, 32, 128, 200], False, False, False),   # ReSTIR GI; a one-band strip: its top and bottom bands coincide
    ("cornell", "pt", [0, 96, 200], False, False, True),        # AutoExposure's all-reduce, the display image gathered
], ids=["pt-two-streams", "pt-cost-schedule", "gi-one-band-strip", "pt-display"])
def test_sharded_threads_equal_unsharded(which, integrator, bounds, two_streams, cost, display):
    import torch
    from zetaray_b200.passes import Scene, Renderer
    from zetaray_b200.sharding import StripPlan
    from zetaray_b200.camera import FrameSequence
    from tests import scene_util
    from tests.test_display_oracle import load_lut
    W, H = 288, 200
    warm, frames = 2, 4
    world = len(bounds) - 1
    plan = StripPlan(H, bounds)
    flat = scene_util.SCENES[which]()
    lut = load_lut() if display else None
    tiles_x, tiles_y = (W + 31) // 32, StripPlan.num_units(H)

    def renderer(streams):
        # every renderer has its own scene: the first frame of each runs prelighting on it
        R = Renderer(Scene(flat), W, H, two_streams=streams)
        if integrator == "gi":
            R.SetMethod(Renderer.RESTIR_GI)
        if display:
            R.SetDisplay(True, lut=lut)
        return R

    def frame_constants():
        seq = FrameSequence(W, H, cam_path=lambda f: (0.02 * f, 1.2, -4.043))
        fcs = [seq.next() for _ in range(warm + frames)]
        for fc in fcs:
            fc.dt = 1 / 60
        return fcs

    # unsharded reference, rendered first on this thread
    ref = renderer(False)
    s0 = torch.cuda.Stream()
    want = []
    for fc in frame_constants():
        ref.Render(fc, C.c_void_p(s0.cuda_stream))
        torch.cuda.synchronize()
        got = {k: _download(img) for k, img in _planes(ref, integrator, display)}
        if display:
            got["exposure"] = _download(ref.auto_exposure.GetOutput())
        want.append(got)

    ranks = [renderer(two_streams) for _ in range(world)]
    shared, sums, barrier, errors = {}, {}, threading.Barrier(world), []
    transports = [ThreadTransport(r, world, shared, sums, barrier, errors) for r in range(world)]
    comms = [t.comm() for t in transports]

    def rank_main(rank):
        R = ranks[rank]
        try:
            torch.cuda.set_device(0)
            st = torch.cuda.Stream()
            d_cost = torch.zeros(tiles_x * tiles_y, dtype=torch.int64, device="cuda")
            if cost:
                R.direct.SetCostMap(d_cost.data_ptr()); R.indirect.SetCostMap(d_cost.data_ptr())
            y0, y1 = plan.rows(rank)
            for f, fc in enumerate(frame_constants()):
                if f == warm:       # unsharded warm-up frames (every rank has the full history), then cut
                    torch.cuda.synchronize()
                    if cost:
                        R.direct.SetCostMap(0); R.indirect.SetCostMap(0)
                        tiles = [float(v) for v in d_cost.tolist()]
                        assert sum(tiles) > 0, "cost map stayed empty"
                        R.direct.SetScheduleCosts(tiles, tiles_x, tiles_y)
                        R.indirect.SetScheduleCosts(tiles, tiles_x, tiles_y)
                    R.SetShard(comms[rank], plan.bounds, gather_output=True)
                R.Render(fc, C.c_void_p(st.cuda_stream))
                torch.cuda.synchronize()
                if f < warm:
                    continue
                got = {k: _download(img) for k, img in _planes(R, integrator, display)}
                if display:
                    got["exposure"] = _download(R.auto_exposure.GetOutput())
                for k in got:
                    g, w = (got[k], want[f][k]) if k == "exposure" else (got[k][y0:y1], want[f][k][y0:y1])
                    if k == "indirect reservoirs" and integrator == "pt":
                        # bytes of an EMPTY reservoir beyond its header are don't-care
                        g4, w4 = g.reshape(y1 - y0, W, 64), w.reshape(y1 - y0, W, 64)
                        care = ~(((w4[..., 0] & 0xf) == 15)[..., None] & (np.arange(64) >= 16)[None, None, :])
                        g, w = g4 * care, w4 * care
                    bad = np.argwhere(g != w)
                    if bad.size:
                        raise AssertionError("rank %d frame %d: %s differs, first at (row, byte) %s of strip [%d, %d)" % (
                            rank, f, k, bad[0].tolist(), y0, y1))
                for k in ("taa", "display") if rank == 0 else ():
                    if k in got and not np.array_equal(got[k], want[f][k]):
                        raise AssertionError("frame %d: %s image gathered on rank 0 differs" % (f, k))
            sent, calls = comms[rank].stats()
            assert calls >= (3 if integrator == "gi" else 4) * frames and sent > 0, (sent, calls)
            # with two streams DirectLighting exchanges its reservoirs on the second comm
            assert (transports[rank].exchanges[1] >= frames) if two_streams else (transports[rank].exchanges[1] == 0), transports[rank].exchanges
        except BaseException as e:      # noqa: BLE001
            errors.append(e)
            barrier.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[0]
