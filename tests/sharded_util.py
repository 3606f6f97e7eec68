"""What the strip-sharded tests share: views and copies of pass planes, a zr_comm transport between ranks that are host threads
on one GPU, the thread runner, the NCCL process spawner, the planes a sharded renderer must reproduce and the one comparison of a
rank's strip with the unsharded frame."""
import os
import socket
import threading
import types

import numpy as np
import pytest

ZR_ERR_CUDA = 2


def _device_bytes(d_ptr, nbytes):
    import torch
    cai = {"shape": (nbytes,), "typestr": "|u1", "data": (int(d_ptr), False), "version": 2}
    return torch.as_tensor(types.SimpleNamespace(__cuda_array_interface__=cai), device="cuda")


def device_rows(img):
    """uint8 [H, pitch] torch view of a zr_image2d on cuda:0, without a copy."""
    return _device_bytes(img.d_ptr, img.height * img.pitch_bytes).view(img.height, img.pitch_bytes)


def host_rows(img):
    """uint8 [height, width * texel] host copy of a zr_image2d, padded or not."""
    from zetaray_b200.passes import download_image_pitched
    return download_image_pitched(img, np.uint8, img.texel_bytes).reshape(img.height, -1)


def check_set_rows(p, height):
    """A sized pass's set_rows contract: an empty or out-of-image row range is refused with ZR_ERR_INVALID_ARG and zr_last_error
    names the pass and the entry point; rows past the image are accepted (clipped when the pass renders); a null pass is refused,
    and so is a null pass's halo hook where the pass has one."""
    from zetaray_b200 import lib
    set_rows = getattr(lib, p.prefix + "_set_rows")
    for y0, y1 in ((0, 0), (40, 20), (height, height + 32), (height + 5, height + 40)):
        assert set_rows(p.handle, y0, y1) == 1, (y0, y1)
        assert lib.zr_last_error() == (p.prefix + "_set_rows: empty row range").encode()
    assert set_rows(None, 0, height) == 1
    p.SetRows(32, height + 100)
    if hasattr(lib, p.prefix + "_set_halo_exchange"):
        assert getattr(lib, p.prefix + "_set_halo_exchange")(None, None, None) == 1
        p.SetHaloExchange(None)


class ThreadTransport:
    """zr_comm_transport between ranks that are host threads of one process on one GPU. Each call synchronises the device (the
    rank's rows of this stage are complete), meets the other ranks at a barrier, takes what it needs from their planes,
    synchronises again and meets them once more (nobody overwrites values a peer is still reading). An exception is recorded,
    aborts the barrier so no peer waits forever, and becomes an error status the renderer returns."""

    def __init__(self, rank, world, shared, barrier, errors):
        self.rank, self.world, self.shared, self.barrier, self.errors = rank, world, shared, barrier, errors
        self.exchanges = [0, 0]         # per which_comm
        self.reductions = 0

    @staticmethod
    def group(world):
        """One transport per rank, sharing one exchange area, one barrier and one error list."""
        shared, barrier, errors = {}, threading.Barrier(world), []
        return [ThreadTransport(r, world, shared, barrier, errors) for r in range(world)]

    def fail(self, e):
        self.errors.append(e)
        self.barrier.abort()

    def comm(self):
        from zetaray_b200.passes import Comm
        return Comm.from_transport(*(self._guarded(fn) for fn in (self._exchange_halos, self._gather_rows, self._allreduce_u32)),
                                   self.rank, self.world)

    def reduce_fn(self):
        """The all-reduce as a lone pass's reduce hook (AutoExposure.SetReduce)."""
        from zetaray_b200 import _lib
        allreduce = self._guarded(self._allreduce_u32)

        def hook(user, d_values, n, stream):
            allreduce(user, 0, d_values, n, stream)
        return _lib.REDUCE_U32_FN(hook)

    def _guarded(self, fn):
        def call(*args):
            try:
                fn(*args)
                return 0
            except BaseException as e:      # noqa: BLE001  (nothing propagates out of a ctypes callback)
                self.fail(e)
                return ZR_ERR_CUDA
        return call

    def _publish(self, mine):
        import torch
        torch.cuda.synchronize()                    # my values of this stage are complete
        self.shared[self.rank] = mine
        self.barrier.wait()

    def _release(self):
        import torch
        torch.cuda.synchronize()
        self.barrier.wait()                         # nobody overwrites values a peer is still reading

    def _exchange_halos(self, user, which_comm, bounds, halo, planes, n, stream):
        b, r = [bounds[q] for q in range(self.world + 1)], self.rank
        mine = [device_rows(planes[i]) for i in range(n)]
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
        mine = device_rows(plane[0])
        self._publish(mine)
        for q in range(self.world) if self.rank == root else ():
            if q != root:
                mine[bounds[q]:bounds[q + 1]].copy_(self.shared[q][bounds[q]:bounds[q + 1]])
        self._release()

    def _allreduce_u32(self, user, which_comm, d_values, n, stream):
        import torch
        mine = _device_bytes(d_values, 4 * n).view(torch.int32)        # two's-complement sums are the uint32 sums
        self._publish(mine)
        total = sum(self.shared[q] for q in range(self.world))
        self._release()
        mine.copy_(total)
        torch.cuda.synchronize()
        self.reductions += 1


def run_threads(transports, rank_main):
    """rank_main(rank) for every rank of `transports` on a host thread of its own (cuda:0). The first error aborts the ranks'
    barrier, so no rank waits forever, and is raised here once every thread has ended."""
    import torch

    def main(rank):
        try:
            torch.cuda.set_device(0)
            rank_main(rank)
        except BaseException as e:      # noqa: BLE001
            transports[rank].fail(e)

    threads = [threading.Thread(target=main, args=(r,)) for r in range(len(transports))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    errors = transports[0].errors
    assert not errors, errors[0]


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def spawn_nccl(worker, world, out_dir, *args):
    """worker(rank, world, port, out_dir, *args) in one process per GPU; each process writes out_dir/ok<rank> when it passed.
    Skips when fewer than `world` GPUs are visible."""
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    mp.spawn(worker, args=(world, free_port(), str(out_dir)) + args, nprocs=world, join=True)
    assert all(os.path.exists(os.path.join(str(out_dir), "ok%d" % r)) for r in range(world))


def renderer_planes(R, integrator):
    """{name: host rows} of every plane a sharded renderer must reproduce in its strip, in the order the frame writes them: DI and
    indirect finals and reservoirs (ReSTIR PT's pass, or the path tracer / ReSTIR GI pass for `integrator` "gi"), composited, the
    SVGF planes when the denoiser is on, TAA, and the exposure state and display image when the display stage is on."""
    ind = R.gi if integrator == "gi" else R.indirect
    out = {"direct final": R.direct.GetOutput(0), "direct reservoirs": R.direct.GetOutput(1),
           "indirect final": ind.GetOutput(0), "indirect reservoirs": ind.GetOutput(1), "composited": R.compositing.GetOutput()}
    if R.svgf is not None:
        for name, i in (("denoised", 0), ("guide", 2), ("history", 3)):         # ZR_SVGF_DENOISED, _GUIDE, _HISTORY
            out["svgf " + name] = R.svgf.GetOutput(i)
    out["taa"] = R.GetOutput()
    if R.display is not None:
        out["exposure"] = R.auto_exposure.GetOutput()
        out["display"] = R.GetDisplayOutput()
    return {k: host_rows(img) for k, img in out.items()}


def compare_strip(got, want, y0, y1, what, gathered=False, empty_reservoirs_dont_care=False):
    """Rows [y0, y1) of every plane of `got` byte-equal to `want`'s; the exposure state, which every rank derives from the summed
    histogram, whole. `gathered`: this rank holds the gathered TAA and display images, which must equal the whole frame.
    `empty_reservoirs_dont_care` (ReSTIR PT only): the bytes of an empty reservoir beyond its header (bytes 16-63 of a 64-byte
    record whose meta & 0xf == 15) are not compared. Reported rows count from y0."""
    assert got.keys() == want.keys(), (what, got.keys(), want.keys())
    for k in got:
        g, w = (got[k], want[k]) if k == "exposure" else (got[k][y0:y1], want[k][y0:y1])
        if k == "indirect reservoirs" and empty_reservoirs_dont_care:
            g4, w4 = g.reshape(g.shape[0], -1, 64), w.reshape(w.shape[0], -1, 64)
            care = ~(((w4[..., 0] & 0xf) == 15)[..., None] & (np.arange(64) >= 16)[None, None, :])
            g, w = g4 * care, w4 * care
        bad = np.argwhere(g != w)
        if bad.size:
            raise AssertionError("%s: %s differs, first at (row, ...) %s of strip [%d, %d)" % (what, k, bad[0].tolist(), y0, y1))
    for k in ("taa", "display") if gathered else ():
        if k in got and not np.array_equal(got[k], want[k]):
            raise AssertionError("%s: %s image gathered on rank 0 differs" % (what, k))
