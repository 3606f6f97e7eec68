"""Strip-sharded frames on 2+ GPUs (one process per GPU, NCCL): every frame, each rank's strip of every pass output is
byte-identical to the same rows of an unsharded render of the same frame on the same GPU, and the gathered image is
the unsharded image. Needs >= 2 visible GPUs; skipped on a 1-GPU machine."""
import ctypes as C
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rows(img, dtype, comps, y0, y1):
    from zetaray_b200.passes import download_image
    a = download_image(img, dtype, comps).reshape(img.height, img.width, comps)
    return a[y0:y1]


def _worker_native(rank, world, port, W, H, warm, frames, out_dir, integrator="pt"):
    """zr_renderer_set_shard + zr_comm (NCCL issued from C++), two streams, strips cut by the measured cost, against an unsharded
    renderer."""
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from zetaray_b200.passes import Scene, Renderer, Comm, download_image
        from zetaray_b200.sharding import StripPlan
        from tests import scene_util, rpt_util
        stream = torch.cuda.Stream()
        torch.cuda.set_stream(stream)
        st = C.c_void_p(stream.cuda_stream)
        scene = Scene(scene_util.glossy_cornell())
        A = Renderer(scene, W, H, two_streams=False)        # unsharded reference on this GPU
        B = Renderer(scene, W, H, two_streams=True)
        if integrator == "gi":          # ReSTIR GI: zr_gi_pass_set_rows + its reservoir-halo hook (BASELINE config 4 runs this way)
            A.SetMethod(Renderer.RESTIR_GI); B.SetMethod(Renderer.RESTIR_GI)
        comm = Comm.from_torch()
        seq = rpt_util.FrameSequence(W, H)
        # the cost of every 32-row band, measured during the unsharded warm-up as bench.py does
        tiles_x, tiles_y = (W + 31) // 32, StripPlan.num_units(H)
        cost = torch.zeros(tiles_x * tiles_y, dtype=torch.int64, device="cuda")
        lit = (B.direct, B.indirect)
        for p in lit:
            p.SetCostMap(cost.data_ptr())
        for _ in range(warm):
            fc = seq.next()
            A.Render(fc, st); B.Render(fc, st)
        torch.cuda.synchronize()
        for p in lit:
            p.SetCostMap(0)
        c = cost.to(torch.float64)
        dist.all_reduce(c, op=dist.ReduceOp.SUM)                # identical plan on every rank
        tiles = [float(v) for v in c.tolist()]
        costs = [sum(tiles[b * tiles_x:(b + 1) * tiles_x]) for b in range(tiles_y)]
        assert sum(costs) > 0, "cost map stayed empty"
        plan = StripPlan.balanced(H, world, costs)
        B.SetShard(comm, plan.bounds, gather_output=True)
        if world == 2:          # world 2 also exercises the expensive-first block order
            for p in lit:
                p.SetScheduleCosts(tiles, tiles_x, tiles_y)
        y0, y1 = plan.rows(rank)
        for f in range(frames):
            fc = seq.next()
            A.Render(fc, st); B.Render(fc, st)
            torch.cuda.synchronize()
            for name, get, dt, comps in (
                    ("direct final", lambda r: r.direct.GetOutput(0), np.float32, 4),
                    ("indirect final", (lambda r: r.gi.GetOutput(0)) if integrator == "gi" else (lambda r: r.indirect.GetOutput(0)), np.float32, 4),
                    ("indirect reservoirs", (lambda r: r.gi.GetOutput(1)) if integrator == "gi" else (lambda r: r.indirect.GetOutput(1)), np.uint32,
                     12 if integrator == "gi" else 16),
                    ("direct reservoirs", lambda r: r.direct.GetOutput(1), np.uint32, 8),
                    ("composited", lambda r: r.compositing.GetOutput(), np.float32, 4),
                    ("taa", lambda r: r.taa.GetOutput(), np.uint16, 4)):
                a = _rows(get(A), dt, comps, y0, y1)
                b = _rows(get(B), dt, comps, y0, y1)
                bad = np.argwhere(a.view(np.uint8).reshape(a.shape[0], a.shape[1], -1) != b.view(np.uint8).reshape(b.shape[0], b.shape[1], -1))
                assert bad.size == 0, "rank %d frame %d: %s differs at (row, col, byte) %s of strip [%d, %d)" % (
                    rank, f, name, bad[0].tolist(), y0, y1)
            if rank == 0:
                full_a = _rows(A.GetOutput(), np.uint16, 4, 0, H)
                full_b = _rows(B.GetOutput(), np.uint16, 4, 0, H)
                assert np.array_equal(full_a, full_b), "frame %d: image gathered on rank 0 differs from the unsharded one" % f
        sent, calls = comm.stats()
        assert calls >= (3 if integrator == "gi" else 4) * frames and sent > 0
        open(os.path.join(out_dir, "ok%d" % rank), "w").write("%s" % plan.bounds)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_native_sharded_renderer_equals_unsharded(tmp_path, world):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    mp.spawn(_worker_native, args=(world, _free_port(), 416, 296, 3, 4, str(tmp_path)), nprocs=world, join=True)
    assert all(os.path.exists(tmp_path / ("ok%d" % r)) for r in range(world))


@pytest.mark.parametrize("world", [2, 4])
def test_native_sharded_restir_gi_equals_unsharded(tmp_path, world):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    mp.spawn(_worker_native, args=(world, _free_port(), 416, 296, 3, 4, str(tmp_path), "gi"), nprocs=world, join=True)
    assert all(os.path.exists(tmp_path / ("ok%d" % r)) for r in range(world))
