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


def _worker(rank, world, port, W, H, warm, frames, out_dir):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from zetaray_b200 import _lib
        from zetaray_b200.passes import Scene, GBuffers, GBufferRT, DirectLighting, IndirectLighting, Compositing, TAA
        from zetaray_b200.sharding import ShardedFrame, StripPlan
        from tests import scene_util, rpt_util
        stream = torch.cuda.Stream()
        torch.cuda.set_stream(stream)
        st = C.c_void_p(stream.cuda_stream)
        scene = Scene(scene_util.glossy_cornell())
        scene.prelighting(st)

        def pipeline():
            passes = dict(gbuffer=GBufferRT(), direct=DirectLighting(W, H), indirect=IndirectLighting(W, H),
                          compositing=Compositing(W, H), taa=TAA(W, H))
            gb = GBuffers(W, H)
            fi = _lib.FrameInputs()
            fi.scene = scene.handle
            return ShardedFrame(passes, gb, W, H, rank, world), fi

        A, fiA = pipeline()          # unsharded reference on this GPU
        B, fiB = pipeline()          # sharded after the warm-up
        A.world = 1
        seq = rpt_util.FrameSequence(W, H)
        B.begin_cost_measurement()
        for _ in range(warm):
            fc = seq.next()
            A.render(fiA, fc, stream, st)
            B.render(fiB, fc, stream, st)
        costs = B.end_cost_measurement(schedule=(world == 2))     # world 2 also exercises the expensive-first block order
        assert sum(costs) > 0, "cost map stayed empty"
        plan = StripPlan.balanced(H, world, costs)
        B.shard(plan, halo_mode="allgather" if world == 2 else "p2p")
        y0, y1 = plan.rows(rank)
        for f in range(frames):
            fc = seq.next()
            A.render(fiA, fc, stream, st)
            B.render(fiB, fc, stream, st)
            torch.cuda.synchronize()
            for name, get, dt, comps in (
                    ("direct final", lambda s: s.p["direct"].GetOutput(0), np.float32, 4),
                    ("indirect final", lambda s: s.p["indirect"].GetOutput(0), np.float32, 4),
                    ("direct reservoirs", lambda s: s.p["direct"].GetOutput(1), np.uint32, 8),
                    ("indirect reservoirs", lambda s: s.p["indirect"].GetOutput(1), np.uint32, 16),
                    ("composited", lambda s: s.p["compositing"].GetOutput(), np.float32, 4),
                    ("taa", lambda s: s.p["taa"].GetOutput(), np.uint16, 4)):
                a = _rows(get(A), dt, comps, y0, y1)
                b = _rows(get(B), dt, comps, y0, y1)
                if name == "indirect reservoirs":
                    # bytes of an EMPTY reservoir beyond its header are don't-care (the reference leaves them stale too)
                    k = a[..., 0] & 0xf
                    keep = (k != 15)[..., None] | (np.arange(16) < 4)[None, None, :]
                    a, b = a * keep, b * keep
                bad = np.argwhere(a.view(np.uint8).reshape(a.shape[0], a.shape[1], -1) != b.view(np.uint8).reshape(b.shape[0], b.shape[1], -1))
                assert bad.size == 0, "rank %d frame %d: %s differs at (row, col, byte) %s of strip [%d, %d)" % (
                    rank, f, name, bad[0].tolist(), y0, y1)
        B.gather_output(stream)
        torch.cuda.synchronize()
        full_a = _rows(A.p["taa"].GetOutput(), np.uint16, 4, 0, H)
        full_b = _rows(B.p["taa"].GetOutput(), np.uint16, 4, 0, H)
        assert np.array_equal(full_a, full_b), "gathered image differs from the unsharded one"
        assert B.halo.calls >= 3 * frames
        open(os.path.join(out_dir, "ok%d" % rank), "w").write("%s" % plan.bounds)
    finally:
        dist.destroy_process_group()


def _worker_native(rank, world, port, W, H, warm, frames, out_dir, integrator="pt"):
    """The native path: zr_renderer_set_shard + zr_comm (NCCL issued from C++), two streams, against an unsharded renderer."""
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
        for _ in range(warm):
            fc = seq.next()
            A.Render(fc, st); B.Render(fc, st)
        plan = StripPlan.uniform(H, world)
        B.SetShard(comm, plan.bounds, gather_output=True)
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


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_frame_equals_unsharded(tmp_path, world):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    mp.spawn(_worker, args=(world, _free_port(), 416, 296, 3, 4, str(tmp_path)), nprocs=world, join=True)
    assert all(os.path.exists(tmp_path / ("ok%d" % r)) for r in range(world))
