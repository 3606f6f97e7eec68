"""Strip-sharded frames on 2+ GPUs (one process per GPU, NCCL): every frame, each rank's strip of every pass output is
byte-identical to the same rows of an unsharded render of the same frame on the same GPU, and the gathered images are
the unsharded images. Needs >= 2 visible GPUs; skipped on a 1-GPU machine."""
import ctypes as C
import os

import pytest

from tests.sharded_util import compare_strip, renderer_planes, spawn_nccl

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, out_dir, integrator, display, W=416, H=296, warm=3, frames=4):
    """zr_renderer_set_shard + zr_comm (NCCL issued from C++), two streams, strips cut by the measured cost, against an unsharded
    renderer; with `display`, the display stage (AutoExposure's all-reduce, the display image gathered)."""
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from zetaray_b200.passes import Scene, Renderer, Comm
        from zetaray_b200.sharding import StripPlan
        from tests import scene_util, rpt_util
        from tests.test_display_oracle import load_lut
        stream = torch.cuda.Stream()
        torch.cuda.set_stream(stream)
        st = C.c_void_p(stream.cuda_stream)
        scene = Scene(scene_util.glossy_cornell())
        A = Renderer(scene, W, H, two_streams=False)        # unsharded reference on this GPU
        B = Renderer(scene, W, H, two_streams=True)
        for r in (A, B):
            if integrator == "gi":      # ReSTIR GI: zr_gi_pass_set_rows + its reservoir-halo hook (BASELINE config 4 runs this way)
                r.SetMethod(Renderer.RESTIR_GI)
            if display:
                r.SetDisplay(True, lut=load_lut())
        comm = Comm.from_torch()
        seq = rpt_util.FrameSequence(W, H)

        def next_frame():
            fc = seq.next()
            fc.dt = 1 / 60
            return fc

        # the cost of every 32-row band, measured during the unsharded warm-up as bench.py does
        tiles_x, tiles_y = (W + 31) // 32, StripPlan.num_units(H)
        cost = torch.zeros(tiles_x * tiles_y, dtype=torch.int64, device="cuda")
        lit = (B.direct, B.indirect)
        for p in lit:
            p.SetCostMap(cost.data_ptr())
        for _ in range(warm):
            fc = next_frame()
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
            fc = next_frame()
            A.Render(fc, st); B.Render(fc, st)
            torch.cuda.synchronize()
            compare_strip(renderer_planes(B, integrator), renderer_planes(A, integrator), y0, y1, "rank %d frame %d" % (rank, f),
                          gathered=rank == 0)
        sent, calls = comm.stats()
        assert calls >= (3 if integrator == "gi" else 4) * frames and sent > 0
        open(os.path.join(out_dir, "ok%d" % rank), "w").write("%s" % plan.bounds)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_native_sharded_renderer_equals_unsharded(tmp_path, world):
    spawn_nccl(_worker, world, tmp_path, "pt", False)


@pytest.mark.parametrize("world", [2, 4])
def test_native_sharded_restir_gi_equals_unsharded(tmp_path, world):
    spawn_nccl(_worker, world, tmp_path, "gi", False)


@pytest.mark.parametrize("world", [2, 4])
def test_native_sharded_display_equals_unsharded(tmp_path, world):
    spawn_nccl(_worker, world, tmp_path, "pt", True)
