"""How much of DirectLighting the frame hides behind IndirectLighting: bench.py's frame (Cornell 1080p, ReSTIR PT + ReSTIR DI +
firefly / TAA, steady state) through the native renderer on two streams and on one, next to the critical chain alone -- the
stand-alone G-buffer, IndirectLighting, Compositing and TAA passes on one stream, as bench.py's per-kernel pass runs them, without
DirectLighting -- and the G-buffer and DirectLighting alone.

    python tools/time_frame_schedule.py [--frames 30] [--rounds 3]

Each configuration is timed with CUDA events over `--frames` frames; the configurations alternate for `--rounds` rounds, and every
round's times and their medians are printed as one JSON line with the card's name, power limit and SM clock. Round 1 times the frames
bench.py times (after five warm-up frames). A frame can be no shorter than the chain alone
(the chain's kernels do not change with the schedule), so `two_streams - chain` is the most any DirectLighting schedule can win."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
W, H = 1920, 1080


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=10)
        return dict(zip(q.split(","), (p.strip() for p in r.stdout.strip().split(","))))
    except (OSError, subprocess.SubprocessError):
        return {"unavailable": True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    from zetaray_b200 import _lib
    from zetaray_b200.passes import Scene, GBuffers, GBufferRT, DirectLighting, IndirectLighting, Compositing, TAA, Renderer
    from zetaray_b200.camera import FrameSequence
    from zetaray_b200.scene import FlatScene
    if not torch.cuda.is_available():
        raise SystemExit("time_frame_schedule.py needs a CUDA device")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    st = C.c_void_p(stream.cuda_stream)
    scene = Scene(FlatScene.load(os.path.join(ROOT, "tests", "golden", "cornell_emissive.npz")))
    scene.prelighting(st)
    two, one = Renderer(scene, W, H, two_streams=True), Renderer(scene, W, H, two_streams=False)
    g, d, ind, comp, taa = GBufferRT(), DirectLighting(W, H), IndirectLighting(W, H), Compositing(W, H), TAA(W, H)
    fi = _lib.FrameInputs()
    fi.scene = scene.handle

    def standalone(gb, fc, lighting):
        gb.flip()
        fi.frame = fc
        gb.fill_inputs(fi)
        g.Render(fi, st)
        if "direct" in lighting:
            d.Render(fi, st)
        if "indirect" in lighting:
            ind.Render(fi, st)
            comp.Render(fi, d.GetOutput(0).d_ptr, ind.GetOutput(0).d_ptr, st)
            taa.Render(fi, comp.GetOutput().d_ptr, st)

    configs = {
        "two_streams": lambda fc: two.Render(fc, st),
        "single_stream": lambda fc: one.Render(fc, st),
        "chain": lambda fc, gb=GBuffers(W, H): standalone(gb, fc, ("indirect",)),
        "gbuffer_direct": lambda fc, gb=GBuffers(W, H): standalone(gb, fc, ("direct",)),
    }
    # Every configuration renders the same frame sequence, so round r times the same frames in each: IndirectLighting's cost still
    # changes after bench.py's five warm-up frames. Temporal and spatial reuse are on from the third frame.
    seqs = {k: FrameSequence(W, H) for k in configs}
    for name, fn in configs.items():
        for _ in range(5):
            fn(seqs[name].next())
    ms = {k: [] for k in configs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, fn in configs.items():
            fcs = [seqs[name].next() for _ in range(args.frames)]
            torch.cuda.synchronize()
            e0.record(stream)
            for fc in fcs:
                fn(fc)
            e1.record(stream)
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / args.frames)
    med = {k: round(statistics.median(v), 4) for k, v in ms.items()}
    print(json.dumps({
        "workload": "Cornell 1080p, bench.py's frame, ms per frame (median of %d rounds x %d frames)" % (args.rounds, args.frames),
        "ms_per_frame": med, "runs": {k: [round(x, 4) for x in v] for k, v in ms.items()},
        "hidden_ms_by_round": [round(a - b, 4) for a, b in zip(ms["single_stream"], ms["two_streams"])],
        "ceiling_ms_by_round": [round(a - b, 4) for a, b in zip(ms["two_streams"], ms["chain"])],
        "card": card()}))


if __name__ == "__main__":
    main()
