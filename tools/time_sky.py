"""Times the sky: k_sky_view_lut (256 x 128) alone (CUDA events around repeated launches on an idle device), and the 1080p
renderer's frame time on the Cornell scene with the sky off and on (CUDA events around zr_renderer_render, two streams), the two
alternated over several rounds. The card's name, power limit and SM clock are printed with the numbers. Needs a GPU.

    python tools/time_sky.py [--frames N] [--rounds R]"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    from time_display import card
    from zetaray_b200.camera import FrameSequence
    from zetaray_b200.passes import Renderer, Scene
    from tests import scene_util
    assert torch.cuda.is_available(), "time_sky.py measures on the GPU; there is no CPU figure"
    print(json.dumps({"card": card()}))
    W, H = 1920, 1080
    flat = scene_util.SCENES["cornell"]()
    renderers = {}
    for sky in (False, True):
        R = Renderer(Scene(flat), W, H, two_streams=True)
        R.SetSky(sky)
        seq = FrameSequence(W, H)
        for _ in range(5):
            R.Render(seq.next())
        renderers[sky] = (R, seq)
    torch.cuda.synchronize()
    st = torch.cuda.current_stream()
    for rnd in range(args.rounds):
        for sky in (False, True):
            R, seq = renderers[sky]
            fcs = [seq.next() for _ in range(args.frames)]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for fc in fcs:
                R.Render(fc, C.c_void_p(st.cuda_stream))
            e1.record(st)
            torch.cuda.synchronize()
            print(json.dumps({"round": rnd, "sky": sky, "width": W, "height": H, "frames": args.frames,
                              "frame_ms": e0.elapsed_time(e1) / args.frames}))
    # the kernel alone on an idle device: in the renderer it runs at the side stream's low priority beside the chain
    from zetaray_b200.passes import SkyPass
    from zetaray_b200._lib import FrameInputs
    sky = SkyPass(256, 128)
    fi = FrameInputs()
    fi.frame = seq.next()
    for _ in range(10):
        sky.Render(fi, C.c_void_p(st.cuda_stream))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(args.frames * 4):
        sky.Render(fi, C.c_void_p(st.cuda_stream))
    e1.record(st)
    torch.cuda.synchronize()
    print(json.dumps({"k_sky_view_lut_ms": e0.elapsed_time(e1) / (args.frames * 4), "lut": [256, 128], "launches": args.frames * 4}))

if __name__ == "__main__":
    main()
