"""Times k_rpt_debug_view per frame at 1080p with zr_profile_* (CUDA events around every launch): the glossy scene, ReSTIR PT
under each reuse setting with the K view on, after warm-up frames with it. The card's name, power limit and SM clock are printed
with the numbers. Needs a GPU.

    python tools/time_rpt_debug_view.py [--frames N]"""
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
    ap.add_argument("--frames", type=int, default=20)
    args = ap.parse_args()
    import torch
    from time_display import card
    from zetaray_b200 import lib, check
    from zetaray_b200.camera import FrameSequence
    from tests import scene_util
    from tests.parity import DeviceFrame
    from tests.rpt_debug_view_util import K, REUSE
    assert torch.cuda.is_available(), "time_rpt_debug_view.py measures on the GPU; there is no CPU figure"
    print(json.dumps({"card": card()}))
    W, H = 1920, 1080
    for reuse, params in REUSE.items():
        f = DeviceFrame(scene_util.SCENES["glossy"](), W, H, ("rpt",), rpt_params=params)
        f.rpt.SetDebugView(K)
        seq = FrameSequence(W, H)
        for _ in range(3):
            f.render(seq.next())
        check(lib.zr_profile_enable(1))
        for _ in range(args.frames):
            f.render(seq.next())
        buf = C.create_string_buffer(1 << 16)
        check(lib.zr_profile_collect(buf, len(buf)))
        check(lib.zr_profile_enable(0))
        kernels = {}
        for item in buf.value.decode().split(";"):
            if item:
                name, calls, ms = item.split(":")
                kernels[name] = {"calls": int(calls), "ms_per_frame": float(ms) / args.frames}
        print(json.dumps({"reuse": reuse, "width": W, "height": H, "frames": args.frames, "view": "K",
                          "k_rpt_debug_view": kernels.get("k_rpt_debug_view"),
                          "frame_ms_sum": sum(k["ms_per_frame"] for k in kernels.values())}))
        f.close()


if __name__ == "__main__":
    main()
