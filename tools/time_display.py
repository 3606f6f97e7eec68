"""Times the post-processing kernels (k_lum_histogram, k_exposure, k_display) with CUDA events at 1080p, 1440p and 4K on
seeded synthetic inputs, and prints them against the HBM bound of the bytes each kernel must move: 16 B/px read for the
histogram, 8 B/px read + 4 B/px written for display (the data sheet's 3.35 TB/s for an H100 SXM). Then the editor kernels at
1080p on Cornell: a debug view (k_display_view, NORMAL) and the outline of the largest instance (k_pick_mask, k_outline). The
card's name, power limit and SM clock are printed with the numbers. Needs a GPU.

    python tools/time_display.py [--iters N] [--tonemapper NEUTRAL|AGX_DEFAULT|...]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
BYTES_PER_PX = {"k_lum_histogram": 16, "k_exposure": 0, "k_display": 8 + 4, "k_display_view": 16 + 4}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"name": "unknown"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--tonemapper", default="NEUTRAL")
    args = ap.parse_args()
    import numpy as np
    import torch
    from zetaray_b200 import lib, check, _lib
    from zetaray_b200.camera import look_at_frame_constants
    from zetaray_b200.passes import AutoExposure, Display
    assert torch.cuda.is_available(), "time_display.py measures on the GPU; there is no CPU figure"
    d = np.load(os.path.join(ROOT, "tests", "golden", "tony_mc_mapface.npz"))
    lut = np.ascontiguousarray(d["lut"], dtype=np.uint32)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    st = C.c_void_p(stream.cuda_stream)
    info = card()
    print(json.dumps({"card": info}))
    for name, (W, H) in (("1080p", (1920, 1080)), ("1440p", (2560, 1440)), ("4K", (3840, 2160))):
        g = torch.Generator(device="cuda").manual_seed(1)
        sig = torch.rand((H * W, 4), device="cuda", generator=g) * 4.0
        taa = (torch.rand((H * W, 4), device="cuda", generator=g) * 20.0).half()
        ae, disp = AutoExposure(W, H), Display(W, H)
        disp.SetLUT(lut)
        disp.SetParams(tonemapper=getattr(Display, args.tonemapper))
        fi = _lib.FrameInputs()
        fi.frame = look_at_frame_constants(W, H)
        fi.frame.dt = 1 / 60
        exposure = ae.GetOutput().d_ptr

        def frame():
            ae.Render(fi, sig.data_ptr(), st)
            disp.Render(fi, taa.data_ptr(), exposure, st)

        print(json.dumps({"size": name, "width": W, "height": H, "tonemapper": args.tonemapper, "iters": args.iters,
                          "kernels": profile(frame, args.iters, W, H)}))
        del ae, disp
    # editor kernels: Cornell at 1080p, the NORMAL view and the outline of the instance with the most triangles
    from zetaray_b200.passes import Scene, GBuffers, GBufferRT
    from tests import scene_util
    W, H = 1920, 1080
    flat = scene_util.cornell()
    scene = Scene(flat)
    gb, gpass = GBuffers(W, H), GBufferRT()
    fi = _lib.FrameInputs()
    fi.frame = look_at_frame_constants(W, H)
    gb.fill_inputs(fi)
    fi.scene = scene.handle
    gpass.Render(fi, st)
    largest = int(np.argmax(flat.instance_num_tris))
    disp = Display(W, H)
    disp.SetView(Display.VIEW_NORMAL)
    disp.SetPicked([largest])
    print(json.dumps({"size": "1080p", "scene": "cornell", "view": "NORMAL", "picked": largest,
                      "picked_tris": int(flat.instance_num_tris[largest]), "iters": args.iters,
                      "kernels": profile(lambda: disp.Render(fi, None, None, st), args.iters, W, H)}))


def profile(frame, iters, W, H):
    """{kernel: mean time per call} over `iters` calls of frame() after 10 warm-up calls"""
    import torch
    from zetaray_b200 import lib, check
    for _ in range(10):
        frame()
    torch.cuda.synchronize()
    check(lib.zr_profile_enable(1))
    for _ in range(iters):
        frame()
    buf = C.create_string_buffer(4096)
    check(lib.zr_profile_collect(buf, 4096))
    check(lib.zr_profile_enable(0))
    kernels = {}
    for k, calls, total in (x.split(":") for x in buf.value.decode().split(";") if x):
        us = float(total) * 1e3 / int(calls)
        kernels[k] = {"us": round(us, 2)}
        if k in BYTES_PER_PX:
            bound_us = BYTES_PER_PX[k] * W * H / HBM_BYTES_PER_S * 1e6
            kernels[k].update(bytes_per_px=BYTES_PER_PX[k], hbm_bound_us=round(bound_us, 2),
                              share_of_hbm_bound=round(bound_us / us, 3) if bound_us else None)
    return kernels


if __name__ == "__main__":
    main()
