"""Rays per second of the BVH traversal alone (zr_scene_trace_closest / zr_scene_trace_any, i.e. zr_scene.cuh::Traverse) on Cornell,
the procedural atrium (C4 stand-in, 3 x 10^5 triangles) and the procedural tunnel (C5 stand-in, 10^6 triangles).

    python tools/time_traversal.py [scene ...] [--iters N] [--seed S]

The three ray sets are built on the device from a seed, the way tests/test_bvh_quality.py's ray_sets builds them: primary rays
through the pixel centres of a 1920 x 1080 image from the scene's camera (closest hit), cosine-distributed secondary rays from the
primary hits (closest hit) and shadow segments from the primary hits to the first vertex of a random emissive triangle (any hit),
about 2 M rays per set. Each set is traced a few times to warm up, then N times between CUDA events. Prints one JSON line with the
device name, its power limit and SM clock next to the numbers."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from zetaray_b200 import lib, check, procedural  # noqa: E402
from zetaray_b200.passes import Scene  # noqa: E402
from zetaray_b200.scene import FlatScene, quat_rotate_np  # noqa: E402

W, H = 1920, 1080
CORNELL_CAMERA = (0.0, 1.2, -4.043)


def load(name):
    if name == "cornell":
        return FlatScene.load(os.path.join(ROOT, "tests", "golden", "cornell_emissive.npz")), CORNELL_CAMERA
    make, cam = procedural.SCENES[name]
    return make(1.0), cam


def geometric_normals(flat):
    """Unit geometric normal per global triangle, in float64 with the instances' quantised rotation / half scale (the normals only
    orient the secondary and shadow rays, they need not match the device's world triangles bit for bit)."""
    out = []
    for inst, nt in zip(flat.instances, flat.instance_num_tris):
        idx = flat.indices[int(inst["BaseIdxOffset"]):int(inst["BaseIdxOffset"]) + 3 * int(nt)].astype(np.int64) + int(inst["BaseVtxOffset"])
        q = (inst["Rotation"].astype(np.float64) / 65535.0) * 2.0 - 1.0
        q /= np.linalg.norm(q)
        s = inst["Scale"].view(np.float16).astype(np.float64)
        p = quat_rotate_np(q, flat.vertices["pos"][idx].astype(np.float64) * s).reshape(-1, 3, 3)
        out.append(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]))
    n = np.concatenate(out)
    return n / (np.linalg.norm(n, axis=1, keepdims=True) + 1e-30)


def ray_sets(flat, cam, sc, seed):
    dev = "cuda"
    tan = np.tan(0.5 * np.pi / 3)
    xs = ((torch.arange(W, device=dev, dtype=torch.float64) + 0.5) / W * 2 - 1) * tan * (W / H)
    ys = (1 - (torch.arange(H, device=dev, dtype=torch.float64) + 0.5) / H * 2) * tan
    Y, X = torch.meshgrid(ys, xs, indexing="ij")
    d = torch.stack([X, Y, torch.ones_like(X)], -1).reshape(-1, 3)
    d = d / d.norm(dim=1, keepdim=True)
    prim = torch.zeros((W * H, 8), dtype=torch.float32, device=dev)
    prim[:, 0:3] = torch.tensor(cam, dtype=torch.float32, device=dev); prim[:, 3] = 1e-4; prim[:, 4:7] = d.float(); prim[:, 7] = 3.0e38
    hits = trace(sc, prim, anyhit=False)
    torch.cuda.synchronize()
    ok = hits[:, 0] < 3e38
    tri = hits[ok, 3].contiguous().view(torch.int32).long()
    P = prim[ok, 0:3].double() + prim[ok, 4:7].double() * hits[ok, 0:1].double()
    ng = torch.from_numpy(geometric_normals(flat)).to(dev)[tri]
    ng = torch.where(((ng * prim[ok, 4:7].double()).sum(1) > 0)[:, None], -ng, ng)
    gen = torch.Generator(device=dev).manual_seed(seed)
    m = len(P)
    u = torch.rand((m, 2), generator=gen, device=dev, dtype=torch.float64)
    r = u[:, 0].sqrt(); ph = 2 * np.pi * u[:, 1]
    tmp = torch.where(ng[:, 0:1].abs() < 0.9, torch.tensor([[1.0, 0, 0]], device=dev, dtype=torch.float64),
                      torch.tensor([[0, 1.0, 0]], device=dev, dtype=torch.float64))
    t1 = torch.linalg.cross(ng, tmp); t1 = t1 / t1.norm(dim=1, keepdim=True)
    t2 = torch.linalg.cross(ng, t1)
    wi = (r * ph.cos())[:, None] * t1 + (r * ph.sin())[:, None] * t2 + (1 - u[:, 0]).sqrt()[:, None] * ng
    sec = torch.zeros((m, 8), dtype=torch.float32, device=dev)
    sec[:, 0:3] = (P + 1e-3 * ng).float(); sec[:, 3] = 1e-6; sec[:, 4:7] = wi.float(); sec[:, 7] = 3e38
    Lv = torch.from_numpy(flat.emissives["Vtx0"].astype(np.float64)).to(dev)
    L = Lv[torch.randint(0, len(Lv), (m,), generator=gen, device=dev)]
    dd = L - P
    ln = dd.norm(dim=1, keepdim=True)
    sh = torch.zeros((m, 8), dtype=torch.float32, device=dev)
    sh[:, 0:3] = (P + 1e-3 * ng).float(); sh[:, 3] = 3e-6; sh[:, 4:7] = (dd / ln).float(); sh[:, 7] = (ln[:, 0] * 0.999).float()
    return (("primary", prim, False), ("secondary", sec, False), ("shadow", sh, True))


def trace(sc, rays, anyhit, out=None):
    n = len(rays)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if anyhit:
        out = out if out is not None else torch.empty(n, dtype=torch.int32, device="cuda")
        check(lib.zr_scene_trace_any(sc.handle, C.c_void_p(rays.data_ptr()), n, C.c_void_p(out.data_ptr()), st))
    else:
        out = out if out is not None else torch.empty((n, 4), dtype=torch.float32, device="cuda")
        check(lib.zr_scene_trace_closest(sc.handle, C.c_void_p(rays.data_ptr()), n, C.c_void_p(out.data_ptr()), st))
    return out


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = [x.strip() for x in q.split(",")]
    except Exception as e:      # the numbers still stand; say why the card's settings are missing
        info["nvidia_smi"] = "unavailable: %s" % e
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("scenes", nargs="*", default=["cornell", "atrium", "tunnel"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_traversal.py times the device traversal and needs a GPU"
    torch.cuda.set_device(0)
    result = {"what": "BVH traversal rays/s (zr_scene_trace_closest / zr_scene_trace_any), %d x %d camera, CUDA events" % (W, H),
              "iters": args.iters, "seed": args.seed, "scenes": {}}
    for name in args.scenes:
        flat, cam = load(name)
        sc = Scene(flat)
        per = {"bvh": sc.bvh_stats()}
        for label, rays, anyhit in ray_sets(flat, cam, sc, args.seed):
            out = trace(sc, rays, anyhit)
            for _ in range(3):
                trace(sc, rays, anyhit, out)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                trace(sc, rays, anyhit, out)
            e1.record()
            e1.synchronize()
            ms = e0.elapsed_time(e1) / args.iters
            per[label] = {"rays": len(rays), "query": "any" if anyhit else "closest", "ms": round(ms, 4),
                          "Mrays_per_s": round(len(rays) / ms / 1e3, 1)}
        result["scenes"][name] = per
        del sc
    result.update(device_info())
    print(json.dumps(result))


if __name__ == "__main__":
    main()
