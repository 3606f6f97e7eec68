"""What a material edit between frames costs next to rebuilding the scene: on Cornell, the procedural atrium and the tunnel (full
size, as tools/bench_scenes.py builds them), the device time of zr_scene_update_materials (CUDA events on the call's stream) for a
light edit, which refreshes the light's emissive triangles and rebuilds the power estimate and alias table, and for a non-emissive
edit, which copies one material; and the host time of zr_scene_create of the same scene (BVH build included), the alternative
without the edit. Prints one JSON line per scene with the card's name and power limit read in the same run.

    python tools/time_scene_edit.py [--reps 20] [cornell atrium tunnel]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"name": "unknown"}


def load(name):
    from zetaray_b200 import procedural
    from zetaray_b200.scene import FlatScene
    if name == "cornell":
        return FlatScene.load(os.path.join(ROOT, "tests", "golden", "cornell_emissive.npz"))
    return procedural.SCENES[name][0](1.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("scenes", nargs="*", default=["cornell", "atrium", "tunnel"])
    args = ap.parse_args()
    import numpy as np
    import torch
    from zetaray_b200.passes import Scene
    from zetaray_b200 import scene as zscene
    assert torch.cuda.is_available(), "time_scene_edit.py measures on the GPU"
    info = card()
    stream = torch.cuda.Stream()
    st = C.c_void_p(stream.cuda_stream)
    for name in args.scenes:
        flat = load(name)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sc = Scene(flat)
        torch.cuda.synchronize()
        t_create = time.perf_counter() - t0
        sc.prelighting(st)
        lit = [int(i["MatIdx"]) for i in flat.instances if int(i["BaseEmissiveTriOffset"]) != 0xffffffff]
        light = max(set(lit), key=lit.count)            # the light material with the most instances
        plain = next(int(i["MatIdx"]) for i in flat.instances if int(i["BaseEmissiveTriOffset"]) == 0xffffffff)
        n_tris = int(sum(int(nt) for i, nt in zip(flat.instances, flat.instance_num_tris) if int(i["MatIdx"]) == light))

        def light_edit(k):          # alternate two strengths, so every call changes the light's bits
            m = flat.materials[light].copy()
            m["EmissiveStrength_IOR"] = (int(m["EmissiveStrength_IOR"]) & 0xffff0000) | int(zscene.half_bits(4.0 + (k & 1)))
            return m

        def plain_edit(k):
            return zscene.make_material(base_color=(0.2 + 0.1 * (k & 1), 0.5, 0.5), roughness=0.4)

        out = {}
        for what, first, edit in (("light", light, light_edit), ("non_emissive", plain, plain_edit)):
            for k in range(-3, 0):      # warm-up, ending on the other strength so that the first timed edit changes the light
                sc.update_materials(first, [edit(k)], st)
            ms, wall = [], []
            for k in range(args.reps):
                m = edit(k)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                a.record(stream)
                sc.update_materials(first, [m], st)
                b.record(stream)
                b.synchronize()
                wall.append((time.perf_counter() - t0) * 1e3)
                ms.append(a.elapsed_time(b))
            out[what] = dict(device_ms_median=float(np.median(ms)), device_ms_min=float(np.min(ms)), host_ms_median=float(np.median(wall)))
        line = dict(scene=name, triangles=flat.num_triangles, emissive_triangles=len(flat.emissives), light_edit_triangles=n_tris,
                    scene_create_host_ms=t_create * 1e3, update_light_edit=out["light"], update_non_emissive_edit=out["non_emissive"],
                    reps=args.reps, gpu=info.get("name"), power_limit=info.get("power.limit"), max_sm_clock=info.get("clocks.max.sm"))
        print(json.dumps(line), flush=True)
        sc.close()


if __name__ == "__main__":
    main()
