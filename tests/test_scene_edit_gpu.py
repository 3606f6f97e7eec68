"""zr_scene_update_materials on the device. Every comparison is byte for byte, and "a fresh scene" is zr_scene_create of the
edited arrays (zetaray_b200.scene.update_materials applied to the FlatScene):
  * a light edit leaves the emissive triangles, the power estimate, the alias table and the next frame's presampled sets of the
    fresh scene;
  * frames after an edit with every lighting pass's history reset are the fresh scene's frames (ReSTIR PT, ReSTIR GI, the path
    tracer, ReSTIR DI), also when the edit turns on clear coat in a plain scene;
  * an edit in the middle of a sequence, history kept, gives the oracle's frames with the oracle's scene built from the edited
    arrays from that frame on;
  * every refusal leaves the tables, the alias table and the material features as they were;
  * an edit that changes no emissive bits launches no kernel;
  * strip-sharded frames on two GPUs: both ranks make the same edit, and the frames stay those of one GPU."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import parity, rpt_util, scene_util
from zetaray_b200 import scene as zscene

pytestmark = pytest.mark.gpu

ZR_ERR_INVALID_ARG = 1


def _lights(flat):
    return sorted({int(i["MatIdx"]) for i in flat.instances if int(i["BaseEmissiveTriOffset"]) != 0xffffffff})


def _light_edits():
    """(scene name, first material, edited materials): colour, strength, strength to zero on one of several lights, and a light
    turned single-sided together with a non-emissive neighbour."""
    return {
        "cornell colour": ("cornell", 5, [zscene.make_material(emissive_factor=(0.9, 0.3, 0.1), emissive_strength=40.0, double_sided=True)]),
        "cornell strength": ("cornell", 5, [zscene.make_material(emissive_factor=(1.0, 0.776, 0.616), emissive_strength=3.5)]),
        "atrium one light off": ("atrium", None, "off"),
        "atrium two": ("atrium", None, "pair"),
    }


def _resolve(name, first, mats):
    flat = scene_util.SCENES[name]()
    lights = _lights(flat)
    if mats == "off":
        first, mats = lights[1], [zscene.make_material(emissive_factor=(0.8, 0.8, 0.5), emissive_strength=0.0)]
    elif mats == "pair":
        first = lights[0] - 1
        mats = [zscene.make_material(base_color=(0.2, 0.6, 0.3), roughness=0.4),
                zscene.make_material(emissive_factor=(0.25, 0.5, 1.0), emissive_strength=12.0, double_sided=False)]
    return flat, first, mats


def _power(scene):
    import torch
    from zetaray_b200 import lib, check
    n = len(scene.tables()[1])
    d = torch.zeros(max(n, 1), dtype=torch.float32, device="cuda")
    check(lib.zr_estimate_emissive_power(scene.handle, C.c_void_p(d.data_ptr()), None))
    torch.cuda.synchronize()
    return d.cpu().numpy()


def _state(scene):
    m, e = scene.tables()
    return {"materials": m.tobytes(), "emissives": e.tobytes(), "power": _power(scene).tobytes(),
            "alias": scene.alias_table().tobytes(), "features": scene.material_features()}


@pytest.mark.parametrize("case", list(_light_edits()))
def test_light_edit_equals_fresh_scene(case):
    from zetaray_b200.passes import Scene
    flat, first, mats = _resolve(*_light_edits()[case])
    edited = zscene.update_materials(flat, first, mats)
    A, B = Scene(flat), Scene(edited)
    for s in (A, B):
        s.prelighting()
        s.set_presampling(8, 128)
    A.presample(1)
    before = _state(A)
    A.update_materials(first, mats)
    after, want = _state(A), _state(B)
    assert after["emissives"] != before["emissives"]
    for k in want:
        assert after[k] == want[k], k
    A.presample(2); B.presample(2)
    assert A.sample_sets().tobytes() == B.sample_sets().tobytes()


def _outputs(f):
    out = {}
    if f.di:
        out["di final"], out["di reservoirs"] = parity.rgba32f_bits(f.di.GetOutput(0)), parity.di_reservoirs(f.di.GetOutput(1))
    if f.rpt:
        out["pt final"], out["pt reservoirs"] = parity.rgba32f_bits(f.rpt.GetOutput(0)), parity.pt_reservoirs(f.rpt.GetOutput(1))
    if f.gi:
        out["gi final"], out["gi reservoirs"] = parity.rgba32f_bits(f.gi.GetOutput(0)), parity.gi_reservoirs(f.gi.GetOutput(1))
    out["gbuffer"] = np.concatenate([p.reshape(len(p), -1).view(np.uint32) for p in f.gb.download("curr")[:4]], axis=1)
    return out


RESET_CASES = {
    "rpt light": (("rdi", "rpt"), "cornell", 5, [zscene.make_material(emissive_factor=(0.9, 0.3, 0.1), emissive_strength=25.0)]),
    "rgi light": (("rgi",), "cornell", 5, [zscene.make_material(emissive_factor=(0.2, 0.9, 0.4), emissive_strength=60.0)]),
    "pt light": (("pt",), "cornell", 5, [zscene.make_material(emissive_factor=(0.5, 0.5, 1.0), emissive_strength=8.0, double_sided=True)]),
    "rpt coat": (("rdi", "rpt"), "cornell", 3, [zscene.make_material(base_color=(0.2, 0.3, 0.7), roughness=0.6, coat_weight=1.0,
                                                                      coat_roughness=0.1, double_sided=True)]),
}


@pytest.mark.parametrize("case", list(RESET_CASES))
def test_frames_after_edit_and_reset_equal_fresh_scene(case):
    """Two frames, the edit, every lighting pass's history reset, three more frames: the same planes as a fresh scene and fresh
    passes rendering those three frames. The coat case turns a plain scene (the lighting passes' plain build) into a coated one."""
    from zetaray_b200.camera import FrameSequence
    passes, name, first, mats = RESET_CASES[case]
    flat = scene_util.SCENES[name]()
    edited = zscene.update_materials(flat, first, mats)
    W, H, warm, frames = 160, 96, 2, 3
    A = parity.DeviceFrame(flat, W, H, passes)
    seqA = FrameSequence(W, H, jitter=False)
    try:
        for _ in range(warm):
            A.render(seqA.next())
        features = A.scene.material_features()
        A.scene.update_materials(first, mats)
        for p in (A.di, A.rpt, A.gi):
            if p:
                p.ResetTemporal()
        if case == "rpt coat":
            assert features == 0 and A.scene.material_features() != 0
        B = parity.DeviceFrame(edited, W, H, passes)
        seqB = FrameSequence(W, H, jitter=False, first_frame=warm + 1)
        try:
            for fr in range(frames):
                A.render(seqA.next()); B.render(seqB.next())
                got, want = _outputs(A), _outputs(B)
                for k in want:
                    msg = parity.diff_report(k, got[k], want[k])
                    assert msg is None, "frame %d after the edit: %s" % (fr, msg)
        finally:
            B.close()
    finally:
        A.close()


def test_edit_mid_sequence_equals_oracle():
    """ReSTIR DI + ReSTIR PT + compositing + TAA on the atrium with the parity harness's planes: two frames, then a light edit
    with all history kept, then two more frames, the oracle's scene built from the edited arrays from the edit on."""
    flat = scene_util.SCENES["atrium"]()
    lights = _lights(flat)
    first, mats = lights[2], [zscene.make_material(emissive_factor=(1.0, 0.2, 0.1), emissive_strength=30.0, double_sided=True)]
    edited = zscene.update_materials(flat, first, mats)
    W, H = 96, 64
    cam = scene_util.CAMERAS["atrium"]
    R = rpt_util.OracleRenderer(flat, W, H)
    f = parity.DeviceFrame(flat, W, H, parity.WHOLE_FRAME)
    seq = rpt_util.FrameSequence(W, H, cam_path=lambda fr: cam)
    checks = parity.CHECKS[parity.WHOLE_FRAME]
    taa_prev = np.zeros((W * H, 2), dtype=np.uint32)
    try:
        for fr in range(4):
            if fr == 2:
                f.scene.update_materials(first, mats)
                R.osc = scene_util.OracleScene(edited)
            fc = seq.next()
            R.gbuffer(fc)
            R.rdi(fc)
            R.rpt(fc)
            post = R.post(fc, taa_prev, fr > 0)
            taa_prev = post[1]
            f.render(fc)
            for name, read, want in parity._planes(f, R, fr, post):
                if name in checks:
                    msg = parity.diff_report(name, read(), want)
                    assert msg is None, "frame %d: %s" % (fc.FrameNum, msg)
    finally:
        f.close()


def test_refusals_change_nothing():
    from zetaray_b200 import lib
    from zetaray_b200.passes import Scene
    flat = scene_util.cornell()
    s = Scene(flat)
    s.prelighting()
    light = _lights(flat)[0]
    before = _state(s)
    n = len(flat.materials)
    one = np.ascontiguousarray(zscene.make_material(roughness=0.9)[None])
    lit = np.ascontiguousarray(zscene.make_material(emissive_factor=(1, 1, 1), emissive_strength=2.0)[None])
    off = np.ascontiguousarray(zscene.make_material(emissive_factor=(1, 1, 1), emissive_strength=0.0)[None])
    dark = np.ascontiguousarray(zscene.make_material(emissive_factor=(0, 0, 0), emissive_strength=5.0)[None])
    two = np.ascontiguousarray(np.concatenate([one, one]))
    cases = {"null scene": (None, 0, 1, one, "null scene"), "null materials": (s.handle, 0, 1, None, "null scene"),
             "count 0": (s.handle, 0, 0, one, "count == 0"), "past the table": (s.handle, n - 1, 2, two, "lie past"),
             "32-bit overflow": (s.handle, 0xffffffff, 2, two, "lie past"), "new light": (s.handle, 0, 1, lit, "has no emissive triangles"),
             "light strength 0": (s.handle, light, 1, off, "zero power"), "light factor 0": (s.handle, light, 1, dark, "zero power")}
    for what, (h, first, count, m, msg) in cases.items():
        st = lib.zr_scene_update_materials(h, first, count, None if m is None else m.ctypes.data_as(C.c_void_p), None)
        assert st == ZR_ERR_INVALID_ARG, what
        err = lib.zr_last_error()
        assert err.startswith(b"zr_scene_update_materials: ") and msg.encode() in err, (what, err)
        assert _state(s) == before, what


def test_non_emissive_edit_launches_no_kernel():
    """A roughness edit launches nothing; a light edit launches the refresh, the power estimate and the alias build."""
    import torch
    from zetaray_b200 import lib, check
    from zetaray_b200.passes import Scene
    flat = scene_util.cornell()
    s = Scene(flat)
    s.prelighting()
    torch.cuda.synchronize()
    n0 = lib.zr_kernel_launch_count()
    s.update_materials(2, [zscene.make_material(base_color=(0.1, 0.8, 0.1), roughness=0.05)])
    # a light material with the same emissive bits but a new base colour changes no emissive triangle either
    same = flat.materials[5].copy()
    same["BaseColorFactor"] = zscene.rgba8((0.3, 0.3, 0.3, 1.0))
    s.update_materials(5, [same])
    assert lib.zr_kernel_launch_count() == n0
    check(lib.zr_profile_enable(1))
    try:
        s.update_materials(5, [zscene.make_material(emissive_factor=(0.5, 0.5, 0.5), emissive_strength=9.0)])
        buf = C.create_string_buffer(1 << 14)
        check(lib.zr_profile_collect(buf, len(buf)))
    finally:
        check(lib.zr_profile_enable(0))
    names = {e.split(":")[0] for e in buf.value.decode().split(";") if e}
    assert {"k_refresh_emissives", "k_emissive_power", "k_kahan_sum", "k_vose"} <= names, names
    assert lib.zr_kernel_launch_count() == n0 + 7


def _sharded_worker(rank, world, port, out_dir, W=288, H=200, warm=2, frames=3):
    """Both ranks: an unsharded renderer and a strip-sharded one over one scene; after a frame of the cut, the same light edit on
    every rank; every later frame's strip equals the unsharded frame's rows and rank 0's gathered image the whole frame."""
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from zetaray_b200.passes import Scene, Renderer, Comm
        from zetaray_b200.sharding import StripPlan
        from tests.sharded_util import compare_strip, renderer_planes
        stream = torch.cuda.Stream()
        torch.cuda.set_stream(stream)
        st = C.c_void_p(stream.cuda_stream)
        scene = Scene(scene_util.glossy_cornell())
        A = Renderer(scene, W, H, two_streams=False)
        B = Renderer(scene, W, H, two_streams=True)
        comm = Comm.from_torch()
        seq = rpt_util.FrameSequence(W, H)
        for _ in range(warm):
            fc = seq.next()
            A.Render(fc, st); B.Render(fc, st)
        plan = StripPlan.uniform(H, world)
        B.SetShard(comm, plan.bounds, gather_output=True)
        y0, y1 = plan.rows(rank)
        for f in range(frames):
            if f == 1:
                scene.update_materials(5, [zscene.make_material(emissive_factor=(0.3, 0.6, 1.0), emissive_strength=25.0)], st)
            fc = seq.next()
            A.Render(fc, st); B.Render(fc, st)
            torch.cuda.synchronize()
            compare_strip(renderer_planes(B, "pt"), renderer_planes(A, "pt"), y0, y1, "rank %d frame %d" % (rank, f),
                          gathered=rank == 0)
        open(os.path.join(out_dir, "ok%d" % rank), "w").write("%s" % plan.bounds)
    finally:
        dist.destroy_process_group()


def test_sharded_edit_equals_single_gpu(tmp_path):
    from tests.sharded_util import spawn_nccl
    spawn_nccl(_sharded_worker, 2, tmp_path)
