"""Device-vs-oracle frame parity for the GPU tests and smoke(): the same frames rendered by the CPU oracle
(rpt_util.OracleRenderer) and by the device passes, every compared plane byte for byte."""
import numpy as np

from tests import rpt_util, scene_util
from zetaray_b200 import _lib, check, lib
from zetaray_b200.passes import (Scene, GBuffers, GBufferRT, DirectLighting, IndirectLighting, IndirectLightingGI, Compositing, TAA,
                                 download_image)


def diff_report(name, a, b):
    """None when a and b hold the same bytes, else where they differ: structured records field by field, plain arrays (flat or
    shaped) row by row."""
    if a.tobytes() == b.tobytes():
        return None
    if a.dtype.fields is not None:
        bad = {f: int((a[f] != b[f]).sum()) for f in a.dtype.names}
        first = int(np.nonzero(a != b)[0][0])
        return "%s differs: per-field mismatches %s; first idx %d got %s want %s" % (
            name, {f: n for f, n in bad.items() if n}, first, a[first], b[first])
    a, b = np.ascontiguousarray(a).reshape(len(a), -1), np.ascontiguousarray(b).reshape(len(b), -1)
    d = np.nonzero((a != b).any(axis=1))[0]
    return "%s differs at %d/%d entries; first idx %d got %s want %s" % (name, len(d), len(a), d[0], a[d[0]], b[d[0]])


# ---- output planes: texel layout and record type of each kind, as the oracle holds them --------------------------------------------
def _records(img, dtype):
    return download_image(img, np.uint8, dtype.itemsize).view(dtype).reshape(-1)


def di_reservoirs(img):
    return _records(img, rpt_util.RDI)


def pt_reservoirs(img):
    return _records(img, rpt_util.RES)


def gi_reservoirs(img):
    return _records(img, rpt_util.RGI)


def rgba32f_bits(img):
    """An RGBA32F plane (lighting finals, the composited image, the ReSTIR PT target) as uint32 bits."""
    return download_image(img, np.uint32, 4)


def uint32x2(img):
    """8-byte texels: the TAA image (RGBA16F) and the ReSTIR DI target."""
    return download_image(img, np.uint32, 2)


def uint16_plane(img):
    """The ReSTIR PT neighbour and thread-map planes."""
    return download_image(img, np.uint16, 1).reshape(-1)


# ---- the device frame ---------------------------------------------------------------------------------------------------------------
# "rdi": ReSTIR DI; "rpt": ReSTIR PT; "rgi": ReSTIR GI; "pt": the plain path tracer; "post": compositing + TAA (needs rdi and rpt)
WHOLE_FRAME = ("rdi", "rpt", "post")


class DeviceFrame:
    """The device side of a frame: the scene, the two G-buffers, GBufferRT and the requested lighting and post passes."""

    def __init__(self, flat, w, h, passes, di_params=None, rpt_params=None, gi_params=None, presample=None, lvg=None):
        self.scene = Scene(flat)
        self.scene.prelighting()
        if presample:
            self.scene.set_presampling(*presample)
        if lvg:
            self.scene.set_light_voxel_grid(*lvg)
        self.gb, self.gpass = GBuffers(w, h), GBufferRT()
        self.di = DirectLighting(w, h) if "rdi" in passes else None
        self.rpt = IndirectLighting(w, h) if "rpt" in passes else None
        self.gi = IndirectLightingGI(w, h) if "rgi" in passes or "pt" in passes else None
        self.comp, self.taa = (Compositing(w, h), TAA(w, h)) if "post" in passes else (None, None)
        if "pt" in passes:
            self.gi.SetMethod(IndirectLightingGI.PATH_TRACING)
        for p, params in ((self.di, di_params), (self.rpt, rpt_params), (self.gi, gi_params)):
            if params:
                p.SetParams(**params)

    def render(self, fc):
        """One frame in the product's order; returns its FrameInputs."""
        self.gb.flip()
        fi = _lib.FrameInputs()
        fi.frame = fc
        self.gb.fill_inputs(fi)
        fi.scene = self.scene.handle
        self.gpass.Render(fi)
        self.scene.presample(fc.FrameNum)            # both return at once when presampling / the grid is off
        self.scene.build_light_voxel_grid(fc)
        for p in (self.di, self.rpt, self.gi):
            if p:
                p.Render(fi)
        if self.comp:
            self.comp.Render(fi, self.di.GetOutput(0).d_ptr, self.rpt.GetOutput(0).d_ptr)
            self.taa.Render(fi, self.comp.GetOutput().d_ptr)
        check(lib.zr_stream_synchronize(None))
        return fi

    def close(self):
        self.gb.close()


# ---- the comparisons ----------------------------------------------------------------------------------------------------------------
# the planes each set of passes compares by default; "presampled sets" and "light voxel grid" on the first frame only
CHECKS = {("rdi",): ("di_reservoir", "di_final", "di_target"),
          ("rpt",): ("presampled sets", "pt_reservoir", "pt_final", "neighbor", "threadmap_ntc", "target"),
          ("rgi",): ("light voxel grid", "gi reservoir", "gi final"),
          ("pt",): ("path tracer final",),
          WHOLE_FRAME: ("di_reservoir", "di_final", "di_target", "pt_final", "composited", "taa")}
GBUFFER_CHECKS = ("gbuffer core", "gbuffer depth", "gbuffer motion/emissive", "gbuffer coat")


def _planes(f, R, fr, post):
    """(name, device plane reader, oracle plane) of every plane frame fr can compare, in order; a plane whose condition does not
    hold on this frame is left out."""
    gb = R.gb[R.cur]
    out = [("gbuffer core", lambda: f.gb.download("curr")[0], gb[0]),
           ("gbuffer depth", lambda: f.gb.download("curr")[1].view(np.uint32), gb[1].view(np.uint32)),
           ("gbuffer motion/emissive", lambda: f.gb.download("curr")[2], gb[2]),
           ("gbuffer coat", lambda: f.gb.download("curr")[3], gb[3])]
    lvg = getattr(R.osc, "lvg_dim", None)
    if fr == 0 and lvg:
        n = lvg[0] * lvg[1] * lvg[2] * 64 * 8
        out.append(("light voxel grid", lambda: f.scene.light_voxel_grid().reshape(-1, 8), R.osc.lvg[:n].reshape(-1, 8)))
    if f.di:
        out += [("di_reservoir", lambda: di_reservoirs(f.di.GetOutput(1)), R.di_curr_reservoirs()),
                ("di_final", lambda: rgba32f_bits(f.di.GetOutput(0)), R.di_final.view(np.uint32))]
        if fr >= 1 and R.di_params.temporal_resample and R.di_params.spatial_resample:
            out.append(("di_target", lambda: uint32x2(f.di.GetOutput(2)), R.di_target))
    if f.rpt:
        p = R.params
        out += [("pt_reservoir", lambda: pt_reservoirs(f.rpt.GetOutput(1)), R.curr_reservoirs()),
                ("pt_final", lambda: rgba32f_bits(f.rpt.GetOutput(0)), R.final.view(np.uint32))]
        if fr >= 1 and p.num_spatial_passes > 0 and p.temporal_resample:
            out.append(("neighbor", lambda: uint16_plane(f.rpt.GetOutput(4)), R.neighbor))
            if p.sort_spatial:
                out.append(("threadmap_ntc", lambda: uint16_plane(f.rpt.GetOutput(6)), R.tmNtC))
        if fr >= 1 and p.temporal_resample:
            out.append(("target", lambda: rgba32f_bits(f.rpt.GetOutput(3)), R.target.view(np.uint32)))
    if f.gi:
        out += [("gi reservoir", lambda: gi_reservoirs(f.gi.GetOutput(1)), R.gi_curr_reservoirs()),
                ("gi final", lambda: rgba32f_bits(f.gi.GetOutput(0)), R.gi_final.view(np.uint32)),
                ("path tracer final", lambda: rgba32f_bits(f.gi.GetOutput(0)), R.gi_final.view(np.uint32))]
    if f.comp:
        out += [("composited", lambda: rgba32f_bits(f.comp.GetOutput()), post[0].view(np.uint32)),
                ("taa", lambda: uint32x2(f.taa.GetOutput()), post[1])]
    return out


def frame_parity(scene, w, h, nframes, passes, checks=None, di_params=None, rpt_params=None, gi_params=None, presample=None, lvg=None,
                 cam_path=None, accumulate=False, dof=False, nthreads=None):
    """Renders nframes of `scene` (a name in scene_util.SCENES or a FlatScene) on the oracle and on the device with the given
    passes, parameters, presampled sets (num_sets, set_size) and light voxel grid (dims, extents, offset_y), and compares the planes
    named in `checks` (by default CHECKS[passes]) in the order _planes lists them. Stops after the first frame with a difference;
    returns (problems, the OracleRenderer)."""
    checks = checks or CHECKS[tuple(passes)]
    flat = scene_util.SCENES[scene]() if isinstance(scene, str) else scene
    if cam_path is None and isinstance(scene, str) and scene in scene_util.CAMERAS:
        cam = scene_util.CAMERAS[scene]
        cam_path = lambda f: cam
    R = rpt_util.OracleRenderer(flat, w, h, nthreads=nthreads)
    if presample:
        R.osc.set_presampling(*presample)
    if lvg:
        R.osc.set_light_voxel_grid(*lvg)
    for k, v in (di_params or {}).items():
        setattr(R.di_params, k, v)
    for k, v in (rpt_params or {}).items():
        setattr(R.params, k, v)
    R.gi_params.update(gi_params or {})
    f = DeviceFrame(flat, w, h, passes, di_params, rpt_params, gi_params, presample, lvg)
    oracle = [getattr(R, p) for p in ("rdi", "rpt", "rgi", "pt") if p in passes]
    seq = rpt_util.FrameSequence(w, h, cam_path=cam_path, accumulate=accumulate)
    taa_prev, post = np.zeros((w * h, 2), dtype=np.uint32), None
    problems = []
    try:
        for fr in range(nframes):
            fc = seq.next()
            if dof:
                fc.DoF, fc.FocusDepth, fc.LensRadius = 1, 4.0, 0.02
            R.gbuffer(fc)
            for run in oracle:
                run(fc)
            if "post" in passes:
                post = R.post(fc, taa_prev, fr > 0)
                taa_prev = post[1]
            f.render(fc)
            if fr == 0 and presample and "presampled sets" in checks:
                assert f.scene.sample_sets().tobytes() == R.osc.sample_sets[:presample[0] * presample[1] * 10].tobytes(), "presampled sets differ"
            for name, read, want in _planes(f, R, fr, post):
                msg = diff_report(name, read(), want) if name in checks else None
                if msg:
                    problems.append("frame %d: %s" % (fc.FrameNum, msg))
            if problems:
                break
    finally:
        f.close()
    return problems, R
