"""Drives the CPU oracle through whole frames (G-buffer -> ReSTIR DI / PT -> post) for parity tests,
smoke() and bench.py's cpu_baseline leg."""
import ctypes as C
import os
import numpy as np

from tests import scene_util, synth
from tests.orc import RptBuffers, ptr
from zetaray_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES = np.dtype([("meta", "<u4"), ("w_sum", "<f4"), ("W", "<f4"), ("L_b", "<u4"),
                ("jacobian_or_seed_nee", "<u4"), ("seed_replay", "<u4"), ("ID", "<u4"), ("x_k_x", "<u4"),
                ("x_k_y", "<u4"), ("x_k_z", "<u4"), ("w_k", "<u4"), ("L_rg", "<u4"),
                ("lightPdf", "<f4"), ("dwdA", "<f4"), ("seed_nee", "<u4"), ("meshIdx", "<u4")])
assert RES.itemsize == 64


def default_rpt_params():
    # IndirectLighting.h:231-244, IndirectLighting.cpp:146-165
    return _lib.IndirectParams(3, 4, 1, 1, 1, 10, 8, 1, 1, 1, np.float32(0.175) * np.float32(0.175))


RDI = np.dtype([("bary", "<u4"), ("le_rg", "<u4"), ("le_b_meta", "<u4"), ("lightIdx", "<u4"), ("w_sum", "<f4"), ("W", "<f4"),
                ("pad0", "<u4"), ("pad1", "<u4")])
assert RDI.itemsize == 32


def default_rdi_params():
    # DirectLighting.cpp:99-107, DirectLighting.h:93-98
    return _lib.DirectParams(1, 1, 1, 1, 20, np.float32(0.05) * np.float32(0.05))


RGI = np.dtype([("pos", "<f4", 3), ("ID", "<u4"), ("Lo_rg", "<u4"), ("Lo_b_M", "<u4"), ("w_sum", "<f4"), ("W", "<f4"),
                ("normal", "<u4"), ("pad", "<u4", 3)])
assert RGI.itemsize == 48


def default_gi_params():
    # IndirectLighting.h:231-244
    return _lib.GIParams(max_non_tr_bounces=3, max_glossy_tr_bounces=4, russian_roulette=1, stochastic_multi_bounce=1,
                         boiling_suppression=1, M_max=10, temporal_resample=1)


from zetaray_b200.camera import halton, FrameSequence  # noqa: E402,F401  (moved into the package)


class OracleRenderer:
    """Reference-shaped frame loop on the CPU oracle."""

    def __init__(self, flat, w, h, nthreads=None):
        # results do not depend on the thread count (scan-line parallel, per-pixel state only); large frames use every core
        if nthreads is None:
            nthreads = 8 if w * h <= 512 * 512 else max(8, min(os.cpu_count() or 8, 128))
        self.osc = scene_util.OracleScene(flat)
        self.o = self.osc.o
        self.w, self.h, self.nthreads = w, h, nthreads
        n = w * h
        self.pattern = np.fromfile(os.path.join(ROOT, "zetaray_b200", "assets", "disk512.bin"), dtype=np.float32)
        assert self.pattern.size == 1024
        self.o.orc_rpt_set_sample_pattern(ptr(self.pattern))
        self.cur = 0
        self.res = [np.zeros(n, dtype=RES), np.zeros(n, dtype=RES)]
        self.target = np.zeros((n, 4), dtype=np.float32)
        self.final = np.zeros((n, 4), dtype=np.float32)
        self.neighbor = np.zeros(n, dtype=np.uint16)
        self.tmCtN = np.zeros(n, dtype=np.uint16)
        self.tmNtC = np.zeros(n, dtype=np.uint16)
        self.state = np.array([0, 0, 1], dtype=np.uint32)     # currTemporalIdx, temporalValid, resetFlag
        self.params = default_rpt_params()
        self.pattern32 = np.fromfile(os.path.join(ROOT, "zetaray_b200", "assets", "disk32.bin"), dtype=np.float32)
        assert self.pattern32.size == 64
        self.o.orc_rdi_set_sample_pattern(ptr(self.pattern32))
        self.di_res = [np.zeros(n, dtype=RDI), np.zeros(n, dtype=RDI)]
        self.di_target = np.zeros((n, 2), dtype=np.uint32)
        self.di_final = np.zeros((n, 4), dtype=np.float32)
        self.di_state = np.array([0, 0, 1], dtype=np.uint32)
        self.di_params = default_rdi_params()
        self.gi_params = default_gi_params()
        self.gi_res = [np.zeros(n, dtype=RGI), np.zeros(n, dtype=RGI)]
        self.gi_final = np.zeros((n, 4), dtype=np.float32)
        self.gi_state = np.array([0, 0, 1], dtype=np.uint32)
        empty = (np.zeros((n, 4), np.uint32), np.zeros(n, np.float32), np.zeros((n, 2), np.uint32), np.zeros((n, 2), np.uint32), None)
        self.gb = [empty, empty]

    def gbuffer(self, fc):
        self.osc.presample(fc.FrameNum)       # PreLighting runs before the lighting passes; no-op unless presampling is on
        self.osc.build_light_voxel_grid(fc)   # no-op unless the light voxel grid is on
        self.cur ^= 1
        self.gb[self.cur] = self.osc.gbuffer(fc, tridiff=False, nthreads=self.nthreads)
        return self.gb[self.cur]

    def rpt(self, fc, last_stage=0):
        c = self.gb[self.cur]; p = self.gb[self.cur ^ 1]
        b = RptBuffers((self.res[0].ctypes.data, self.res[1].ctypes.data), self.target.ctypes.data, self.final.ctypes.data,
                       self.neighbor.ctypes.data, self.tmCtN.ctypes.data, self.tmNtC.ctypes.data)
        self.o.orc_rpt_render(self.osc.h, C.byref(fc), ptr(c[0]), ptr(c[2]), ptr(c[3]), ptr(p[0]), ptr(p[3]),
                              C.byref(self.params), C.byref(b), ptr(self.state), last_stage, self.nthreads)

    def rdi(self, fc):
        c = self.gb[self.cur]; p = self.gb[self.cur ^ 1]
        self.o.orc_rdi_render(self.osc.h, C.byref(fc), ptr(c[0]), ptr(c[2]), ptr(c[3]), ptr(p[0]), ptr(p[3]), C.byref(self.di_params),
                              ptr(self.di_res[0]), ptr(self.di_res[1]), ptr(self.di_target), ptr(self.di_final), ptr(self.di_state),
                              self.nthreads)

    def rgi(self, fc):
        """IndirectLighting with INTEGRATOR::ReSTIR_GI"""
        c = self.gb[self.cur]; p = self.gb[self.cur ^ 1]
        self.o.orc_rgi_render(self.osc.h, C.byref(fc), ptr(c[0]), ptr(c[2]), ptr(c[3]), ptr(p[0]), ptr(p[3]), C.byref(self.gi_params),
                              ptr(self.gi_res[0]), ptr(self.gi_res[1]), ptr(self.gi_final), ptr(self.gi_state), self.nthreads)

    def pt(self, fc):
        """IndirectLighting with INTEGRATOR::PATH_TRACING (the plain path tracer); writes gi_final like rgi()."""
        c = self.gb[self.cur]
        self.o.orc_pt_render(self.osc.h, C.byref(fc), ptr(c[0]), ptr(c[2]), ptr(c[3]), C.byref(self.gi_params), ptr(self.gi_final),
                             self.nthreads)

    def gi_curr_reservoirs(self):
        return self.gi_res[1 - int(self.gi_state[0])]

    def di_curr_reservoirs(self):
        return self.di_res[1 - int(self.di_state[0])]

    def post(self, fc, taa_prev, taa_valid, firefly=True):
        """Compositing (+ firefly) and TAA on the oracle; returns (composited float4, taa half4)."""
        n = self.w * self.h
        c = self.gb[self.cur]
        comp = np.zeros((n, 4), dtype=np.float32)
        self.o.orc_compositing(C.byref(fc), ptr(c[0]), ptr(self.di_final), ptr(self.final), ptr(comp))
        if firefly:
            out = np.zeros((n, 4), dtype=np.float32)
            self.o.orc_firefly(C.byref(fc), ptr(c[0]), ptr(comp), ptr(out))
            comp = out
        taa = np.zeros((n, 2), dtype=np.uint32)
        self.o.orc_taa(C.byref(fc), ptr(c[0]), ptr(c[2]), ptr(comp), ptr(taa_prev), ptr(taa), 0.1, int(taa_valid))
        return comp, taa

    def curr_reservoirs(self):
        """The buffer holding this frame's output == next frame's 'previous' (state[0] was advanced)."""
        return self.res[1 - int(self.state[0])]
