"""ReSTIR PT debug views (zr_rpt_debug_view) for the tests: a numpy restatement of RPT_Util::DebugColor
(ReSTIR_PT/Util.hlsli:69-139), the oracle frame loop with a view, and the reuse settings the view tests run."""
import ctypes as C
import os
import subprocess

import numpy as np

from tests import orc, rpt_util
from tests.orc import RptBuffers, ptr
from zetaray_b200 import _lib

VIEWS_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "rpt_views")

NONE, K, CASE, FOUND_CONNECTION, CONNECTION_LOBE_K_MIN_1, CONNECTION_LOBE_K = range(6)
VIEWS = (K, CASE, FOUND_CONNECTION, CONNECTION_LOBE_K_MIN_1, CONNECTION_LOBE_K)

# the reuse settings the views are written under: the path-trace write, the TtC write, the last StC write
REUSE = {"pathtrace": dict(temporal_resample=0, num_spatial_passes=0), "temporal": dict(num_spatial_passes=0),
         "spatial1": dict(num_spatial_passes=1), "spatial2": dict(num_spatial_passes=2)}

DIFFUSE_R, DIFFUSE_T, GLOSSY_R, GLOSSY_T = 0, 1, 2, 3
_f = lambda *c: np.array(c, dtype=np.float32)


def debug_color(view, meta, li):
    """DebugColor over the reconnections packed in meta (uint32 record words) and the colours li (n x 3 float32)."""
    meta = np.asarray(meta, dtype=np.uint32)
    c = np.array(li, dtype=np.float32, copy=True)
    if view == NONE:
        return c
    kk = meta & 0xf
    k = np.where(kk == 0xf, 0xf, kk + 2)            # Reservoir.hlsli:143-144: a stored 13 decodes to k == 15 == EMPTY
    empty = k == 0xf
    y, z = (meta >> 8) & 0xff, (meta >> 16) & 0xff
    lobe = lambda v: np.where(v <= 4, v, 5)       # BSDF::LobeFromValue; 4 = COAT, 5 = ALL
    l1, lk = lobe(y & 7), lobe((y >> 3) & 7)
    case3, case2 = ((y >> 6) & 3) != 0, (z & 3) != 0
    case1 = ~case2 & ~case3
    ne = ~empty
    if view == K:
        c[empty] = 0
        c[ne & (k == 2)] = _f(0.1, 0.25, 0.88)
        c[ne & (k == 3)] = _f(0.13, 0.55, 0.14)
        c[ne & (k == 4)] = _f(0.69, 0.45, 0.1)
        c[ne & (k >= 5)] = _f(0.88, 0.08, 0.1)
    elif view == CASE:
        c[empty] = 0
        c[ne & case1] = _f(0.85, 0.096, 0.1)
        c[ne & ~case1 & case2] = _f(0.13, 0.6, 0.14)
        c[ne & ~case1 & ~case2 & case3] = _f(0.1, 0.27, 0.888)
    elif view == FOUND_CONNECTION:
        c[:] = np.where(ne[:, None], _f(0.234, 0.12, 0.2134), 0)
    elif view == CONNECTION_LOBE_K_MIN_1:
        c[empty] = 0
        c[ne] = _f(0.55, 0.55, 0.0)
        for l, col in ((DIFFUSE_T, _f(0.25, 0.25, 0.25)), (GLOSSY_T, _f(0.1134, 0.12, 0.634)), (GLOSSY_R, _f(0.12, 0.4284, 0.2134)),
                       (DIFFUSE_R, _f(0.384, 0.12, 0.2134))):
            c[ne & (l1 == l)] = col
    elif view == CONNECTION_LOBE_K:
        black = empty | case3
        c[black] = 0
        c[~black] = _f(0.25, 0.25, 0.25)
        for l, col in ((DIFFUSE_T, _f(0.25, 0.25, 0.0)), (GLOSSY_T, _f(0.1134, 0.12, 0.634)), (GLOSSY_R, _f(0.12, 0.284, 0.2134)),
                       (DIFFUSE_R, _f(0.384, 0.12, 0.2134))):
            c[~black & (lk == l)] = col
    return c


def palette(view):
    """Every colour view can show besides black, as a set of RGB tuples."""
    metas = np.array([kk | (y << 8) | (z << 16) for kk in range(15) for y in range(256) for z in range(4)], dtype=np.uint32)
    cols = debug_color(view, metas, np.zeros((len(metas), 3), np.float32))
    return {tuple(c) for c in cols.tolist()} - {(0.0, 0.0, 0.0)}


_views = None


def load():
    """oracle/rpt_views/librpt_views.so (built by build(); compiled here when missing) with the types of rpt_views_api.h."""
    global _views
    if _views is None:
        so = os.path.join(VIEWS_DIR, "librpt_views.so")
        if not os.path.exists(so):
            subprocess.check_call(["bash", os.path.join(VIEWS_DIR, "build.sh")])
        _views = _lib.declare(C.CDLL(so), orc.prototypes(os.path.join(VIEWS_DIR, "rpt_views_api.h"), "RPTV_API", "rptv_"))
    return _views


PATHTRACE, TTC, STC = 0, 1, 2       # RPTV_* write points


class ViewOracle(rpt_util.OracleRenderer):
    """OracleRenderer whose ReSTIR PT frames show debug view `view`. The frame is the oracle's frame without a view (the view
    changes FINAL only); its write points are then redone with the view (rpt_views_api.h) from the planes each read. What the
    frame overwrites before the end -- the path tracer's reservoirs with temporal reuse off, the first spatial pass's planes of
    two -- comes from the same frame rendered on copies of the planes with the reset flag set or one spatial pass."""
    view = NONE

    def _render(self, params, state, planes):
        c = self.gb[self.cur]; p = self.gb[self.cur ^ 1]
        b = RptBuffers((planes["res"][0].ctypes.data, planes["res"][1].ctypes.data), planes["target"].ctypes.data,
                       planes["final"].ctypes.data, planes["neighbor"].ctypes.data, planes["tmCtN"].ctypes.data, planes["tmNtC"].ctypes.data)
        self.o.orc_rpt_render(self.osc.h, C.byref(self.fc), ptr(c[0]), ptr(c[2]), ptr(c[3]), ptr(p[0]), ptr(p[3]), C.byref(params),
                              C.byref(b), ptr(state), 0, self.nthreads)

    def _copy(self, **changes):
        """The frame rendered on copies of the planes with the parameter changes; returns the copies and their state."""
        planes = dict(res=[self.res[0].copy(), self.res[1].copy()], target=self.target.copy(), final=self.final.copy(),
                      neighbor=self.neighbor.copy(), tmCtN=self.tmCtN.copy(), tmNtC=self.tmNtC.copy())
        params = _lib.IndirectParams.from_buffer_copy(self.params)
        state = self.state.copy()
        for k, v in changes.items():
            if k == "reset":
                state[2] = 1
            else:
                setattr(params, k, v)
        self._render(params, state, planes)
        return planes, state

    def _write_point(self, stage, res_out, res_gate, neighbor, thread_map, before, final):
        c = self.gb[self.cur]; p = self.gb[self.cur ^ 1]
        sorted_ = self.params.sort_spatial if stage == STC else self.params.sort_temporal
        gate = res_gate if res_gate is not None else res_out
        load().rptv_write_point(self.osc.h, C.byref(self.fc), ptr(c[0]), ptr(c[2]), ptr(c[3]), ptr(p[0]), ptr(p[3]), stage, self.view,
                                int(sorted_), ptr(res_out), ptr(gate), ptr(neighbor), ptr(thread_map), ptr(before), ptr(final))

    def rpt(self, fc, last_stage=0):
        if self.view == NONE:
            return super().rpt(fc, last_stage)
        self.fc = fc
        p = self.params
        cur, reset = int(self.state[0]), bool(self.state[2])
        do_temporal = bool(p.temporal_resample and self.state[1])
        passes = p.num_spatial_passes if do_temporal else 0
        before = self.final.copy()
        # (write point, reservoirs it colours from, its gate reservoirs, neighbours, thread map) in the frame's order
        stages = []
        if not do_temporal and not reset:
            records = self._copy(reset=1)[0]["res"][cur]        # the path tracer keeps no reservoirs after the first frame
        for k in range(1, passes):
            planes, st = self._copy(num_spatial_passes=k)
            stages.append((STC, planes["res"][1 - int(st[0])], planes["res"][int(st[0])], planes["neighbor"], planes["tmNtC"]))
        prev = self.res[1 - cur].copy()
        super().rpt(fc)
        if not do_temporal:
            stages.append((PATHTRACE, self.res[cur] if reset else records, None, self.neighbor, self.tmNtC))
        elif passes == 0:
            stages.append((TTC, self.curr_reservoirs(), prev, self.neighbor, self.tmNtC))
        else:
            stages.append((STC, self.curr_reservoirs(), self.res[int(self.state[0])], self.neighbor, self.tmNtC))
        for stage in stages:
            after = self.final.copy()
            self._write_point(*stage, before, after)
            self.final[:] = before = after
