"""ReSTIR PT debug views on the CPU oracle (no GPU): the colour function against a numpy restatement of Util.hlsli:69-139, and
oracle frames under every reuse setting -- palette colours or black, black where the reference's write points put it, and the
reservoirs, target, neighbour and thread-map planes the same bytes as without a view."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import scene_util
from tests.orc import ptr
from tests.rpt_debug_view_util import (NONE, K, CASE, FOUND_CONNECTION, CONNECTION_LOBE_K_MIN_1, CONNECTION_LOBE_K, VIEWS, REUSE,
                                       ViewOracle, debug_color, load, palette)
from zetaray_b200 import _lib
from zetaray_b200.camera import FrameSequence

W, H, FRAMES = 128, 72, 3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_colour_function_matches_util_hlsli():
    """Every stored k (0..15, 15 = empty), lobe pair, case (lt_k, lt_{k+1}) and motion bit, over a radiance the view replaces."""
    o = load()
    metas = np.array([kk | ((l1 | (lk << 3) | (ltk << 6)) << 8) | ((ltk1 | (mot << 2)) << 16) | (m << 4)
                      for kk in range(16) for l1 in range(8) for lk in range(8) for ltk in range(4) for ltk1 in range(4)
                      for mot in (0, 1) for m in (0, 9)], dtype=np.uint32)
    n = len(metas)
    li = np.random.default_rng(3).random((n, 3), dtype=np.float32) * 4
    for view in (NONE,) + VIEWS:
        out = np.zeros((n, 3), np.float32)
        o.rptv_debug_color(view, ptr(metas), ptr(li), n, ptr(out))
        want = debug_color(view, metas, li)
        assert out.tobytes() == want.tobytes(), "view %d: %d colours differ" % (view, int((out != want).any(axis=1).sum()))
    # the constants as the reference has them, GLOSSY_R's two values included
    lobe = lambda v, l1, lk, case3=False: debug_color(v, np.array([(l1 | (lk << 3) | ((3 if case3 else 0) << 6)) << 8], np.uint32),
                                                      np.zeros((1, 3), np.float32))[0].tolist()
    assert lobe(CONNECTION_LOBE_K_MIN_1, 2, 0) == np.float32([0.12, 0.4284, 0.2134]).tolist()
    assert lobe(CONNECTION_LOBE_K, 0, 2) == np.float32([0.12, 0.284, 0.2134]).tolist()
    assert lobe(CONNECTION_LOBE_K, 0, 2, case3=True) == [0.0, 0.0, 0.0]


def _run(scene, reuse, view):
    """FRAMES oracle frames of `scene` with the reuse setting and the view; per frame: FINAL's colours, the planes the view must not
    change, the valid-pixel mask, the output reservoirs and, for the spatial settings, the last spatial pass's input reservoirs."""
    R = ViewOracle(scene_util.SCENES[scene](), W, H)
    R.view = view
    for k, v in REUSE[reuse].items():
        setattr(R.params, k, v)
    seq = FrameSequence(W, H)
    out = []
    for _ in range(FRAMES):
        fc = seq.next()
        gb = R.gbuffer(fc)
        R.rpt(fc)
        flags = gb[0][:, 3] & 0xff
        planes = {"res0": R.res[0].copy(), "res1": R.res[1].copy(), "target": R.target.copy(), "neighbor": R.neighbor.copy(),
                  "tmCtN": R.tmCtN.copy(), "tmNtC": R.tmNtC.copy()}
        out.append(dict(rgb=R.final[:, :3].copy(), planes=planes, valid=(flags & 0x6) == 0, res_out=R.curr_reservoirs()["meta"].copy(),
                        res_in=R.res[int(R.state[0])]["meta"].copy(), neighbor=R.neighbor.copy()))
    return out


_cache = {}


def _frames(scene, reuse, view):
    key = (scene, reuse, view)
    if key not in _cache:
        _cache[key] = _run(scene, reuse, view)
    return _cache[key]


def _black(rgb):
    return (rgb == 0).all(axis=1)


@pytest.mark.parametrize("reuse", list(REUSE))
@pytest.mark.parametrize("scene", ["glossy", "cornell"])
def test_oracle_frames_show_palette_colours_and_black_where_the_write_points_put_it(scene, reuse):
    base = _frames(scene, reuse, NONE)
    views = {v: _frames(scene, reuse, v) for v in VIEWS}
    empty = lambda meta: (np.where((meta & 0xf) == 0xf, 0xf, (meta & 0xf) + 2)) == 0xf
    for fr in range(FRAMES):
        b = base[fr]
        for v, frames in views.items():
            f = frames[fr]
            # the view changes FINAL only
            for name, plane in b["planes"].items():
                assert plane.tobytes() == f["planes"][name].tobytes(), "frame %d view %d: %s differs" % (fr, v, name)
            # every valid pixel shows one of the view's colours or black; the others are as without the view
            pal = palette(v)
            cols = set(map(tuple, f["rgb"][f["valid"]].tolist())) - {(0.0, 0.0, 0.0)}
            assert cols <= pal, "frame %d view %d: colours outside the palette %s" % (fr, v, sorted(cols - pal)[:4])
            assert f["rgb"][~f["valid"]].tobytes() == b["rgb"][~b["valid"]].tobytes()
            assert cols, "frame %d view %d: all black" % (fr, v)
        # where a view writes its colour is the same for all views: black in FOUND_CONNECTION <=> black in K, CASE and
        # CONNECTION_LOBE_K_MIN_1; CONNECTION_LOBE_K is also black for case 3
        found = _black(views[FOUND_CONNECTION][fr]["rgb"])
        for v in (K, CASE, CONNECTION_LOBE_K_MIN_1):
            assert (_black(views[v][fr]["rgb"]) == found).all(), "frame %d view %d" % (fr, v)
        case3 = (views[CASE][fr]["rgb"] == np.float32([0.1, 0.27, 0.888])).all(axis=1)
        assert (_black(views[CONNECTION_LOBE_K][fr]["rgb"]) == (found | case3)).all(), "frame %d" % fr
        written = ~found & b["valid"]
        # where it is coloured, the colour is the one of the reservoir the frame produced (the path-trace write keeps no
        # reservoir after the first frame)
        if reuse != "pathtrace" or fr == 0:
            for v, frames in views.items():
                want = debug_color(v, b["res_out"], np.zeros((W * H, 3), np.float32))
                assert frames[fr]["rgb"][written].tobytes() == want[written].tobytes(), "frame %d view %d" % (fr, v)
            assert not (written & empty(b["res_out"])).any()
        if reuse.startswith("spatial") and fr > 0:
            # Reconnect_StC: black exactly where there is no neighbour, the neighbour's input reservoir has no reconnection or the
            # output reservoir has none
            x, y = np.arange(W * H) % W, np.arange(W * H) // W
            nb = b["neighbor"]
            has_n = (nb & 0xff) != 0xff
            nx = np.clip(x + (nb & 0xff).astype(np.int64) - 32, 0, W - 1)
            ny = np.clip(y + (nb >> 8).astype(np.int64) - 32, 0, H - 1)
            n_empty = empty(b["res_in"][ny * W + nx])
            want_black = ~has_n | n_empty | empty(b["res_out"])
            assert (found[b["valid"]] == want_black[b["valid"]]).all(), "frame %d: %d pixels" % (
                fr, int((found[b["valid"]] != want_black[b["valid"]]).sum()))
            assert (~has_n & b["valid"]).any() and (has_n & n_empty & b["valid"]).any()
        if reuse == "pathtrace" and fr == 0:
            assert (found[b["valid"]] == empty(b["res_out"])[b["valid"]]).all()


def test_view_library_exports_what_its_header_declares():
    import subprocess
    from tests import orc
    protos = orc.prototypes(os.path.join(ROOT, "oracle", "rpt_views", "rpt_views_api.h"), "RPTV_API", "rptv_")
    load()
    so = os.path.join(ROOT, "oracle", "rpt_views", "librpt_views.so")
    out = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True, check=True).stdout
    assert set(protos) == {l.split()[-1] for l in out.splitlines() if l.split() and l.split()[-1].startswith("rptv_")}


def test_entry_point_is_declared_and_bound():
    protos = _lib.prototypes()
    assert protos["zr_indirect_pass_set_debug_view"] == (C.c_int32, [C.c_void_p, C.c_uint32])
    f = _lib.lib.zr_indirect_pass_set_debug_view
    assert f.restype is C.c_int32 and list(f.argtypes) == [C.c_void_p, C.c_uint32]
    with open(os.path.join(ROOT, "include", "zr_abi.h")) as h:
        hdr = h.read()
    body = hdr[hdr.index("typedef enum zr_rpt_debug_view"):hdr.index("} zr_rpt_debug_view;")]
    names = [n.strip() for n in body[body.index("{") + 1:].split(",")]
    assert names == ["ZR_RPT_DEBUG_VIEW_" + n for n in ("NONE = 0", "K", "CASE", "FOUND_CONNECTION", "CONNECTION_LOBE_K_MIN_1",
                                                        "CONNECTION_LOBE_K")]
    assert _lib.lib.zr_abi_version() == (1 << 16) | 11
    from zetaray_b200.passes import IndirectLighting
    assert IndirectLighting.DEBUG_VIEW_CONNECTION_LOBE_K == CONNECTION_LOBE_K

