"""Compositing, the firefly filter and TAA kernels (zetaray_b200/csrc/post.cu) on the inputs of tests/test_post_oracle.py: bit for
bit against the CPU oracle, and within that file's tolerances of the independent float64 truth (oracle/indep_post.py). Also row
ranges (strip-sharded frames): inside the strip the output is the full-image result, outside it the output plane is left as it
was -- checked against a sentinel written into the plane before the render (TAA writes the plane it is not currently showing)."""
import ctypes as C

import numpy as np
import pytest

from tests import synth
from tests import test_post_oracle as po
from tests.orc import ptr

ip = po.ip


def _frame_inputs(fc, d_core, d_depth, d_me):
    from zetaray_b200 import _lib
    fi = _lib.FrameInputs()
    fi.frame = fc
    fi.curr.d_core = d_core.data_ptr()
    fi.curr.d_depth = d_depth.data_ptr()
    fi.curr.d_motion_emissive = d_me.data_ptr()
    return fi


def _d2h(d_ptr, shape, dtype):
    from zetaray_b200 import lib, check
    out = np.zeros(shape, dtype=dtype)
    check(lib.zr_memcpy_d2h(ptr(out), C.c_void_p(d_ptr), C.c_size_t(out.nbytes), None))
    check(lib.zr_stream_synchronize(None))
    return out


def _h2d(d_ptr, arr):
    from zetaray_b200 import lib, check
    a = np.ascontiguousarray(arr)
    check(lib.zr_memcpy_h2d(C.c_void_p(d_ptr), ptr(a), C.c_size_t(a.nbytes), None))
    check(lib.zr_stream_synchronize(None))


def _sentinel(n, words, seed):
    return np.random.default_rng(seed).integers(0, 1 << 32, size=(n, words), dtype=np.uint64).astype(np.uint32)


def device_taa(w, h, core, depth, me, sig, prev, bw=None, valid=1, rows=None):
    """One TAA render on the device with `prev` as its history. Returns (output uint2 plane, the sentinel the output plane held
    before the render). bw None leaves the pass's default blend weight."""
    import torch
    from zetaray_b200 import lib, check, _lib
    from tests.gpu_util import dev, dptr, stream
    fc = synth.look_at_frame_constants(w, h, frame=2)
    d_core, d_depth, d_me, d_sig = dev(core), dev(depth), dev(me), dev(sig)
    fi = _frame_inputs(fc, d_core, d_depth, d_me)
    p = C.c_void_p()
    check(lib.zr_taa_pass_create(w, h, C.byref(p)))
    img = _lib.Image2D()
    try:
        check(lib.zr_taa_pass_get_output(p, C.byref(img)))
        target = img.d_ptr                  # the plane the second render writes (the passes ping-pong)
        if valid:
            check(lib.zr_taa_pass_render(p, C.byref(fi), dptr(d_sig), stream()))
            torch.cuda.synchronize()
            check(lib.zr_taa_pass_get_output(p, C.byref(img)))
            assert img.d_ptr != target
            _h2d(img.d_ptr, prev)           # the history the next render reads
        else:
            target = None
        if bw is not None:
            check(lib.zr_taa_pass_set_blend_weight(p, C.c_float(bw)))
        if rows is not None:
            check(lib.zr_taa_pass_set_rows(p, rows[0], rows[1]))
        if target is not None:
            before = _sentinel(w * h, 2, w + h)
            _h2d(target, before)
        check(lib.zr_taa_pass_render(p, C.byref(fi), dptr(d_sig), stream()))
        torch.cuda.synchronize()
        check(lib.zr_taa_pass_get_output(p, C.byref(img)))
        if target is None:
            before = None
        else:
            assert img.d_ptr == target
        return _d2h(img.d_ptr, (w * h, 2), np.uint32), before
    finally:
        lib.zr_taa_pass_destroy(p)


def device_compositing(w, h, fc, core, depth, direct, indirect, params, rows=None):
    import torch
    from zetaray_b200 import lib, check, _lib
    from tests.gpu_util import dev, stream
    d_core, d_depth, d_me = dev(core), dev(depth), dev(np.zeros((w * h, 2), np.uint32))
    d_dir = dev(direct) if direct is not None else None
    d_ind = dev(indirect) if indirect is not None else None
    fi = _frame_inputs(fc, d_core, d_depth, d_me)
    p = C.c_void_p()
    check(lib.zr_compositing_pass_create(w, h, C.byref(p)))
    try:
        check(lib.zr_compositing_pass_set_params(p, C.byref(_lib.CompositingParams(*params))))
        if rows is not None:
            check(lib.zr_compositing_pass_set_rows(p, rows[0], rows[1]))
        img = _lib.Image2D()
        check(lib.zr_compositing_pass_get_output(p, C.byref(img)))
        before = _sentinel(w * h, 4, w * h).view(np.float32)
        _h2d(img.d_ptr, before)
        check(lib.zr_compositing_pass_render(p, C.byref(fi), C.c_void_p(d_dir.data_ptr() if d_dir is not None else 0),
                                             C.c_void_p(d_ind.data_ptr() if d_ind is not None else 0), stream()))
        torch.cuda.synchronize()
        return _d2h(img.d_ptr, (w * h, 4), np.float32), before
    finally:
        lib.zr_compositing_pass_destroy(p)


# ----------------------------------------------------------------------------------------------------------------- cases
def taa_cases():
    """(name, w, h, depth, motion, signal rgb or rgba, history, blend weight) -- the CPU tier's edges, generated the same way."""
    out = []
    for w, h in po.SIZES:
        depth, motion, sig = po.random_frame(w, h, 40, motion_px=2.0)
        out.append(("random %dx%d" % (w, h), w, h, depth, motion, sig, po.random_history(w, h, 1), 0.1))
    for w, h in ((7, 3), (33, 17), (257, 131)):
        depth, motion, sig = po.random_frame(w, h, 60, motion_px=max(w, h) / 3.0)
        out.append(("footprint %dx%d" % (w, h), w, h, depth, motion, sig, po.random_history(w, h, 2), 0.1))
        rng = np.random.default_rng(w)
        out.append(("dilation %dx%d" % (w, h), w, h, rng.choice(np.float32([1.0, 2.0, 3.0]), size=w * h),
                    po.distinct_motion(w, h, 3), synth.synth_hdr(w, h, 4),
                    po.half_plane(np.where(rng.random((w * h, 1)) < 0.5, 0.05, 8.0) * rng.random((w * h, 3))), 0.1))
    w, h = 9, 7
    zero = (np.zeros(w * h), np.zeros(w * h))
    flat = np.tile(np.float32([0.75, 1.5, 0.375]), (w * h, 1))
    out.append(("flat outside", w, h, np.full(w * h, 4.0), zero, flat, po.half_plane(flat * 2), 0.1))
    rng = np.random.default_rng(5)
    neg = (rng.random((w * h, 3)) * 4 - 2).astype(np.float32)
    out.append(("negative", w, h, np.full(w * h, 4.0), po.distinct_motion(w, h, 6, px=1.0), neg, po.random_history(w, h, 7), 0.1))
    frac = (np.full(w * h, round(0.3 * 32767 / w)), np.full(w * h, round(0.4 * 32767 / h)))
    bad = (rng.random((w * h, 3)) * 2).astype(np.float32)
    bad[31, 1], bad[40, 0], bad[12, 2] = np.nan, np.inf, -np.inf
    hist = rng.random((w * h, 3)) * 2
    hist[22, 0], hist[50, 1] = np.nan, np.inf
    out.append(("nan inf", w, h, np.full(w * h, 4.0), frac, bad, po.half_plane(hist), 0.1))
    big = np.full((w * h, 3), 1e6, dtype=np.float32)
    big[:, 1] = 65519.0
    out.append(("overflow", w, h, np.full(w * h, 4.0), zero, big, po.half_plane(np.full((w * h, 3), 65504.0)), 0.1))
    for bw in (0.0, 0.5, 1.0, 1.5):
        depth, motion, sig = po.random_frame(33, 17, 100, motion_px=2.0)
        out.append(("bw %g" % bw, 33, 17, depth, motion, sig, po.random_history(33, 17, 8), bw))
    for target in (0.0, 1.0):
        size, col, k = po.uv_landing(target)
        m = np.zeros((3, size), dtype=np.int64)
        m[:, col] = k
        _, _, sig = po.random_frame(size, 3, 90)
        out.append(("land %g" % target, size, 3, np.full(3 * size, 4.0), (m, np.zeros_like(m)), sig, po.random_history(size, 3, 9), 0.1))
    return out


def same_taa_bits(got, ref):
    """RGBA16F planes equal bit for bit, except that a NaN matches any NaN: the sign and payload of a NaN made by arithmetic
    (Inf * 0, Inf - Inf) are the platform's -- x86 makes the negative default NaN, the GPU 0x7fffffff."""
    a, b = got.view(np.uint16), ref.view(np.uint16)
    nan_a = ((a & 0x7c00) == 0x7c00) & ((a & 0x3ff) != 0)
    nan_b = ((b & 0x7c00) == 0x7c00) & ((b & 0x3ff) != 0)
    return bool(((a == b) | (nan_a & nan_b)).all())


def _oracle_and_truth(oracle, w, h, core, d, me, sig, prev, bw, valid):
    ref = po.oracle_taa(oracle, w, h, core, me, sig, prev, bw, valid)
    truth = ip.taa(w, h, d, me[:, 0], sig, prev, bw, valid)
    return ref, truth


@pytest.mark.gpu
def test_taa_edges_device(oracle):
    st = po.TaaStats()
    for name, w, h, depth, motion, sig, prev, bw in taa_cases():
        core, d, me = po.planes(w, h, depth, motion=motion)
        sig = po.rgba(sig) if np.asarray(sig).shape[-1] == 3 else sig
        got, _ = device_taa(w, h, core, d, me, sig, prev, bw=bw)
        ref, truth = _oracle_and_truth(oracle, w, h, core, d, me, sig, prev, bw, 1)
        assert same_taa_bits(got, ref), name
        st.check(got, truth, w, h, name)
    st.finish()


@pytest.mark.gpu
def test_taa_blend_weight_setter(oracle):
    """The pass's blend weight reaches the kernel: the default is 0.1, and a set weight replaces it."""
    w, h = 33, 17
    depth, motion, sig = po.random_frame(w, h, 110, motion_px=2.0)
    core, d, me = po.planes(w, h, depth, motion=motion)
    prev = po.random_history(w, h, 11)
    default, _ = device_taa(w, h, core, d, me, sig, prev, bw=None)
    half, _ = device_taa(w, h, core, d, me, sig, prev, bw=0.5)
    assert default.tobytes() == po.oracle_taa(oracle, w, h, core, me, sig, prev, 0.1, 1).tobytes()
    assert half.tobytes() == po.oracle_taa(oracle, w, h, core, me, sig, prev, 0.5, 1).tobytes()
    assert default.tobytes() != half.tobytes()


STRIPS = [(13, 59), (37, 38), (0, 1), (100, 131), (130, 131), (5, 131)]


@pytest.mark.gpu
@pytest.mark.parametrize("y0,y1", STRIPS)
def test_taa_rows(oracle, y0, y1):
    """A row range whose ends are not multiples of the 8-row TAA tile: inside, the full-image result; outside, the plane as it
    was."""
    w, h = 257, 131
    depth, motion, sig = po.random_frame(w, h, 120, motion_px=3.0)
    core, d, me = po.planes(w, h, depth, motion=motion)
    prev = po.random_history(w, h, 12)
    got, before = device_taa(w, h, core, d, me, sig, prev, rows=(y0, y1))
    ref, truth = _oracle_and_truth(oracle, w, h, core, d, me, sig, prev, 0.1, 1)
    r = slice(y0 * w, y1 * w)
    assert got[r].tobytes() == ref[r].tobytes()
    assert got[:y0 * w].tobytes() == before[:y0 * w].tobytes()
    assert got[y1 * w:].tobytes() == before[y1 * w:].tobytes()
    st = po.TaaStats()
    sub = {k: v[r] for k, v in truth.items()}
    st.check(got[r], sub, w, y1 - y0, "rows %d-%d" % (y0, y1))


def comp_inputs(w, h, seed):
    rng = np.random.default_rng(seed)
    n = w * h
    flags = rng.choice(np.array([0, 0, 0, po.F_EMISSIVE, po.F_INVALID], dtype=np.uint32), size=n)
    depth = np.where(flags & po.F_INVALID, po.FLT_MAX, 1.0 + 9.0 * rng.random(n)).astype(np.float32)
    core, d, _ = po.planes(w, h, depth, flags)
    return core, d, synth.synth_hdr(w, h, seed + 1), synth.synth_hdr(w, h, seed + 2)


def _comp_reference(oracle, w, h, fc, core, d, direct, indirect, params):
    dr = direct if params[0] else None
    ir = indirect if params[1] else None
    comp = po.oracle_compositing(oracle, fc, core, dr, ir)
    truth = ip.compositing(w, h, core[:, 3], dr, ir, fc.Accumulate, fc.CameraStatic, fc.NumFramesCameraStatic)
    if not params[2]:
        return comp, truth
    fire = po.oracle_firefly(oracle, fc, core, comp)
    ftruth, margin = ip.firefly(w, h, d, comp)
    low = margin < 4 * po.EPS32
    assert low.sum() <= max(1, 0.001 * w * h)
    ok = (fire[:, :3].astype(np.float64) == ftruth).all(axis=1)
    assert ok[~low].all()
    return fire, None


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", po.SIZES)
def test_compositing_edges_device(oracle, w, h):
    core, d, direct, indirect = comp_inputs(w, h, w * 7 + h)
    for params in ((1, 1, 1), (1, 1, 0), (1, 0, 1), (0, 1, 0), (0, 0, 1)):
        for acc, nf in ((0, 1), (1, 3), (1, 7)):
            fc = po.frame_constants(w, h, acc, acc, nf)
            got, _ = device_compositing(w, h, fc, core, d, direct, indirect, params)
            ref, truth = _comp_reference(oracle, w, h, fc, core, d, direct, indirect, params)
            assert got.tobytes() == ref.tobytes(), (params, acc, nf)
            if truth is not None:
                ulp32 = np.spacing(np.abs(truth).astype(np.float32)).astype(np.float64)
                assert (np.abs(got[:, :3] - truth) <= 2 * ulp32).all()


@pytest.mark.gpu
@pytest.mark.parametrize("y0,y1", STRIPS + [(15, 33)])
@pytest.mark.parametrize("firefly", [0, 1])
def test_compositing_rows(oracle, y0, y1, firefly):
    """Row ranges against the 16-row firefly tile and the 8-row compositing tile."""
    w, h = 257, 131
    core, d, direct, indirect = comp_inputs(w, h, 130)
    fc = po.frame_constants(w, h)
    params = (1, 1, firefly)
    got, before = device_compositing(w, h, fc, core, d, direct, indirect, params, rows=(y0, y1))
    ref, _ = _comp_reference(oracle, w, h, fc, core, d, direct, indirect, params)
    r = slice(y0 * w, y1 * w)
    assert got[r].tobytes() == ref[r].tobytes()
    assert got[:y0 * w].tobytes() == before[:y0 * w].tobytes()
    assert got[y1 * w:].tobytes() == before[y1 * w:].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(1920, 1080), (2560, 1440)])
def test_full_size(oracle, w, h):
    """Both benchmark sizes once: compositing with the firefly filter and TAA over a history, device = oracle, both within the
    truth's tolerance."""
    core, d, direct, indirect = comp_inputs(w, h, 140)
    fc = po.frame_constants(w, h)
    got, _ = device_compositing(w, h, fc, core, d, direct, indirect, (1, 1, 1))
    ref, _ = _comp_reference(oracle, w, h, fc, core, d, direct, indirect, (1, 1, 1))
    assert got.tobytes() == ref.tobytes()
    depth, motion, _ = po.random_frame(w, h, 141, motion_px=4.0)
    core, d, me = po.planes(w, h, depth, motion=motion)
    prev = po.random_history(w, h, 14)
    sig = got
    out, _ = device_taa(w, h, core, d, me, sig, prev)
    ref, truth = _oracle_and_truth(oracle, w, h, core, d, me, sig, prev, 0.1, 1)
    assert out.tobytes() == ref.tobytes()
    st = po.TaaStats()
    st.check(out, truth, w, h, "%dx%d" % (w, h))
    st.finish()
    print("%dx%d TAA: worst %.1f fp16 ulps, worst k %.2f, exact %.5f of %d gated channels"
          % (w, h, st.worst_ulps, st.worst_k, st.n_gated_exact / max(1, st.n_gated), st.n_gated))
