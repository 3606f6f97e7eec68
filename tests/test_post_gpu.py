"""Compositing / firefly / TAA kernels vs the CPU oracle on seeded synthetic frames (bit-exact)."""
import ctypes as C
import numpy as np
import pytest

from tests.orc import ptr


def _frame_inputs(fc, d_core, d_depth, d_me):
    from zetaray_b200 import _lib
    fi = _lib.FrameInputs()
    fi.frame = fc
    fi.curr.d_core = d_core.data_ptr()
    fi.curr.d_depth = d_depth.data_ptr()
    fi.curr.d_motion_emissive = d_me.data_ptr()
    return fi


@pytest.mark.gpu
# images smaller than one 32 x 16 tile of the firefly kernel (every tap near an edge), partial tiles, and both full sizes the
# benchmarks render, with and without accumulation
@pytest.mark.parametrize("w,h,accum", [(64, 40, 0), (257, 131, 0), (257, 131, 1), (1920, 1080, 0),
                                       (7, 3, 0), (31, 17, 1), (1920, 1080, 1), (2560, 1440, 0)])
def test_compositing_firefly(oracle, w, h, accum):
    import torch
    from zetaray_b200 import lib, check, _lib
    from tests import synth
    from tests.gpu_util import dev, dptr, host, stream
    fc = synth.look_at_frame_constants(w, h, frame=3)
    if accum:
        fc.Accumulate, fc.CameraStatic, fc.NumFramesCameraStatic = 1, 1, 5
    core, depth, me = synth.synth_gbuffer(w, h, 11)
    direct = synth.synth_hdr(w, h, 12)
    indirect = synth.synth_hdr(w, h, 13)
    comp = np.zeros((w * h, 4), dtype=np.float32)
    fire = np.zeros((w * h, 4), dtype=np.float32)
    oracle.orc_compositing(C.byref(fc), ptr(core), ptr(direct), ptr(indirect), ptr(comp))
    oracle.orc_firefly(C.byref(fc), ptr(core), ptr(comp), ptr(fire))

    d_core, d_depth, d_me = dev(core), dev(depth), dev(me)
    d_dir, d_ind = dev(direct), dev(indirect)
    fi = _frame_inputs(fc, d_core, d_depth, d_me)
    p = C.c_void_p()
    check(lib.zr_compositing_pass_create(w, h, C.byref(p)))
    img = _lib.Image2D()
    # fused (default)
    check(lib.zr_compositing_pass_render(p, C.byref(fi), dptr(d_dir), dptr(d_ind), stream()))
    torch.cuda.synchronize()
    check(lib.zr_compositing_pass_get_output(p, C.byref(img)))
    out = np.zeros((w * h, 4), dtype=np.float32)
    check(lib.zr_memcpy_d2h(ptr(out), C.c_void_p(img.d_ptr), C.c_size_t(out.nbytes), None))
    check(lib.zr_stream_synchronize(None))
    assert out.tobytes() == fire.tobytes()
    # filter off -> plain compositing
    prm = _lib.CompositingParams(1, 1, 0)
    check(lib.zr_compositing_pass_set_params(p, C.byref(prm)))
    check(lib.zr_compositing_pass_render(p, C.byref(fi), dptr(d_dir), dptr(d_ind), stream()))
    torch.cuda.synchronize()
    check(lib.zr_memcpy_d2h(ptr(out), C.c_void_p(img.d_ptr), C.c_size_t(out.nbytes), None))
    check(lib.zr_stream_synchronize(None))
    assert out.tobytes() == comp.tobytes()
    lib.zr_compositing_pass_destroy(p)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(64, 40), (257, 131), (1920, 1080)])
def test_taa_three_frames(oracle, w, h):
    import torch
    from zetaray_b200 import lib, check, _lib
    from tests import synth
    from tests.gpu_util import dev, dptr, stream
    p = C.c_void_p()
    check(lib.zr_taa_pass_create(w, h, C.byref(p)))
    prev = np.zeros((w * h, 2), dtype=np.uint32)
    valid = 0
    for frame in range(1, 4):
        fc = synth.look_at_frame_constants(w, h, frame=frame)
        core, depth, me = synth.synth_gbuffer(w, h, 100 + frame)
        if frame == 3:
            me[:, 0] = 0      # static frame: motion vectors zero
        signal = synth.synth_hdr(w, h, 200 + frame)
        ref = np.zeros((w * h, 2), dtype=np.uint32)
        oracle.orc_taa(C.byref(fc), ptr(core), ptr(me), ptr(signal), ptr(prev), ptr(ref), 0.1, valid)
        d_core, d_depth, d_me, d_sig = dev(core), dev(depth), dev(me), dev(signal)
        fi = _frame_inputs(fc, d_core, d_depth, d_me)
        check(lib.zr_taa_pass_render(p, C.byref(fi), dptr(d_sig), stream()))
        torch.cuda.synchronize()
        img = _lib.Image2D()
        check(lib.zr_taa_pass_get_output(p, C.byref(img)))
        assert img.texel_bytes == 8
        out = np.zeros((w * h, 2), dtype=np.uint32)
        check(lib.zr_memcpy_d2h(ptr(out), C.c_void_p(img.d_ptr), C.c_size_t(out.nbytes), None))
        check(lib.zr_stream_synchronize(None))
        assert out.tobytes() == ref.tobytes(), "frame %d" % frame
        prev = ref
        valid = 1
    lib.zr_taa_pass_destroy(p)
