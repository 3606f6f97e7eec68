"""Compositing, the firefly filter and TAA of the CPU oracle (oracle/orc_post.cpp) against the independent float64 truth
(oracle/indep_post.py), on inputs built to reach the edges where stencils go wrong: images narrower than the 3 x 3 stencil, flat
neighbourhoods, negatives, NaN / Inf, fp16 overflow, exact luminance and depth ties, motions that put the history footprint over
every edge or land prevUV exactly on 0 and 1. No GPU; tests/test_post_independent_gpu.py runs the same inputs through the kernels.

Tolerances:
  * Compositing: 2 float32 ulps of the truth (one rounding of the sum, one of the division), and exact bits with one source and
    N = 1.
  * Firefly: exact bits. It only selects colours, so the one float32 effect is a near-tie of luminances; a pixel whose decision
    margin (indep_post.firefly) is below 4 eps32 may only have picked one of the candidates, and such pixels must be under 0.1 %.
  * TAA, per channel: |oracle - truth| <= 1 fp16 ulp of the truth + K eps32 S, where S is the truth's `scale`: the largest |rgb|
    over the centre, the clamped neighbours and the 4 x 4 history texels under the Catmull-Rom footprint. K is derived, not
    fitted (see taa_k). On top, among channels whose truth lies further than K eps32 S from an fp16 rounding midpoint (so that
    float32 error within the bound cannot change the rounding), at least 99.9 % are exact at fp16 -- a systematic 1-ulp bias
    would break that. The channels left out are mostly exact midpoints: float32 signals are often exactly halfway between two
    fp16 values, and the reconstruction's ~1e-6 departure from the centre (the Mitchell quirk) then decides the rounding."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from tests import synth
from tests.orc import ptr

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import indep_post as ip  # noqa: E402

EPS32 = float(np.finfo(np.float32).eps)
FLT_MAX = np.float32(3.402823466e+38)
SIZES = [(1, 1), (1, 9), (9, 1), (2, 2), (7, 3), (33, 17), (257, 131)]
F_EMISSIVE, F_INVALID = 0x02, 0x04


def taa_k():
    """K of the TAA bound, in units of eps32 * S.

    The reference calls Mitchell1D with the integer tap offset, so the neighbour weights are exactly 0 in float64 and
    q = Mitchell1D_f32(1) / Mitchell1D_f32(0) ~ 10.5 eps32 in float32 (evaluated here the reference's way). The reconstruction
    then moves from the centre by sum_k w_k (n_k - c) / sum w over the four edge neighbours (the corner ones carry q^2), and
    |n_k - c| <= 2 S with 1 / (1 + L) <= 1 for the clamped neighbours: at most 8 q S. What remains is ordinary float32 rounding,
    each step of it bounded by a few eps32 S: the nine-term moments, the variance, ClipAABB's centre and ray, the Catmull-Rom sum
    of nine taps with weights summing to 1, and the blend (weights in [0, 1], normalised). 12 eps32 S covers those together, since
    the clip and the blend are convex combinations that do not amplify their inputs' error."""
    f = np.float32
    b = f(0.33)

    def m(x):
        x = f(abs(f(2) * f(x)))
        if x > 1:
            return ((-b - f(6) * b) * x * x * x + (f(6) * b + f(30) * b) * x * x + (f(-12) * b - f(48) * b) * x
                    + (f(8) * b + f(24) * b)) * (f(1) / f(6))
        return ((f(12) - f(9) * b - f(6) * b) * x * x * x + (f(-18) + f(12) * b + f(6) * b) * x * x + (f(6) - f(2) * b)) * (f(1) / f(6))
    q = float(m(1)) / float(m(0)) / EPS32
    return 8.0 * q + 12.0


K = taa_k()


# ------------------------------------------------------------------------------------------------------------------- planes
def planes(w, h, depth, flags=None, motion=None):
    """core uint4 / depth f32 / motion_emissive uint2 from a depth plane, flag bytes and (mx, my) snorm16 integers."""
    n = w * h
    depth = np.asarray(depth, dtype=np.float32).reshape(n)
    core = np.zeros((n, 4), dtype=np.uint32)
    core[:, 0] = depth.view(np.uint32)
    fl = np.zeros(n, dtype=np.uint32) if flags is None else np.asarray(flags, dtype=np.uint32).reshape(n)
    core[:, 3] = fl | (77 << 8)
    me = np.zeros((n, 2), dtype=np.uint32)
    if motion is not None:
        mx, my = (np.asarray(a).reshape(n).astype(np.int16).view(np.uint16).astype(np.uint32) for a in motion)
        me[:, 0] = mx | (my << 16)
    return core, depth.copy(), me


def frame_constants(w, h, accumulate=0, camera_static=0, n_frames=1):
    fc = synth.look_at_frame_constants(w, h, frame=3)
    fc.Accumulate, fc.CameraStatic, fc.NumFramesCameraStatic = accumulate, camera_static, n_frames
    return fc


def rgba(rgb):
    rgb = np.asarray(rgb, dtype=np.float32).reshape(-1, 3)
    out = np.zeros((rgb.shape[0], 4), dtype=np.float32)
    out[:, :3] = rgb
    return out


def half_plane(rgb):
    """(n, 3) values -> RGBA16F uint2 plane (fp16 RNE)."""
    hb = ip.to_half(np.asarray(rgb, dtype=np.float64).reshape(-1, 3)).view(np.uint16).astype(np.uint32)
    out = np.zeros((hb.shape[0], 2), dtype=np.uint32)
    out[:, 0] = hb[:, 0] | (hb[:, 1] << 16)
    out[:, 1] = hb[:, 2]
    return out


def decode(u2, w, h):
    return ip.decode_half4(u2, w, h).reshape(-1, 3)


# ------------------------------------------------------------------------------------------------------------------- runners
def oracle_compositing(oracle, fc, core, direct, indirect):
    out = np.zeros((fc.RenderWidth * fc.RenderHeight, 4), dtype=np.float32)
    oracle.orc_compositing(C.byref(fc), ptr(core), None if direct is None else ptr(direct),
                           None if indirect is None else ptr(indirect), ptr(out))
    return out


def oracle_firefly(oracle, fc, core, comp):
    out = np.zeros_like(comp)
    oracle.orc_firefly(C.byref(fc), ptr(core), ptr(comp), ptr(out))
    return out


def oracle_taa(oracle, w, h, core, me, sig, prev, bw=0.1, valid=1):
    fc = synth.look_at_frame_constants(w, h, frame=2)
    out = np.zeros((w * h, 2), dtype=np.uint32)
    oracle.orc_taa(C.byref(fc), ptr(core), ptr(me), ptr(sig), ptr(prev), ptr(out), bw, int(valid))
    return out


class TaaStats:
    """Deviation of fp16 TAA outputs from the truth, accumulated over a test."""

    def __init__(self):
        self.worst_ulps = self.worst_k = 0.0
        self.n_gated = self.n_gated_exact = 0

    def check(self, got_u2, truth, w, h, what=""):
        got = decode(got_u2, w, h)
        t = truth["out"]
        t16 = ip.to_half(t).astype(np.float64)
        fin = np.isfinite(t16)
        # non-finite truths (Inf from fp16 overflow, a NaN centre passed through) must be reproduced exactly
        same_special = (got == t16) | (np.isnan(got) & np.isnan(t16))
        bad = ~fin & ~same_special
        assert not bad.any(), "%s: non-finite channels differ at %s" % (what, np.argwhere(bad)[:5].tolist())
        s = np.broadcast_to(truth["scale"][:, None], t.shape)
        with np.errstate(invalid="ignore", over="ignore"):
            ulp = np.spacing(np.abs(t16.astype(np.float16))).astype(np.float64)
            d = np.abs(got - t16)
            bound = ulp + K * EPS32 * s
            over = fin & ~(d <= bound)
        if over.any():
            i = np.argwhere(over)[0]
            p = i[0]
            raise AssertionError("%s: %d channels beyond 1 ulp + K eps32 S; first px (%d, %d) ch %d oracle %r truth %r S %r path %d"
                                 % (what, over.sum(), p % w, p // w, i[1], got[p], t[p], truth["scale"][p], truth["path"][p]))
        fs = fin & np.isfinite(s) & (s > 0)
        if fs.any():
            self.worst_ulps = max(self.worst_ulps, float((d[fs] / ulp[fs]).max()))
            self.worst_k = max(self.worst_k, float((np.maximum(d[fs] - ulp[fs], 0.0) / (EPS32 * s[fs])).max()))
        h16 = t16.astype(np.float16)
        with np.errstate(invalid="ignore", over="ignore"):
            lo = np.nextafter(h16, np.float16(-np.inf)).astype(np.float64)
            hi = np.nextafter(h16, np.float16(np.inf)).astype(np.float64)
            to_mid = np.minimum(np.abs(t - 0.5 * (t16 + lo)), np.abs(t - 0.5 * (t16 + hi)))
        gated = fin & np.isfinite(to_mid) & (to_mid > K * EPS32 * s)
        self.n_gated += int(gated.sum())
        self.n_gated_exact += int((gated & (d == 0)).sum())

    def finish(self, min_exact=0.999):
        if self.n_gated:
            frac = self.n_gated_exact / self.n_gated
            assert frac >= min_exact or self.n_gated - self.n_gated_exact <= 1, \
                "only %.4f%% of %d channels exact at fp16" % (100 * frac, self.n_gated)
        return self


def run_taa_case(oracle, stats, w, h, depth, motion, sig, prev, bw=0.1, valid=1, what=""):
    core, d, me = planes(w, h, depth, motion=motion)
    sig = rgba(sig) if np.asarray(sig).shape[-1] == 3 else sig
    got = oracle_taa(oracle, w, h, core, me, sig, prev, bw, valid)
    truth = ip.taa(w, h, d, me[:, 0], sig, prev, bw, valid)
    stats.check(got, truth, w, h, what)
    return got, truth


def random_frame(w, h, seed, motion_px=0.5, miss_frac=0.05):
    rng = np.random.default_rng(seed)
    n = w * h
    depth = (1.0 + 9.0 * rng.random(n)).astype(np.float32)
    depth[rng.random(n) < miss_frac] = FLT_MAX
    sig = synth.synth_hdr(w, h, seed + 1)
    lim = max(1, int(motion_px * 32767 / max(w, h)))
    motion = (rng.integers(-lim, lim + 1, n), rng.integers(-lim, lim + 1, n))
    return depth, motion, sig


def random_history(w, h, seed):
    rng = np.random.default_rng(seed)
    return half_plane(rng.random((w * h, 3)) * 2.0)


# ======================================================================================================== compositing
@pytest.mark.parametrize("w,h", SIZES)
def test_compositing_every_toggle(oracle, w, h):
    rng = np.random.default_rng(w * 1000 + h)
    n = w * h
    flags = rng.choice(np.array([0, F_EMISSIVE, F_INVALID, F_EMISSIVE | F_INVALID], dtype=np.uint32), size=n)
    flags[0] = F_EMISSIVE                   # every size has an emissive pixel and (below) an invalid one
    flags[-1] |= F_INVALID
    depth = np.where(flags & F_INVALID, FLT_MAX, 2.0).astype(np.float32)
    core, _, _ = planes(w, h, depth, flags)
    direct = rgba(rng.random((n, 3)) * 3.0 - 0.5)
    indirect = rgba(rng.random((n, 3)) * 3.0)
    for emissive_di in (0, 1):
        for indirect_on in (0, 1):
            for accumulate in (0, 1):
                for static in (0, 1):
                    for nf in (1, 3, 7):
                        fc = frame_constants(w, h, accumulate, static, nf)
                        dr = direct if emissive_di else None
                        ir = indirect if indirect_on else None
                        got = oracle_compositing(oracle, fc, core, dr, ir)[:, :3].astype(np.float64)
                        truth = ip.compositing(w, h, core[:, 3], dr, ir, accumulate, static, nf)
                        what = "di %d ind %d acc %d static %d N %d" % (emissive_di, indirect_on, accumulate, static, nf)
                        ulp32 = np.spacing(np.abs(truth).astype(np.float32)).astype(np.float64)
                        assert (np.abs(got - truth) <= 2 * ulp32).all(), what
                        acc = accumulate and static
                        if emissive_di + indirect_on <= 1 and (nf == 1 or not acc):
                            assert got.astype(np.float32).tobytes() == truth.astype(np.float32).tobytes(), what
                        # the flags do what the reference says
                        inv = (flags & F_INVALID) != 0
                        if not acc:
                            assert (got[inv] == 0).all(), what
                        em = ((flags & F_EMISSIVE) != 0) & ~inv
                        if indirect_on and not emissive_di:
                            assert (got[em] == 0).all(), what


# ======================================================================================================== firefly
def firefly_check(oracle, w, h, depth, comp, what="", max_low=0.001):
    core, d, _ = planes(w, h, depth)
    fc = frame_constants(w, h)
    got = oracle_firefly(oracle, fc, core, comp)[:, :3]
    truth, margin = ip.firefly(w, h, d, comp)
    low = margin < 4 * EPS32
    ok = (got.astype(np.float64) == truth).all(axis=1) | np.isnan(truth).all(axis=1) & np.isnan(got).all(axis=1)
    assert ok[~low].all(), "%s: %d pixels differ, first %d" % (what, (~ok & ~low).sum(), np.argwhere(~ok & ~low)[0][0])
    assert low.sum() <= max(1, max_low * w * h), "%s: %d low-margin pixels" % (what, low.sum())
    # a low-margin pixel picked its own colour or one of its neighbours'
    cols = comp[:, :3].reshape(h, w, 3)
    for p in np.flatnonzero(low & ~ok):
        y, x = divmod(int(p), w)
        cand = cols[max(y - 1, 0):y + 2, max(x - 1, 0):x + 2].reshape(-1, 3)
        assert (cand == got[p]).all(axis=1).any(), what
    return got, truth


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("accumulate", [0, 1])
def test_firefly_random(oracle, w, h, accumulate):
    """Seeded frames through compositing and the filter; with accumulation, invalid pixels keep their colour in the image and
    (no geometry) never act as neighbours."""
    core, depth, _ = synth.synth_gbuffer(w, h, 31 + w + h, miss_frac=0.15)
    direct, indirect = synth.synth_hdr(w, h, 32), synth.synth_hdr(w, h, 33)
    fc = frame_constants(w, h, accumulate, accumulate, 5)
    comp = oracle_compositing(oracle, fc, core, direct, indirect)
    firefly_check(oracle, w, h, depth, comp, "random")


def tie_colours(scale=1.0):
    """Two different colours of exactly equal luminance in float32 and float64: c_r * c_g in red and in green."""
    cr, cg = (np.float32(v) for v in (0.2126, 0.7152))
    a = np.array([cg, 0, 0], dtype=np.float32) * np.float32(scale)
    b = np.array([0, cr, 0], dtype=np.float32) * np.float32(scale)
    return a, b


@pytest.mark.parametrize("centre", ["darker", "brighter", "equal"])
def test_firefly_luminance_ties(oracle, centre):
    """Neighbours whose luminances tie exactly: the first valid neighbour in y-outer, x-inner order lands in min, the next one in
    max (strict <, else-if), so a darker centre takes the first and a brighter one the second."""
    w, h = 5, 4
    a, b = tie_colours(2.0)
    rng = np.random.default_rng(5)
    cols = np.where(rng.random((w * h, 1)) < 0.5, a, b).astype(np.float32)
    la = ip.luminance(a.astype(np.float64))
    assert la == ip.luminance(b.astype(np.float64)) and np.float32(la) == np.float32(np.dot(a, np.float32([0.2126, 0.7152, 0.0722])))
    centre_col = {"darker": a * np.float32(0.5), "brighter": a * np.float32(2.0), "equal": b}[centre]
    for p in range(w * h):
        c = cols.copy()
        c[p] = centre_col
        got, truth = firefly_check(oracle, w, h, np.full(w * h, 3.0), rgba(c), "tie %s px %d" % (centre, p), max_low=0)
        y, x = divmod(p, w)
        order = [(y + i) * w + x + j for i in (-1, 0, 1) for j in (-1, 0, 1)
                 if (i or j) and 0 <= y + i < h and 0 <= x + j < w]
        expect = {"darker": c[order[0]], "brighter": c[order[1]], "equal": c[p]}[centre]
        assert (got[p] == expect).all(), (centre, p)


def test_firefly_no_geometry_around(oracle):
    """Every neighbour without geometry: min stays FLT_MAX and max 0, so the centre is kept; an invalid centre passes through
    whatever its neighbours are."""
    w, h = 7, 5
    rng = np.random.default_rng(9)
    col = rgba(rng.random((w * h, 3)) * 50.0)
    depth = np.full(w * h, FLT_MAX, dtype=np.float32)
    isolated = [0, 2 * w + 3, w * h - 1, 4]
    for p in isolated:
        depth[p] = 2.0
    got, _ = firefly_check(oracle, w, h, depth, col, "isolated")
    assert (got == col[:, :3]).all()
    # invalid centres inside a valid neighbourhood of fireflies
    depth = np.full(w * h, 2.0, dtype=np.float32)
    depth[[8, 9, 17, 33]] = FLT_MAX
    col[[1, 10, 16]] *= 400
    got, _ = firefly_check(oracle, w, h, depth, col, "invalid centre")
    assert (got[[8, 9, 17, 33]] == col[[8, 9, 17, 33], :3]).all()


# ======================================================================================================== TAA
@pytest.mark.parametrize("w,h", SIZES)
def test_taa_sequence(oracle, w, h):
    """Four frames, each taking the oracle's previous output as history (the first frame has none)."""
    st = TaaStats()
    prev = np.zeros((w * h, 2), dtype=np.uint32)
    for fr in range(4):
        depth, motion, sig = random_frame(w, h, 40 + fr, motion_px=2.0)
        prev, _ = run_taa_case(oracle, st, w, h, depth, motion, sig, prev, valid=fr > 0, what="frame %d" % fr)
    st.finish()


@pytest.mark.parametrize("w,h", [(7, 3), (33, 17), (257, 131)])
def test_taa_footprint_over_edges(oracle, w, h):
    """Motions of up to a third of the image: the 4 x 4 Catmull-Rom footprint covers every edge and corner (clamp addressing),
    and many pixels lose their history (prevUV outside [0, 1])."""
    st = TaaStats()
    for seed in range(3):
        depth, motion, sig = random_frame(w, h, 60 + seed, motion_px=max(w, h) / 3.0)
        got, t = run_taa_case(oracle, st, w, h, depth, motion, sig, random_history(w, h, seed), what="seed %d" % seed)
        assert (t["path"] == 1).any() and (t["path"] == 2).any()
    # prevUV pushed onto each corner texel: motion = currUV - corner centre
    for cx, cy in ((0, 0), (w - 1, 0), (0, h - 1), (w - 1, h - 1)):
        ys, xs = np.mgrid[0:h, 0:w]
        mx = np.round(((xs + 0.5) / w - (cx + 0.3) / w) * 32767).astype(np.int64)
        my = np.round(((ys + 0.5) / h - (cy + 0.7) / h) * 32767).astype(np.int64)
        depth, _, sig = random_frame(w, h, 70)
        run_taa_case(oracle, st, w, h, depth, (mx, my), sig, random_history(w, h, 71), what="corner %d %d" % (cx, cy))
    st.finish()


def test_taa_flat_neighbourhood(oracle):
    """A flat 3 x 3 neighbourhood has std exactly 0 (dyadic colours): history inside the box (equal to it) is kept, history
    outside collapses onto the centre; extents 0 makes 0/0 and x/0 in ClipAABB, which max's NaN rule resolves."""
    w, h = 9, 7
    st = TaaStats()
    flat = np.array([0.75, 1.5, 0.375], dtype=np.float32)
    sig = np.tile(flat, (w * h, 1))
    depth = np.full(w * h, 4.0)
    zero = (np.zeros(w * h), np.zeros(w * h))
    for hist, expect in ((flat, flat), (flat * 2, flat), (np.array([0.75, 1.5, 9.0]), flat), (np.zeros(3), flat)):
        got, t = run_taa_case(oracle, st, w, h, depth, zero, sig, half_plane(np.tile(hist, (w * h, 1))), what=str(hist))
        assert (decode(got, w, h) == flat.astype(np.float64)).all()
        assert (t["path"] == 2).all()
    st.finish()


def test_taa_negative_centre(oracle):
    """Negative signal: the centre enters the moments as it is, the neighbours clamped to 0."""
    w, h = 8, 6
    st = TaaStats()
    rng = np.random.default_rng(3)
    for seed in range(4):
        sig = (rng.random((w * h, 3)) * 4.0 - 2.0).astype(np.float32)
        depth, motion, _ = random_frame(w, h, 80 + seed, motion_px=1.0, miss_frac=0.0)
        got, t = run_taa_case(oracle, st, w, h, depth, motion, sig, random_history(w, h, seed), what="neg %d" % seed)
        assert (t["out"] < 0).any()
    st.finish()


def test_taa_nan_inf(oracle):
    """NaN / Inf in the signal and in the history: a NaN neighbour is clamped to 0 (maxNum), an Inf one poisons the moments, a
    NaN or Inf history texel under the footprint turns the blend NaN, and the NaN guard then returns the reconstruction. The
    history cases move by a fraction of a texel, so every texel under the footprint has a non-zero bilinear weight (DESIGN 6.3:
    a non-finite texel of zero weight is outside what the truth and the kernels agree on)."""
    w, h = 9, 7
    st = TaaStats()
    rng = np.random.default_rng(12)
    base = rng.random((w * h, 3)) * 2.0
    depth = np.full(w * h, 4.0)
    zero = (np.zeros(w * h), np.zeros(w * h))
    c = 3 * w + 4
    frac = (np.full(w * h, round(0.3 * 32767 / w)), np.full(w * h, round(0.4 * 32767 / h)))
    for name, sval, hval in (("nan neighbour", np.nan, None), ("inf neighbour", np.inf, None), ("-inf neighbour", -np.inf, None),
                             ("nan history", None, np.nan), ("inf history", None, np.inf)):
        sig = base.copy()
        hist = rng.random((w * h, 3)) * 2.0
        if sval is not None:
            sig[c + 1, 1] = sval
        if hval is not None:
            hist[c, 0] = hval
        got, t = run_taa_case(oracle, st, w, h, depth, frac, sig.astype(np.float32), half_plane(hist), what=name)
        if hval is not None:
            assert (t["out"][c] == t["rec"][c]).all(), name          # the guard fired
    for name, val in (("nan centre", np.nan), ("inf centre", np.inf)):
        sig = base.copy()
        sig[c, 2] = val
        got, t = run_taa_case(oracle, st, w, h, depth, zero, sig.astype(np.float32), random_history(w, h, 1), what=name)
    st.finish()


def test_taa_fp16_overflow(oracle):
    """Results beyond 65504 round to Inf at the store, just below stay finite."""
    w, h = 6, 5
    st = TaaStats()
    zero = (np.zeros(w * h), np.zeros(w * h))
    for v in (65504.0, 65519.0, 65520.0, 1e6, 3e38):
        sig = np.full((w * h, 3), v, dtype=np.float32)
        sig[:, 1] = 1.0
        run_taa_case(oracle, st, w, h, np.full(w * h, 4.0), zero, sig, np.zeros((w * h, 2), np.uint32), valid=0, what="pass %g" % v)
        got, t = run_taa_case(oracle, st, w, h, np.full(w * h, 4.0), zero, sig, half_plane(np.minimum(sig, 65504.0)),
                              what="blend %g" % v)
    assert np.isinf(decode(got, w, h)[:, 0]).all()
    st.finish()


def distinct_motion(w, h, seed, px=3.0):
    """A different motion vector at every pixel, up to px pixels, so whichever tap's motion is read shows in the history."""
    rng = np.random.default_rng(seed)
    lim = int(px * 32767 / max(w, h))
    codes = rng.choice((2 * lim + 1) ** 2, size=w * h, replace=False)
    return codes % (2 * lim + 1) - lim, codes // (2 * lim + 1) - lim


@pytest.mark.parametrize("w,h", [(2, 2), (7, 3), (33, 17)])
def test_taa_depth_dilation(oracle, w, h):
    """The motion is read at the closest-depth tap. Distinct motion per pixel and a high-contrast history make the chosen tap
    visible; depths drawn from three values make exact ties, which the first tap in (dx outer, dy inner) order must win."""
    st = TaaStats()
    rng = np.random.default_rng(w + h)
    for seed in range(4):
        motion = distinct_motion(w, h, seed)
        depth = rng.choice(np.float32([1.0, 2.0, 3.0]), size=w * h) if seed % 2 else (1.0 + rng.random(w * h) * 9).astype(np.float32)
        sig = synth.synth_hdr(w, h, seed)
        hist = half_plane(np.where(rng.random((w * h, 1)) < 0.5, 0.05, 8.0) * rng.random((w * h, 3)))
        _, t = run_taa_case(oracle, st, w, h, depth, motion, sig, hist, what="seed %d" % seed)
        assert len(np.unique(t["dil"])) > 1
    st.finish()


def uv_landing(target, sizes=range(2, 400)):
    """(size, column, k): the first image size with a pixel column whose float32 prevUV = currUV - k / 32767 is exactly target
    (0 or 1). Such columns exist at one pixel in a few hundred: they are where the float32 rounding of currUV and of the snorm
    decode meet."""
    for size in sizes:
        cu = ((np.arange(size) + 0.5) / size).astype(np.float32)
        k = np.round((cu.astype(np.float64) - target) * 32767).astype(np.int64)
        for dk in (0, -1, 1):
            kk = k + dk
            mv = (kk / 32767.0).astype(np.float32)
            hit = np.flatnonzero((np.abs(kk) <= 32767) & ((cu - mv) == np.float32(target)))
            if hit.size:
                return size, int(hit[0]), int(kk[hit[0]])
    raise AssertionError("no exact landing on %g" % target)


@pytest.mark.parametrize("target", [0.0, 1.0])
@pytest.mark.parametrize("axis", [0, 1])
def test_taa_reprojection_edges(oracle, target, axis):
    """prevUV exactly 0.0 or 1.0 is inside (the reference rejects < 0 and > 1); one snorm step beyond is outside, one step back
    inside."""
    size, col, k = uv_landing(target)
    w, h = (size, 3) if axis == 0 else (3, size)
    st = TaaStats()
    depth = np.full(w * h, 4.0)
    _, _, sig = random_frame(w, h, 90)
    hist = random_history(w, h, 91)
    for step in (0, -1, 1):
        m = [np.zeros((h, w), dtype=np.int64), np.zeros((h, w), dtype=np.int64)]
        sel = (slice(None), col) if axis == 0 else (col, slice(None))
        m[axis][sel] = k + step
        _, t = run_taa_case(oracle, st, w, h, depth, (m[0], m[1]), sig, hist, what="step %d" % step)
        beyond = (step == 1) if target == 0.0 else (step == -1)
        assert ((t["path"].reshape(h, w)[sel] == 1) == beyond).all(), step
    st.finish()


def test_taa_snorm_minimum(oracle):
    """snorm -32768 decodes to -1 like -32767; both, and +32767, on either axis."""
    w, h = 33, 17
    st = TaaStats()
    depth = np.full(w * h, 4.0)
    _, _, sig = random_frame(w, h, 92)
    hist = random_history(w, h, 93)
    outs = {}
    for code in (-32768, -32767, 32767):
        for axis in (0, 1):
            m = [np.zeros(w * h), np.zeros(w * h)]
            m[axis] = np.full(w * h, code)
            outs[code, axis], _ = run_taa_case(oracle, st, w, h, depth, (m[0], m[1]), sig, hist, what="snorm %d %d" % (code, axis))
    for axis in (0, 1):
        assert outs[-32768, axis].tobytes() == outs[-32767, axis].tobytes()
    st.finish()


@pytest.mark.parametrize("bw", [0.0, 0.1, 0.5, 1.0, 1.5])
def test_taa_blend_weight(oracle, bw):
    """The blend weight over its range (1.5 saturates the current weight and makes the history weight negative, saturated
    to 0); at 1 with an infinite-luminance reconstruction the current weight is 0/Inf -> 0, histWeight 0, and 0/0 is caught by
    the NaN guard."""
    w, h = 33, 17
    st = TaaStats()
    for seed in range(2):
        depth, motion, sig = random_frame(w, h, 100 + seed, motion_px=2.0)
        run_taa_case(oracle, st, w, h, depth, motion, sig, random_history(w, h, seed), bw=bw, what="bw %g" % bw)
    if bw == 1.0:
        sig = np.full((w * h, 3), 2.0, dtype=np.float32)
        sig[5 * w + 7] = (np.inf, 1.0, 1.0)
        got, t = run_taa_case(oracle, st, w, h, np.full(w * h, 4.0), (np.zeros(w * h), np.zeros(w * h)), sig,
                              random_history(w, h, 7), bw=bw, what="inf rec")
        p = 5 * w + 7
        assert np.isinf(t["out"][p, 0]) and t["path"][p] == 2 and (t["out"][p] == t["rec"][p]).all()
    st.finish()


def test_taa_static_fixed_point(oracle):
    """Static camera, zero motion, constant signal: after the first frame, the output equals the signal on every frame."""
    w, h = 33, 17
    st = TaaStats()
    sig = np.tile(np.float32([0.25, 1.125, 3.5]), (w * h, 1))
    depth = (1.0 + np.random.default_rng(1).random(w * h) * 9).astype(np.float32)
    zero = (np.zeros(w * h), np.zeros(w * h))
    prev = np.zeros((w * h, 2), dtype=np.uint32)
    for fr in range(5):
        prev, t = run_taa_case(oracle, st, w, h, depth, zero, sig, prev, valid=fr > 0, what="frame %d" % fr)
        assert (decode(prev, w, h) == sig.astype(np.float64)).all(), fr
        assert np.allclose(t["out"], sig, rtol=1e-12, atol=0), fr
    st.finish()


def test_taa_mitchell_quirk(oracle):
    """Reference quirk kept on purpose (DESIGN 6.5): Mitchell1D gets the integer tap offset, |2x| = 2 is the filter's zero, so
    the reconstruction is the centre. The truth's neighbour weight is 0; the oracle's float32 one is Mitchell1D_f32(1) ~ 1.1e-6,
    i.e. a neighbour counts at most 2e-6 of the centre. A 'fixed' filter (x / 2) would weigh it near 0.5."""
    w, h = 2, 1
    st = TaaStats()
    sig = np.float32([[0.0, 0.0, 0.0], [0.0, 0.0, 1.0]])     # centre black, its one neighbour blue
    got, t = run_taa_case(oracle, st, w, h, np.full(2, 4.0), (np.full(2, 32767), np.zeros(2)), sig,
                          np.zeros((2, 2), np.uint32), what="quirk")
    assert t["path"][0] == 1 and abs(ip.mitchell1d(1.0)) < 1e-15 and (t["rec"][0] == 0).all()
    v = decode(got, w, h)[0]
    ratio = v[2] * (1.0 + float(np.float32(0.0722))) / 1.0    # neighbour weight relative to the centre's
    assert 0 < ratio < 2e-6 and v[0] == 0 and v[1] == 0
    st.finish()
