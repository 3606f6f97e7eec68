"""ORACLE -- test infrastructure, not product code.

Independent float64 truth of the stencils between lighting and display: Compositing, the firefly filter and TAA. It is written
from the reference's formulas (cited, not copied) and shares nothing with oracle/orc_post.cpp, zetaray_b200/csrc/post.cu or
oracle/liborc.so; its inputs are the same numpy planes the oracle and the kernels read (float32 colours, the G-buffer's core
flags and depth, R16G16_SNORM motion, the RGBA16F history). Every function is vectorised over pixels; only the eight 3 x 3 taps
and the nine Catmull-Rom taps are loops.

IEEE semantics are mirrored where the reference depends on them: HLSL max / min are maxNum / minNum (np.fmax / np.fmin: a NaN
operand loses), every comparison with NaN is false, saturate(NaN) = 0, and a result is stored to fp16 with round-to-nearest-even
and overflow to Inf (to_half).

Compositing (Compositing/Compositing.hlsl:30-73):
  * accumulate = Accumulate && CameraStatic (:41); an invalid pixel without accumulation writes the background (:43-47), 0 here
    because sky lighting is out of scope (DESIGN 6.3);
  * the emissive-DI image is added when its toggle is on (:58-62), the indirect image when its toggle is on and the pixel is not
    emissive (:65-69): the emissive flag drops indirect only;
  * the sum is divided by NumFramesCameraStatic only when accumulating (:50, :72).

Firefly filter (Compositing/FireflyFilter.hlsl:35-124), on the composited image:
  * a pixel without geometry (depth == FLT_MAX) keeps its colour (:108-112);
  * neighbours are visited y outer, x inner (:49-57); one that is outside the image is skipped -- the test is written
    any(addr) < 0 || any(addr >= renderDim) with renderDim a uint2, so the first half is always false and negative addresses are
    skipped only because they compare as unsigned -- and so is one without geometry (:61-63);
  * min / max luminance update with a strict < and an else-if (:73-82): the first valid neighbour always lands in min;
  * the centre is replaced by the min colour if darker than every neighbour, by the max colour if brighter, and kept when
    minLum > maxLum (:86-87).
  Luminance is Math.hlsli:693-696 with the float32 coefficients the literals denote.

TAA (TAA/TAA.hlsl:68-189 with DEPTH_DILATION and CATMULL_ROM_FILTERING on, Common/Common.hlsli:65-101):
  * no valid history or no geometry: the signal passes through (:81-85);
  * 3 x 3 neighbourhood with the offset (i, j) = (dx, dy), i outer (:100-136): out-of-image taps skipped, neighbours clamped to >= 0
    (the centre is not), weight Mitchell1D(i) Mitchell1D(j) / (1 + L), first and second moments, and the closest depth with a strict
    < so the first tap in order wins a tie;
  * Mitchell1D (:29-45) is called with the integer offset, so |2x| = 2 sits on the filter's zero: the neighbour weights are 0 here
    (and about 1e-6 in float32), and the reconstruction is the centre. That is a reference quirk kept on purpose (DESIGN 6.5);
  * motion is read at the dilated neighbour (:144) and decoded as R16G16_SNORM: -32768 and -32767 both map to -1;
  * currUV = (p + 0.5) / renderDim, prevUV = currUV - motion (:150-152), and a prevUV outside [0, 1] returns the reconstruction
    (:155-159). These values, and samplePos = prevUV * texSize (Common.hlsli:67), are the float32 numbers the reference forms:
    each is one IEEE operation, which float64 followed by rounding to float32 reproduces exactly (53 >= 2 * 24 + 2). They locate
    the history rather than compute with it: the truth makes the same in / out decision on motions that land prevUV exactly on
    0 or 1, and at 2560 pixels a float32 samplePos is only good to 1/8000 of a texel, which moves a Catmull-Rom sample of a
    high-contrast history by far more than the stencil's arithmetic error;
  * history: nine SampleLevel taps at texPos{0,12,3} / texSize, each a clamp-addressed bilinear with exact weights (DESIGN 6.3).
    The sampler maps uv back to texel space by uv * texSize, which the truth does exactly, and a texel whose bilinear weight is
    exactly 0 contributes nothing;
  * mean and standard deviation with Bessel's correction (:170-174), ClipAABB towards the box centre (:48-62), the inverse-luminance
    blend with saturated weights (:180-182) and the NaN guard (:186)."""
import numpy as np

FLT_MAX = float(np.float32(3.402823466e+38))
LUM = np.float32([0.2126, 0.7152, 0.0722]).astype(np.float64)
MITCHELL_B = MITCHELL_C = float(np.float32(0.33))
FLAG_EMISSIVE, FLAG_INVALID = 0x02, 0x04


def to_half(v):
    """float64 -> fp16 with round-to-nearest-even, overflow to +-Inf (numpy rounds the double directly)."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(v, dtype=np.float64).astype(np.float16)


def f32(v):
    """Round float64 to float32 (used only for the float32 coordinates that locate the history, see the module docstring)."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(v, dtype=np.float64).astype(np.float32).astype(np.float64)


def luminance(c):
    return c[..., 0] * LUM[0] + c[..., 1] * LUM[1] + c[..., 2] * LUM[2]


def saturate(v):
    return np.fmin(np.fmax(v, 0.0), 1.0)


def decode_half4(prev, w, h):
    """RGBA16F history stored as uint2 per pixel -> (h, w, 3) float64."""
    p = np.asarray(prev, dtype=np.uint32).reshape(h, w, 2)
    lo = (p & 0xffff).astype(np.uint16).view(np.float16)
    hi = (p >> 16).astype(np.uint16).view(np.float16)
    return np.stack([lo[..., 0], hi[..., 0], lo[..., 1]], axis=-1).astype(np.float64)


def decode_snorm16(u):
    """R16G16_SNORM channel: i / 32767, with -32768 mapped to -1 like -32767."""
    i = (np.asarray(u, dtype=np.uint32) & 0xffff).astype(np.uint16).view(np.int16).astype(np.float64)
    return np.where(i == -32768, -1.0, i / 32767.0)


def mitchell1d(x, b=MITCHELL_B, c=MITCHELL_C):
    x = abs(2.0 * x)
    if x > 1:
        return ((-b - 6 * c) * x ** 3 + (6 * b + 30 * c) * x ** 2 + (-12 * b - 48 * c) * x + (8 * b + 24 * c)) / 6.0
    return ((12 - 9 * b - 6 * c) * x ** 3 + (-18 + 12 * b + 6 * c) * x ** 2 + (6 - 2 * b)) / 6.0


def _rgb(a, w, h):
    return np.asarray(a, dtype=np.float32).reshape(h, w, -1)[..., :3].astype(np.float64)


def _shift(a, dx, dy, fill):
    """b[y, x] = a[y + dy, x + dx], fill where that lies outside the image."""
    h, w = a.shape[:2]
    b = np.full_like(a, fill)
    ys, yd = slice(max(dy, 0), h + min(dy, 0)), slice(max(-dy, 0), h + min(-dy, 0))
    xs, xd = slice(max(dx, 0), w + min(dx, 0)), slice(max(-dx, 0), w + min(-dx, 0))
    b[yd, xd] = a[ys, xs]
    return b


def _inside(w, h, dx, dy):
    return _shift(np.ones((h, w), dtype=bool), dx, dy, False)


# ---------------------------------------------------------------------------------------------------------------------------
def compositing(w, h, flags, direct, indirect, accumulate, camera_static, num_frames):
    """Composited colour, (h * w, 3) float64. direct / indirect: float4[w * h] or None (toggle off); flags: the core plane's low
    byte (or the whole .w word)."""
    flags = np.asarray(flags, dtype=np.uint32).reshape(-1) & 0xff
    acc = bool(accumulate) and bool(camera_static)
    color = np.zeros((w * h, 3))
    if direct is not None:
        color = color + _rgb(direct, w, h).reshape(-1, 3)
    if indirect is not None:
        color = color + np.where((flags & FLAG_EMISSIVE)[:, None] != 0, 0.0, _rgb(indirect, w, h).reshape(-1, 3))
    if acc:
        color = color / float(num_frames)
    return np.where(((flags & FLAG_INVALID) != 0)[:, None] & (not acc), 0.0, color)


def firefly(w, h, depth, color):
    """Firefly filter of a composited float32 image. Returns (out (h * w, 3) float64, margin (h * w,)).

    margin is the pixel's smallest relative luminance gap |a - b| / max(|a|, |b|) over every comparison that drove its selection
    (neighbour against the running min and max, centre against both, min against max); exact ties are left out, since float32
    reproduces them. A pixel whose margin is within a few float32 epsilons may have picked the other side of a near-tie."""
    c = _rgb(color, w, h)
    d = np.asarray(depth, dtype=np.float32).reshape(h, w).astype(np.float64)
    L = luminance(c)
    min_l = np.full((h, w), FLT_MAX)
    max_l = np.zeros((h, w))
    min_c = c.copy()
    max_c = np.zeros_like(c)
    margin = np.full((h, w), np.inf)

    def gap(a, b, where):
        with np.errstate(invalid="ignore", divide="ignore"):
            g = np.abs(a - b) / np.fmax(np.abs(a), np.abs(b))
        return np.where(where & (a != b), g, np.inf)

    for dy in (-1, 0, 1):                       # FireflyFilter.hlsl:49-57: i is the row offset, j the column offset
        for dx in (-1, 0, 1):
            if dx == 0 and dy == 0:
                continue
            ok = _inside(w, h, dx, dy) & (_shift(d, dx, dy, FLT_MAX) != FLT_MAX)
            nl = _shift(L, dx, dy, 0.0)
            nc = _shift(c, dx, dy, 0.0)
            lt = ok & (nl < min_l)
            gt = ok & ~lt & (nl > max_l)
            margin = np.fmin(margin, gap(nl, min_l, ok))
            margin = np.fmin(margin, gap(nl, max_l, ok & ~lt))
            min_l = np.where(lt, nl, min_l)
            min_c = np.where(lt[..., None], nc, min_c)
            max_l = np.where(gt, nl, max_l)
            max_c = np.where(gt[..., None], nc, max_c)
    darker = L < min_l
    brighter = ~darker & (L > max_l)
    ret = np.where(darker[..., None], min_c, np.where(brighter[..., None], max_c, c))
    ret = np.where((min_l <= max_l)[..., None], ret, c)
    geom = d != FLT_MAX
    margin = np.fmin(margin, gap(L, min_l, geom))
    margin = np.fmin(margin, gap(L, max_l, geom & ~darker))
    margin = np.fmin(margin, gap(min_l, max_l, geom))
    out = np.where(geom[..., None], ret, c)
    return out.reshape(-1, 3), np.where(geom, margin, np.inf).reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------------
def _bilinear(img, px, py):
    """Clamp-addressed bilinear with exact weights at texel-space position (px, py) (texel centres at k + 0.5)."""
    h, w = img.shape[:2]
    sx, sy = px - 0.5, py - 0.5
    x0, y0 = np.floor(sx), np.floor(sy)
    fx, fy = sx - x0, sy - y0
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
    out = np.zeros(px.shape + (3,))
    for ox, wx in ((0, 1.0 - fx), (1, fx)):
        for oy, wy in ((0, 1.0 - fy), (1, fy)):
            wt = wx * wy
            t = img[np.clip(y0 + oy, 0, h - 1), np.clip(x0 + ox, 0, w - 1)]
            with np.errstate(invalid="ignore"):
                out = out + np.where((wt != 0)[..., None], t * wt[..., None], 0.0)
    return out


def catmull_rom(img, u, v):
    """Common.hlsli:65-101: nine bilinear taps at texPos{0,12,3} / texSize, weighted by the Catmull-Rom weights."""
    h, w = img.shape[:2]
    taps = []
    for s in (f32(u * w), f32(v * h)):         # samplePos = uv * texSize, a float32 in the reference (see the module docstring)
        t1 = np.floor(s - 0.5) + 0.5
        f = s - t1
        w0 = f * (-0.5 + f * (1.0 - 0.5 * f))
        w1 = 1.0 + f * f * (-2.5 + 1.5 * f)
        w2 = f * (0.5 + f * (2.0 - 1.5 * f))
        w3 = f * f * (-0.5 + 0.5 * f)
        w12 = w1 + w2
        taps.append(((t1 - 1.0, w0), (t1 + w2 / w12, w12), (t1 + 2.0, w3)))
    out = np.zeros(u.shape + (3,))
    with np.errstate(invalid="ignore", over="ignore"):
        for py, wy in taps[1]:
            for px, wx in taps[0]:
                out = out + _bilinear(img, px, py) * (wx * wy)[..., None]
    return out


def clip_aabb(lo, hi, hist):
    """TAA.hlsl:48-62: move the history towards the box centre until it lies on the box (max is maxNum)."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        center = 0.5 * (hi + lo)
        extents = 0.5 * (hi - lo)
        ray = hist - center
        unit = np.abs(ray / extents)
        m = np.fmax(unit[..., 0], np.fmax(unit[..., 1], unit[..., 2]))
        return np.where((m > 1.0)[..., None], center + ray / m[..., None], hist)


def taa(w, h, depth, motion, signal, prev, blend_weight, temporal_valid):
    """TAA of one frame. depth: float32[w * h]; motion: the motion_emissive plane's .x words (uint32[w * h]); signal: float4[w * h];
    prev: the previous output, uint2[w * h] RGBA16F. Returns a dict of (h * w, ...) float64 arrays:
      out    the result before the fp16 store,
      rec    the reconstruction (the centre, up to the Mitchell quirk),
      path   0 = signal passed through, 1 = reconstruction (no history), 2 = blended with the clipped history,
      dil    index 0-8 of the tap whose motion was read (4 = the pixel itself, dx-major like the reference's loop),
      scale  largest |rgb| over the centre, the clamped neighbours and the 4 x 4 history texels under the Catmull-Rom footprint
             (the magnitude the float32 rounding of the moments, the clip and the blend scales with)."""
    blend_weight = float(np.float32(blend_weight))          # a float32 constant in the reference
    sig = _rgb(signal, w, h)
    d = np.asarray(depth, dtype=np.float32).reshape(h, w).astype(np.float64)
    mv = np.asarray(motion, dtype=np.uint32).reshape(h, w)
    hist_img = decode_half4(prev, w, h)
    m0 = mitchell1d(0.0)
    wsum = np.full((h, w), m0 * m0)
    rec = sig * (m0 * m0)
    m1 = sig.copy()
    m2 = sig * sig
    closest = d.copy()
    cdx = np.zeros((h, w), dtype=np.int64)
    cdy = np.zeros((h, w), dtype=np.int64)
    n = np.ones((h, w))
    with np.errstate(invalid="ignore", over="ignore"):
        scale = np.fmax.reduce(np.abs(sig), axis=-1)
        for i in (-1, 0, 1):                    # TAA.hlsl:101-103: i is the column offset, j the row offset
            for j in (-1, 0, 1):
                if i == 0 and j == 0:
                    continue
                ok = _inside(w, h, i, j)
                nc = np.fmax(_shift(sig, i, j, 0.0), 0.0)
                wt = mitchell1d(i) * mitchell1d(j) / (1.0 + luminance(nc))
                okc = ok[..., None]
                rec = np.where(okc, rec + nc * wt[..., None], rec)
                wsum = np.where(ok, wsum + wt, wsum)
                m1 = np.where(okc, m1 + nc, m1)
                m2 = np.where(okc, m2 + nc * nc, m2)
                nd = _shift(d, i, j, FLT_MAX)
                closer = ok & (nd < closest)
                closest = np.where(closer, nd, closest)
                cdx = np.where(closer, i, cdx)
                cdy = np.where(closer, j, cdy)
                n = n + ok
                scale = np.where(ok, np.fmax(scale, np.fmax.reduce(nc, axis=-1)), scale)
        rec = rec / np.fmax(wsum, 1e-5)[..., None]

        ys, xs = np.mgrid[0:h, 0:w]
        word = mv[ys + cdy, xs + cdx]
        mvx, mvy = f32(decode_snorm16(word)), f32(decode_snorm16(word >> 16))
        pu = f32(f32((xs + 0.5) / w) - mvx)
        pv = f32(f32((ys + 0.5) / h) - mvy)
        in_range = (pu >= 0.0) & (pv >= 0.0) & (pu <= 1.0) & (pv <= 1.0)

        hist = catmull_rom(hist_img, pu, pv)
        fx = np.floor(f32(pu * w) - 0.5).astype(np.int64)
        fy = np.floor(f32(pv * h) - 0.5).astype(np.int64)
        for k in range(-1, 3):
            for l in range(-1, 3):
                t = hist_img[np.clip(fy + k, 0, h - 1), np.clip(fx + l, 0, w - 1)]
                scale = np.where(in_range, np.fmax(scale, np.fmax.reduce(np.abs(t), axis=-1)), scale)

        mean = m1 / n[..., None]
        std = np.sqrt(np.abs(m2 - m1 * m1 / n[..., None]) / (n[..., None] - 1.0))
        clipped = clip_aabb(mean - std, mean + std, hist)
        cw = saturate(blend_weight / (1.0 + luminance(rec)))
        hw = saturate((1.0 - blend_weight) / (1.0 + luminance(clipped)))
        res = (cw[..., None] * rec + hw[..., None] * clipped) / (cw + hw)[..., None]
        res = np.where(np.isnan(res).any(axis=-1)[..., None], rec, res)

    passthrough = np.broadcast_to(not temporal_valid, (h, w)) | (d == FLT_MAX)
    out = np.where(passthrough[..., None], sig, np.where(in_range[..., None], res, rec))
    path = np.where(passthrough, 0, np.where(in_range, 2, 1))
    dil = (cdx + 1) * 3 + (cdy + 1)
    return {"out": out.reshape(-1, 3), "rec": rec.reshape(-1, 3), "path": path.reshape(-1), "dil": dil.reshape(-1),
            "scale": scale.reshape(-1)}
