"""The post-processing oracle (oracle/orc_display.cpp: luminance bins, exposure, tone mappers, sRGB OETF) against an
independent float64 restatement written here from the reference's formulas (AutoExposure_Histogram.hlsl,
AutoExposure_WeightedAvg.hlsl, Tonemap.hlsli, IEC 61966-2-1). Bins must match exactly; values within float32-vs-float64
tolerances. No GPU."""
import ctypes as C
import hashlib
import os
import re

import numpy as np
import pytest

from tests.orc import ptr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LW = np.array([0.2126, 0.7152, 0.0722])
AGX_MAT = np.array([[0.842479062253094, 0.0423282422610123, 0.0423756549057051],
                    [0.0784335999999992, 0.878468636469772, 0.0784336],
                    [0.0792237451477643, 0.0791661274605434, 0.879142973793104]])
AGX_MAT_INV = np.array([[1.19687900512017, -0.0528968517574562, -0.0529716355144438],
                        [-0.0980208811401368, 1.15190312990417, -0.0980434501171241],
                        [-0.0990297440797205, -0.0989611768448433, 1.15107367264116]])
NONE, NEUTRAL, AGX_DEFAULT, AGX_GOLDEN, AGX_PUNCHY, AGX_CUSTOM = range(6)


def load_lut():
    d = np.load(os.path.join(ROOT, "tests", "golden", "tony_mc_mapface.npz"))
    lut = np.ascontiguousarray(d["lut"], dtype=np.uint32)
    assert lut.shape == (48, 48, 48)
    assert hashlib.sha256(lut.astype("<u4").tobytes()).hexdigest() == str(d["sha256"])
    return lut


def ae_params(min_lum=5e-3, max_lum=4.0, lum_map_exp=0.5, adaptation_rate=1.0):
    from zetaray_b200 import _lib
    return _lib.AutoExposureParams(min_lum, max_lum, lum_map_exp, adaptation_rate)


def disp_params(tonemapper=NEUTRAL, auto_exposure=1, saturation=1.0, agx_exp=1.0):
    from zetaray_b200 import _lib
    return _lib.DisplayParams(tonemapper, auto_exposure, saturation, agx_exp)


# ---- float64 restatement ----
def decode_rgb9e5(v):
    v = np.asarray(v, dtype=np.uint64)
    scale = np.exp2(((v >> 27) & 31).astype(np.float64) - 24.0)
    return np.stack([((v >> (9 * c)) & 511).astype(np.float64) * scale for c in range(3)], axis=-1)


def srgb_oetf(v):
    v = np.asarray(v, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        return np.where(v <= 0.0031308, 12.92 * v, 1.055 * np.power(np.maximum(v, 0.0), 1.0 / 2.4) - 0.055)


def tony(rgb, lut):
    enc = rgb / (rgb + 1.0)
    t = np.clip((enc * 47.0 / 48.0 + 0.5 / 48.0) * 48.0 - 0.5, 0.0, 47.0)
    i0 = np.floor(t).astype(np.int64)
    i1 = np.minimum(i0 + 1, 47)
    f = t - i0
    tex = decode_rgb9e5(lut)            # [z][y][x][c]
    out = np.zeros_like(rgb)
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                x = np.where(dx, i1[:, 0], i0[:, 0])
                y = np.where(dy, i1[:, 1], i0[:, 1])
                z = np.where(dz, i1[:, 2], i0[:, 2])
                w = (np.where(dx, f[:, 0], 1 - f[:, 0]) * np.where(dy, f[:, 1], 1 - f[:, 1]) * np.where(dz, f[:, 2], 1 - f[:, 2]))
                out += w[:, None] * tex[z, y, x]
    return out


def agx(rgb, look=None, m=AGX_MAT, m_inv=AGX_MAT_INV):
    with np.errstate(invalid="ignore", divide="ignore"):
        v = rgb @ m                                         # mul(row, M): out_j = sum_i v_i M[i][j]
        v = (np.clip(np.log2(v), -12.47393, 4.026069) + 12.47393) / (4.026069 + 12.47393)
        v = np.nan_to_num(v, nan=0.0)                       # HLSL clamp(NaN) -> lower bound
        x = v
        v = (-17.86 * x ** 7 + 78.01 * x ** 6 - 126.7 * x ** 5 + 92.06 * x ** 4 - 28.72 * x ** 3 + 4.361 * x ** 2 - 0.1718 * x + 0.002857)
        if look is not None:
            slope, power, sat = look
            luma = v @ LW
            v = np.power(v * np.asarray(slope), power)
            v = luma[:, None] + sat * (v - luma[:, None])
        return np.power(v @ m_inv, 2.2)


def tonemap(rgb, tm, lut=None, saturation=1.0, agx_exp=1.0):
    if tm == NONE:
        return rgb
    if tm == NEUTRAL:
        t = tony(rgb, lut)
        luma = (t @ LW)[:, None]
        return luma + saturation * (t - luma)
    looks = {AGX_DEFAULT: None, AGX_GOLDEN: ((1.0, 0.9, 0.5), 0.8, 0.8), AGX_PUNCHY: (1.0, 1.35, 1.4),
             AGX_CUSTOM: (1.0, agx_exp, saturation)}
    return agx(rgb, looks[tm])


def bins64(rgba, p):
    c = rgba[:, :3].astype(np.float16).astype(np.float64)
    lum = c @ LW
    with np.errstate(invalid="ignore"):
        t = np.nan_to_num((lum - p.min_lum) / (p.max_lum - p.min_lum), nan=0.0)
        t = np.clip(t, 0.0, 1.0) ** p.lum_map_exp
        b = np.minimum(np.floor(t * 254).astype(np.int64) + 1, 255)
        return np.where(lum <= 1e-4, 0, b), t * 254, lum


def exposure64(hist, num_pixels, p, dt, prev):
    i = np.arange(256)
    vals = np.where(i == 0, 0.0, hist.astype(np.float64) * (i - 1 + 0.5) / 256.0)
    n = max(int(num_pixels) - int(hist[0]), 1)
    mean = vals.sum() / n
    result = mean ** (1.0 / p.lum_map_exp) * (p.max_lum - p.min_lum) + p.min_lum
    if prev < 1e8:
        result = prev + (result - prev) * (1.0 - np.exp(-dt * 1000.0 * p.adaptation_rate))
    ev100 = np.log2(result * 100.0 / 12.5)
    return 1.0 / ((78.0 / 65.0) * 2.0 ** ev100), result


# ---- tests ----
def test_lut_fixture_is_the_packed_48_cube():
    lut = load_lut()
    e = lut >> 27
    assert e.min() >= 3 and e.max() == 16
    assert lut[47, 47, 47] == 0x7fffffff            # white corner: 511 * 2^-9 in every channel


def test_rgb9e5_decode_every_exponent_and_mantissa_edge(oracle):
    mant = np.array([0, 1, 2, 255, 256, 510, 511], dtype=np.uint32)
    v = []
    for e in range(32):
        for r in mant:
            for g in (0, 511):
                v.append((e << 27) | (int(mant[-1] - r if g else r) << 18) | (g << 9) | int(r))
    v = np.array(v, dtype=np.uint32)
    got = np.zeros((len(v), 3), dtype=np.float32)
    oracle.orc_rgb9e5_decode(ptr(v), C.c_int64(len(v)), ptr(got))
    assert np.array_equal(got.astype(np.float64), decode_rgb9e5(v))      # exact: a 9-bit integer times a power of two


def test_srgb_oetf_all_binary16_inputs(oracle):
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
    x = h[np.isfinite(h)].astype(np.float32)
    got = np.zeros_like(x)
    oracle.orc_srgb_oetf(ptr(x), C.c_int64(len(x)), ptr(got))
    want = srgb_oetf(x.astype(np.float64))
    big = np.abs(want) > 1e30
    assert np.all(np.isinf(got[big]) | (np.abs(got[big] / want[big] - 1) < 1e-5))
    np.testing.assert_allclose(got[~big], want[~big], rtol=2e-6, atol=2e-8)
    # the 8-bit codes the display writes
    u = x[(x >= 0) & (x <= 1)]
    g8 = np.zeros_like(u)
    oracle.orc_srgb_oetf(ptr(u), C.c_int64(len(u)), ptr(g8))
    code32 = np.floor(g8.astype(np.float64) * 255 + 0.5)
    code64 = np.floor(srgb_oetf(u) * 255 + 0.5)
    assert np.abs(code32 - code64).max() <= 1


@pytest.mark.parametrize("tm,saturation,agx_exp", [(NEUTRAL, 1.0, 1.0), (NEUTRAL, 0.4, 1.0), (NEUTRAL, 1.3, 1.0),
                                                    (AGX_DEFAULT, 1.0, 1.0), (AGX_GOLDEN, 1.0, 1.0), (AGX_PUNCHY, 1.0, 1.0),
                                                    (AGX_CUSTOM, 1.2, 0.7), (NONE, 1.0, 1.0)])
def test_tonemappers(oracle, tm, saturation, agx_exp):
    lut = load_lut()
    rng = np.random.default_rng(31 + tm)
    rgb = np.exp(rng.uniform(np.log(1e-3), np.log(60.0), size=(4000, 3))).astype(np.float32)
    rgb[:8] = [[0, 0, 0], [1, 1, 1], [1e4, 0, 0], [0, 5, 0], [0.18, 0.18, 0.18], [0.5, 0.2, 0.9], [100, 100, 100], [2, 0.01, 0.3]]
    got = np.zeros_like(rgb)
    p = disp_params(tm, 0, saturation, agx_exp)
    oracle.orc_tonemap(ptr(rgb), C.c_int64(len(rgb)), C.byref(p), ptr(lut), ptr(got))
    want = tonemap(rgb.astype(np.float64), tm, lut, saturation, agx_exp)
    # what reaches the display: saturate (NaN -> 0 as HLSL's saturate does)
    g = np.clip(np.nan_to_num(got.astype(np.float64), nan=0.0), 0, 1)
    w = np.clip(np.nan_to_num(want, nan=0.0), 0, 1)
    np.testing.assert_allclose(g, w, atol=2e-4 if tm >= AGX_DEFAULT else 4e-6, rtol=0)


def test_agx_matrices_are_applied_as_row_vector_times_matrix(oracle):
    """mul(row, M) with the GLSL column-major constants: a pure-red input picks up M's first ROW, not its first column."""
    x = np.float32(2.0 ** -3)
    rgb = np.array([[x, 0, 0], [0, x, 0], [0, 0, x]], dtype=np.float32)
    got = np.zeros_like(rgb)
    p = disp_params(AGX_DEFAULT, 0)
    oracle.orc_tonemap(ptr(rgb), C.c_int64(3), C.byref(p), None, ptr(got))
    want_row = agx(rgb.astype(np.float64))
    want_col = agx(rgb.astype(np.float64), m=AGX_MAT.T, m_inv=AGX_MAT_INV.T)          # M applied to a column vector
    assert np.abs(got - want_row).max() < 1e-5
    assert np.abs(got - want_col).max() > 5e-4             # ~100 x the error above: the conventions are told apart


def _check_bins(oracle, rgba, p, tol=1e-3):
    got = np.zeros(len(rgba), dtype=np.uint32)
    oracle.orc_lum_bins(ptr(rgba), C.c_int64(len(rgba)), C.byref(p), ptr(got))
    want, t254, lum = bins64(rgba, p)
    # float32 and float64 may straddle a bin edge or the 1e-4 threshold only within rounding distance of it
    safe = (np.abs(t254 - np.round(t254)) > tol) & (np.abs(lum - 1e-4) > 1e-9) | np.isnan(lum)
    assert np.array_equal(got[safe], want[safe])
    return got


@pytest.mark.parametrize("prm", [dict(), dict(min_lum=0.0, max_lum=1.0, lum_map_exp=1.0), dict(min_lum=0.05, max_lum=40.0, lum_map_exp=0.25)])
def test_bin_mapping_random(oracle, prm):
    rng = np.random.default_rng(5)
    rgba = np.zeros((20000, 4), dtype=np.float32)
    rgba[:, :3] = np.exp(rng.uniform(np.log(1e-6), np.log(200.0), size=(20000, 3)))
    got = _check_bins(oracle, rgba, ae_params(**prm))
    assert len(np.unique(got)) > 200


def test_bin_mapping_edges(oracle):
    # a pixel (0, g, 0) has luminance float32(0.7152 * g) exactly (the other two products are zero)
    g = np.float16(np.arange(1 << 15, dtype=np.uint16).view(np.float16)).astype(np.float32)
    g = g[np.isfinite(g)]
    lum = np.float32(0.7152) * g
    g_lo = g[lum <= np.float32(1e-4)].max()             # last value at or below the threshold, then the first above it
    g_hi = g[lum > np.float32(1e-4)].min()
    gm, gM = np.float32(np.float16(0.25)), np.float32(np.float16(3.0))
    p = ae_params(float(np.float32(0.7152) * gm), float(np.float32(0.7152) * gM), 0.5, 1.0)
    rgba = np.zeros((7, 4), dtype=np.float32)
    rgba[:, 1] = [g_lo, g_hi, gm, gM, 2 * gM, 0, 0]
    rgba[5, 0] = np.nan
    rgba[6, 0] = np.inf
    got = np.zeros(7, dtype=np.uint32)
    oracle.orc_lum_bins(ptr(rgba), C.c_int64(7), C.byref(p), ptr(got))
    assert got[0] == 0                  # lum <= 1e-4
    assert got[1] == 1                  # just above: below MinLum saturates to 0 -> bin 1
    assert got[2] == 1                  # exactly MinLum
    assert got[3] == 255                # exactly MaxLum
    assert got[4] == 255                # above MaxLum
    assert got[5] == 1                  # NaN: saturate(NaN) = 0
    assert got[6] == 255                # +inf
    hist = np.zeros(256, dtype=np.uint32)
    oracle.orc_lum_histogram(ptr(rgba), C.c_uint32(1), C.c_uint32(0), C.c_uint32(7), C.byref(p), ptr(hist))
    assert hist.sum() == 7 and hist[0] == 1 and hist[1] == 3 and hist[255] == 3


@pytest.mark.parametrize("prm", [dict(), dict(min_lum=0.01, max_lum=10.0, lum_map_exp=0.7, adaptation_rate=0.3)])
def test_exposure_sequence(oracle, prm):
    p = ae_params(**prm)
    rng = np.random.default_rng(9)
    W, H = 640, 360
    state = np.zeros(2, dtype=np.float32)
    prev64 = 0.0
    for dt in (1 / 60, 1 / 30, 0.0, 0.25, 1e-3, 1 / 144):
        hist = rng.multinomial(W * H, rng.dirichlet(np.ones(256) * 0.3)).astype(np.uint32)
        oracle.orc_exposure(ptr(hist), C.c_uint32(W * H), C.byref(p), C.c_float(dt), ptr(state))
        exp64, adapted64 = exposure64(hist, W * H, p, np.float32(dt), prev64)
        assert abs(state[1] / adapted64 - 1) < 2e-5, (dt, state, adapted64)
        assert abs(state[0] / exp64 - 1) < 5e-5, (dt, state, exp64)
        prev64 = float(state[1])
    # every pixel in bin 0: numSamples clamps to 1, the mean is 0 and the inverse mapping gives MinLum
    state = np.zeros(2, dtype=np.float32)
    hist = np.zeros(256, dtype=np.uint32)
    hist[0] = W * H
    oracle.orc_exposure(ptr(hist), C.c_uint32(W * H), C.byref(p), C.c_float(10.0), ptr(state))
    assert abs(state[1] / p.min_lum - 1) < 1e-6


def _header_struct(name):
    txt = open(os.path.join(ROOT, "include", "zr_abi.h")).read()
    body = re.search(r"typedef struct %s\s*\{(.*?)\}\s*%s;" % (name, name), txt, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return re.findall(r"(uint32_t|float)\s+(\w+);", body)


@pytest.mark.parametrize("cname,pyname", [("zr_auto_exposure_params", "AutoExposureParams"), ("zr_display_params", "DisplayParams")])
def test_param_struct_layout_matches_header(cname, pyname):
    from zetaray_b200 import _lib
    cls = getattr(_lib, pyname)
    fields = _header_struct(cname)
    ctype = {"uint32_t": C.c_uint32, "float": C.c_float}
    assert [(n, ctype[t]) for t, n in fields] == [(n, t) for n, t in cls._fields_]
    assert C.sizeof(cls) == 4 * len(fields)
    for i, (n, _) in enumerate(cls._fields_):
        assert getattr(cls, n).offset == 4 * i


def test_tonemapper_enum_matches_header():
    from zetaray_b200.passes import Display
    txt = open(os.path.join(ROOT, "include", "zr_abi.h")).read()
    vals = dict((k, int(v)) for k, v in re.findall(r"ZR_TONEMAPPER_(\w+)\s*=\s*(\d+)", txt))
    assert vals == dict(NONE=Display.NONE, NEUTRAL=Display.NEUTRAL, AGX_DEFAULT=Display.AGX_DEFAULT, AGX_GOLDEN=Display.AGX_GOLDEN,
                        AGX_PUNCHY=Display.AGX_PUNCHY, AGX_CUSTOM=Display.AGX_CUSTOM)
