"""The sky on the CPU: zr_atan2f against float64, the host build of the device header against the oracle bit for bit, the oracle's
LUT against the independent float64 estimate (oracle/indep_sky.py), the LUT lookup against a float64 bilinear tap, the sun-disk
pixels against a float64 cone test, and the reference's atmosphere defaults in the frame constants."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import indep_sky
from tests import sky_util
from tests.sky_util import frame, oracle, oracle_background, oracle_lut, ptr

SUN_IN_VIEW = (0.0, -0.3, -1.0)         # the disk 16.7 degrees up, ahead of the default camera


def test_library_exports_what_its_header_declares():
    protos = sky_util._protos(sky_util.SKY_HEADER, "SKY_API", "sky_")
    oracle()
    out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(sky_util.SKY_DIR, "libsky.so")], check=True,
                         capture_output=True, text=True).stdout
    assert set(protos) == {l.split()[-1] for l in out.splitlines() if l.split() and l.split()[-1].startswith("sky_")}
    assert protos["sky_view_lut"] == (None, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p])


def _atan2(y, x):
    y, x = np.ascontiguousarray(y, dtype=np.float32), np.ascontiguousarray(x, dtype=np.float32)
    out = np.zeros_like(y)
    oracle().sky_atan2f(ptr(y), ptr(x), len(y), ptr(out))
    return out


def test_atan2f_within_two_ulp():
    rng = np.random.default_rng(3)
    ang = np.linspace(-np.pi, np.pi, 2_000_001)
    r = 10.0 ** rng.uniform(-30, 30, ang.size)
    y, x = (r * np.sin(ang)).astype(np.float32), (r * np.cos(ang)).astype(np.float32)
    bits = rng.integers(0, 2 ** 32, size=(2, 1_000_000), dtype=np.uint64).astype(np.uint32).view(np.float32)
    ok = np.isfinite(bits).all(axis=0)
    y, x = np.concatenate([y, bits[0][ok]]), np.concatenate([x, bits[1][ok]])
    got = _atan2(y, x).astype(np.float64)
    want = np.arctan2(y.astype(np.float64), x.astype(np.float64))
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(got - want) / ulp
    assert err.max() <= 2.0, (err.max(), y[err.argmax()], x[err.argmax()])


def test_atan2f_signed_zeros_axes_and_infinities():
    inf = np.float32(np.inf)
    cases = [(0.0, 0.0), (-0.0, 0.0), (0.0, -0.0), (-0.0, -0.0), (1.0, 0.0), (-1.0, 0.0), (0.0, 1.0), (0.0, -1.0), (-0.0, -1.0),
             (inf, 1.0), (-inf, 1.0), (1.0, inf), (1.0, -inf), (-1.0, -inf), (inf, inf), (inf, -inf), (-inf, -inf), (3e38, 3e38),
             (-3e38, -3.1e38), (1e-45, 1.0), (1.0, 1e-45)]
    y = np.array([c[0] for c in cases], dtype=np.float32)
    x = np.array([c[1] for c in cases], dtype=np.float32)
    got = _atan2(y, x)
    want = np.arctan2(y.astype(np.float64), x.astype(np.float64)).astype(np.float32)
    assert np.array_equal(np.signbit(got), np.signbit(want)), (got, want)
    ulp = np.spacing(np.abs(want)).astype(np.float64)
    assert (np.abs(got.astype(np.float64) - np.arctan2(y.astype(np.float64), x.astype(np.float64))) <= 2 * ulp).all(), (got, want)
    assert np.isnan(_atan2(np.array([np.nan, 1.0]), np.array([1.0, np.nan]))).all()


FRAMES = {
    "default": lambda w, h: frame(w, h),
    "sun-in-view": lambda w, h: frame(w, h, sun=SUN_IN_VIEW, cos_radius=np.cos(np.radians(4.0))),
    "sun-below-horizon": lambda w, h: frame(w, h, sun=(0.3, 0.2, 0.9)),
    "thick-haze": lambda w, h: frame(w, h, sun=(0.5, -0.6, 0.4), g=0.6, MieSigmaS=0.02, MieSigmaA=0.01, RayleighSigmaSScale=0.05),
}


@pytest.mark.parametrize("name", list(FRAMES))
@pytest.mark.parametrize("size", [(256, 128), (64, 32), (255, 127)])
def test_host_build_of_device_header_equals_oracle(name, size):
    fc = FRAMES[name](96, 54)
    lut = oracle_lut(fc, *size)
    dev = np.zeros_like(lut)
    sky_util.host_device().hsky_view_lut(C.byref(fc), size[0], size[1], ptr(dev))
    assert np.array_equal(dev, lut), np.argwhere(dev != lut)[:5]
    want, _ = oracle_background(fc, lut, *size)
    got = np.zeros_like(want)
    sky_util.host_device().hsky_background(C.byref(fc), ptr(lut), size[0], size[1], ptr(got))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("name", list(FRAMES))
def test_oracle_lut_matches_independent_estimate(name):
    fc = FRAMES[name](16, 16)
    w, h = 64, 32
    got = sky_util.decode_r11g11b10(oracle_lut(fc, w, h)).reshape(h, w, 3)
    want = indep_sky.sky_view_lut(fc, w, h)
    tol = sky_util.r11g11b10_step(want) + 1e-4 * want
    bad = np.abs(got - want) > tol
    assert not bad.any(), (np.argwhere(bad)[:5], got[bad][:5], want[bad][:5])
    assert (got > 0).any()


def test_lut_lookup_is_a_bilinear_wrap_tap():
    """Le_Sky against a float64 bilinear tap at texel-centre mapping with wrap on both axes, over directions that cross the seam at
    phi = 0 and the poles (where v wraps between the top and bottom rows)."""
    fc = frame(16, 16)
    w, h = 64, 32
    lut = oracle_lut(fc, w, h)
    tex = sky_util.decode_r11g11b10(lut).reshape(h, w, 3)
    rng = np.random.default_rng(5)
    d = rng.normal(size=(20000, 3))
    d[:200, 2] = rng.uniform(-1e-4, 1e-4, 200)          # phi near 0 / 2 pi
    d[200:400, :2] *= 1e-3                              # near the poles
    d[400:600, 1] = rng.uniform(-1e-3, 1e-3, 200)       # the horizon
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    out = np.zeros_like(d)
    oracle().sky_le_sky(ptr(lut), w, h, ptr(d), len(d), ptr(out))
    d64 = d.astype(np.float64)
    theta = np.arccos(np.clip(d64[:, 1], -1, 1))
    phi = np.mod(np.arctan2(-d64[:, 2], d64[:, 0]), 2 * np.pi)
    u = phi / (2 * np.pi)
    v = 0.5 + np.sign(theta - np.pi / 2 + 1e-300) * np.sqrt(np.abs(0.5 * theta - np.pi / 4) / np.pi)
    tx, ty = u * w - 0.5, v * h - 0.5
    x0, y0 = np.floor(tx), np.floor(ty)
    fx, fy = (tx - x0)[:, None], (ty - y0)[:, None]
    x0, y0 = x0.astype(int) % w, y0.astype(int) % h
    x1, y1 = (x0 + 1) % w, (y0 + 1) % h
    want = (tex[y0, x0] * (1 - fx) * (1 - fy) + tex[y0, x1] * fx * (1 - fy) + tex[y1, x0] * (1 - fx) * fy + tex[y1, x1] * fx * fy)
    # the reference's ArcCos polynomial is good to about 7e-5 rad; the tap's slope turns that into a small relative error
    assert np.allclose(out, want, rtol=2e-2, atol=1e-3 * want.max()), np.abs(out - want).max()


def test_sun_disk_pixels_match_a_float64_cone_test():
    w, h = 160, 90
    cos_r = np.float32(np.cos(np.radians(6.0)))
    fc = frame(w, h, sun=SUN_IN_VIEW, cos_radius=cos_r, CurrCameraJitter=(0.25, -0.375))
    _, sun = oracle_background(fc, oracle_lut(fc, 64, 32), 64, 32)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    uv_x = (xs + 0.5 + fc.CurrCameraJitter[0]) / w
    uv_y = (ys + 0.5 + fc.CurrCameraJitter[1]) / h
    dv = np.stack([(2 * uv_x - 1) * fc.AspectRatio * fc.TanHalfFOV, (1 - 2 * uv_y) * fc.TanHalfFOV, np.ones_like(uv_x)], axis=-1)
    view = np.array(fc.CurrView[:], dtype=np.float64).reshape(3, 4)[:, :3]
    wc = dv @ view
    wc /= np.linalg.norm(wc, axis=-1, keepdims=True)
    sun_dir = np.array(fc.SunDir[:], dtype=np.float64)
    cone = -(wc @ sun_dir) - np.float64(fc.SunCosAngularRadius)
    # the disk's lower edge: the ray lowered by the angular radius must not meet the planet from 0.1 km above the ground
    wy = wc[..., 1] * fc.SunCosAngularRadius + np.sqrt(1 - wc[..., 1] ** 2) * fc.SunSinAngularRadius
    R, y0 = np.float64(fc.PlanetRadius), np.float64(fc.PlanetRadius) + 0.1
    disc = (wy * y0) ** 2 - y0 * y0 + R * R
    edge_above = (disc < 0) | (-wy * y0 - np.sqrt(np.maximum(disc, 0)) < 0)
    want = (cone >= 0) & edge_above
    sure = np.abs(cone) > 1e-5
    assert want.sum() > 100
    assert np.array_equal(sun.reshape(h, w)[sure], want[sure])


def test_frame_constants_carry_the_reference_atmosphere():
    from zetaray_b200.camera import look_at_frame_constants
    fc = look_at_frame_constants(64, 32)
    assert (fc.PlanetRadius, fc.AtmosphereAltitude, fc.SunIlluminance) == (6360.0, 100.0, 20.0)
    assert np.isclose(fc.g, 0.8) and np.isclose(np.linalg.norm(fc.SunDir[:]), 1, atol=1e-6)
    assert np.allclose(np.array(fc.RayleighSigmaSColor[:]) * fc.RayleighSigmaSScale, [5.802e-3, 13.558e-3, 33.1e-3], rtol=1e-6)
    assert np.allclose(np.array(fc.OzoneSigmaAColor[:]) * fc.OzoneSigmaAScale, [0.65e-3, 1.881e-3, 0.085e-3], rtol=1e-6)
    assert np.isclose(fc.SunCosAngularRadius, np.cos(np.radians(0.263)), atol=1e-7)
    assert np.isclose(fc.SunCosAngularRadius ** 2 + fc.SunSinAngularRadius ** 2, 1, atol=1e-6)
    assert (fc.MieSigmaS, fc.MieSigmaA) == (pytest.approx(3.996e-3), pytest.approx(4.4e-3))
