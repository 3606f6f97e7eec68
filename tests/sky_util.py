"""The sky's test libraries and helpers: the oracle's restatement (oracle/sky/libsky.so), the host build of the device header
(tests/hostsim/libhostsim_sky.so), frame constants with a chosen sun or atmosphere, and the R11G11B10F decoding."""
import ctypes as C
import os
import subprocess

import numpy as np

from tests import hostsim
from zetaray_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SKY_DIR = os.path.join(ROOT, "oracle", "sky")
SKY_HEADER = os.path.join(SKY_DIR, "sky_api.h")
HSKY_SRC = os.path.join(hostsim.HERE, "hostsim_sky.cpp")
HSKY_HEADER = os.path.join(hostsim.HERE, "hostsim_sky_api.h")
HSKY_SO = os.path.join(hostsim.HERE, "libhostsim_sky.so")
LUT_W, LUT_H = 256, 128        # the renderer's LUT (DefaultRendererImpl.h:165-166)

_libs = {}


def _protos(header, macro, prefix):
    with open(header) as f:
        return _lib.prototypes(f.read(), macro, prefix)


def build_hostsim(force=False):
    hostsim._build(HSKY_SRC, HSKY_SO, force)
    return HSKY_SO


def oracle():
    """oracle/sky/libsky.so (built by build(); compiled here when missing) with the types of sky_api.h."""
    if "sky" not in _libs:
        so = os.path.join(SKY_DIR, "libsky.so")
        if not os.path.exists(so):
            subprocess.check_call(["bash", os.path.join(SKY_DIR, "build.sh")])
        _libs["sky"] = _lib.declare(C.CDLL(so), _protos(SKY_HEADER, "SKY_API", "sky_"))
    return _libs["sky"]


def host_device():
    """The device header compiled for the host, with the types of hostsim_sky_api.h."""
    if "hsky" not in _libs:
        _libs["hsky"] = _lib.declare(C.CDLL(build_hostsim()), _protos(HSKY_HEADER, "HSKY_API", "hsky_"))
    return _libs["hsky"]


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def frame(w, h, sun=None, cos_radius=None, **atmosphere):
    """Frame constants of the default camera with the reference's atmosphere; sun: the direction the light travels (SunDir, the
    disk is at -sun); cos_radius: the disk's angular radius as its cosine; atmosphere: any other field (PlanetRadius, g, ...)."""
    from zetaray_b200.camera import look_at_frame_constants
    fc = look_at_frame_constants(w, h)
    if sun is not None:
        s = np.asarray(sun, dtype=np.float64)
        s = (s / np.linalg.norm(s)).astype(np.float32)
        fc.SunDir[0], fc.SunDir[1], fc.SunDir[2] = (float(v) for v in s)
    if cos_radius is not None:
        fc.SunCosAngularRadius = float(np.float32(cos_radius))
        fc.SunSinAngularRadius = float(np.sqrt(np.float32(1) - np.float32(cos_radius) ** 2))
    for k, v in atmosphere.items():
        if isinstance(v, (tuple, list)):
            arr = getattr(fc, k)
            for i, c in enumerate(v):
                arr[i] = c
        else:
            setattr(fc, k, v)
    return fc


def oracle_lut(fc, w=LUT_W, h=LUT_H):
    out = np.zeros(w * h, dtype=np.uint32)
    oracle().sky_view_lut(C.byref(fc), w, h, ptr(out))
    return out


def oracle_background(fc, lut, w=LUT_W, h=LUT_H):
    """(rgb per pixel, sun-disk mask) of Le_SkyWithSunDisk over the whole frame."""
    n = fc.RenderWidth * fc.RenderHeight
    rgb, sun = np.zeros((n, 3), dtype=np.float32), np.zeros(n, dtype=np.uint8)
    oracle().sky_background(C.byref(fc), ptr(lut), w, h, ptr(rgb), ptr(sun))
    return rgb, sun.astype(bool)


def _ufloat(v, mbits):
    e, m = (v >> mbits).astype(np.int64), (v & ((1 << mbits) - 1)).astype(np.float64)
    return np.where(e == 0, m / (1 << mbits) * 2.0 ** -14, (1 + m / (1 << mbits)) * 2.0 ** (e - 15))


def decode_r11g11b10(p):
    p = np.asarray(p, dtype=np.uint32)
    return np.stack([_ufloat(p & 0x7ff, 6), _ufloat((p >> 11) & 0x7ff, 6), _ufloat(p >> 22, 5)], axis=-1)


def r11g11b10_step(v):
    """The spacing of the R11G11B10F values around v (per channel: 6, 6 and 5 mantissa bits)."""
    v = np.maximum(np.asarray(v, dtype=np.float64), 2.0 ** -14)
    e = np.floor(np.log2(v))
    return np.stack([2.0 ** (e[..., 0] - 6), 2.0 ** (e[..., 1] - 6), 2.0 ** (e[..., 2] - 5)], axis=-1)
