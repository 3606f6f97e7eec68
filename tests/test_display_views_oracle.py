"""CPU: the oracle's Display debug views, pick-mask rasteriser and picked-instance outline (oracle/orc_display_views.cpp) against
independent numpy restatements of Display.hlsl:53-170, a float64 point-in-triangle test and Sobel.hlsl:27-105."""
import ctypes as C

import numpy as np
import pytest

from tests import orc
from tests.orc import ptr
from zetaray_b200 import _lib

FLT_MAX = np.float32(3.402823466e38)
OUTLINE = (0.913098693, 0.332451582, 0.048171822)


@pytest.fixture(scope="module")
def o():
    lib = orc.load()
    lib.orc_gbuffer_pick.restype = C.c_uint32
    lib.orc_pack_r11g11b10.restype = C.c_uint32
    lib.orc_pack_r11g11b10.argtypes = [C.c_float] * 3
    return lib


def srgb8(c):
    c = np.clip(np.asarray(c, dtype=np.float64), 0.0, 1.0)
    v = np.where(c <= 0.0031308, 12.92 * c, 1.055 * np.power(c, 1.0 / 2.4) - 0.055)
    return np.floor(np.clip(v, 0.0, 1.0) * 255.0 + 0.5).astype(np.int64)


def ufloat(v, mbits):
    e, m = v >> mbits, v & ((1 << mbits) - 1)
    return np.where(e == 0, m / 2.0 ** mbits * 2.0 ** -14, (1 + m / 2.0 ** mbits) * 2.0 ** (e.astype(np.float64) - 15))


def oct_decode(e):
    u = np.stack([(e & 0xffff) / 65535.0, (e >> 16) / 65535.0], -1) * 2 - 1
    n = np.stack([u[:, 0], u[:, 1], 1 - np.abs(u[:, 0]) - np.abs(u[:, 1])], -1)
    t = np.clip(-n[:, 2], 0, 1)
    n[:, 0] += np.where(n[:, 0] >= 0, -t, t)
    n[:, 1] += np.where(n[:, 1] >= 0, -t, t)
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def views_numpy(core, me, coat, view, th, near):
    """Display.hlsl:53-170 in float64: RGBA bytes per pixel"""
    n = len(core)
    w = core[:, 3]
    z = core[:, 0].view(np.float32).astype(np.float64)
    rough = ((w >> 8) & 0xff) / 255.0
    base = np.stack([(core[:, 2] >> s) & 0xff for s in (0, 8, 16)], -1) / 255.0
    tr, em, coated, metal = w & 1, (w >> 1) & 1, (w >> 5) & 1, (w >> 7) & 1
    cpy = coat[:, 0] >> 16
    d = np.zeros((n, 3))
    if view == 1:
        d = base
    elif view == 2:
        d = oct_decode(core[:, 1]) * 0.5 + 0.5
    elif view == 3:
        d = np.stack([metal, rough, np.zeros(n)], -1)
    elif view == 4:
        d = np.repeat(((cpy >> 8) & 0xff)[:, None] / 255.0, 3, 1) * coated[:, None]
    elif view == 5:
        cc = (coat[:, 0] & 0xffff) | ((cpy & 0xff) << 16)
        d = np.stack([(cc >> s) & 0xff for s in (0, 8, 16)], -1) / 255.0 * coated[:, None]
    elif view == 6:
        d = (rough >= th)[:, None] * np.array([0.26, 0.014, 0.021])
    elif view == 7:
        e = me[:, 1]
        emc = np.stack([ufloat(e & 0x7ff, 6), ufloat((e >> 11) & 0x7ff, 6), ufloat(e >> 22, 5)], -1)
        d = np.where(em[:, None] == 1, emc, base * 0.005)
    elif view == 8:
        d = np.stack([tr, 1 - tr, np.zeros(n)], -1)
    elif view == 9:
        d = np.repeat((near / z)[:, None], 3, 1)
    rgba = np.concatenate([srgb8(d), np.full((n, 1), 255)], 1)
    rgba[z == np.float64(FLT_MAX)] = 0
    return rgba


def gbuffer_records(o, n, seed):
    """synthetic records: every combination of the six flag bits, coat on and off, background pixels"""
    rng = np.random.default_rng(seed)
    core = np.zeros((n, 4), dtype=np.uint32)
    me = np.zeros((n, 2), dtype=np.uint32)
    coat = np.zeros((n, 2), dtype=np.uint32)
    bits = np.array([1, 2, 8, 16, 32, 128], dtype=np.uint32)
    combo = np.arange(n) % 64
    flags = np.zeros(n, dtype=np.uint32)
    for k, b in enumerate(bits):
        flags |= np.where((combo >> k) & 1, b, 0).astype(np.uint32)
    core[:, 0] = rng.uniform(0.05, 50.0, n).astype(np.float32).view(np.uint32)
    core[:, 1] = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    core[:, 2] = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    core[:, 3] = flags | (rng.integers(0, 256, n).astype(np.uint32) << 8) | (rng.integers(0, 256, n).astype(np.uint32) << 16)
    coat[:, 0] = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    coat[:, 1] = rng.integers(0, 2 ** 16, n).astype(np.uint32)
    for i in range(n):
        me[i, 1] = o.orc_pack_r11g11b10(*rng.uniform(0, 40, 3))
    bg = rng.random(n) < 0.1
    core[bg] = [FLT_MAX.view(np.uint32), 0, 0, 4]
    return core, me, coat


@pytest.mark.parametrize("view", range(1, 10))
def test_views_match_numpy(o, view):
    W, H = 32, 16
    core, me, coat = gbuffer_records(o, W * H, view)
    for th in (0.0, 0.5, 1.0):
        out = np.zeros(W * H, dtype=np.uint32)
        o.orc_display_view(ptr(core), ptr(me), ptr(coat), W, 0, H, view, C.c_float(th), C.c_float(0.2), ptr(out))
        got = out.view(np.uint8).reshape(-1, 4).astype(np.int64)
        want = views_numpy(core, me, coat, view, th, np.float32(0.2))
        assert np.abs(got - want).max() <= 1, (view, th)
        assert (got[core[:, 0] == FLT_MAX.view(np.uint32)] == 0).all()


def frame(W, H, jitter=(0.0, 0.0), near=0.5, tan=0.6):
    fc = _lib.FrameConstants()
    for r in range(3):
        fc.CurrView[r * 4 + r] = 1.0
    fc.RenderWidth, fc.RenderHeight, fc.DisplayWidth, fc.DisplayHeight = W, H, W, H
    fc.AspectRatio, fc.TanHalfFOV, fc.CameraNear = W / H, tan, near
    fc.CurrCameraJitter[0], fc.CurrCameraJitter[1] = jitter
    return fc


def coverage_f64(tris, W, H, fc):
    """float64: per pixel, the number of clipped, projected triangles whose interior holds the centre, and the distance of the
    centre to the nearest edge (pixels closer than 1e-5 px are not compared)"""
    near, tan, asp = float(fc.CameraNear), float(np.float32(fc.TanHalfFOV)), float(np.float32(fc.AspectRatio))
    jx, jy = fc.CurrCameraJitter[0], fc.CurrCameraJitter[1]
    ys, xs = np.mgrid[0:H, 0:W]
    P = np.stack([xs.ravel() + 0.5, ys.ravel() + 0.5], -1)
    count = np.zeros(W * H, dtype=np.int64)
    dmin = np.full(W * H, np.inf)
    for t in tris.reshape(-1, 3, 3).astype(np.float64):
        poly = []
        for e in range(3):
            a, b = t[e], t[(e + 1) % 3]
            if a[2] >= near:
                poly.append(a)
            if (a[2] >= near) != (b[2] >= near):
                s = (near - a[2]) / (b[2] - a[2])
                poly.append(a + s * (b - a))
        if len(poly) < 3:
            continue
        q = np.array([[(p[0] / p[2] / tan / asp * 0.5 + 0.5) * W - jx, (-p[1] / p[2] / tan * 0.5 + 0.5) * H - jy] for p in poly])
        area = sum(q[i, 0] * q[(i + 1) % len(q), 1] - q[(i + 1) % len(q), 0] * q[i, 1] for i in range(len(q)))
        if area == 0:
            continue
        sgn = np.sign(area)
        inside = np.ones(len(P), dtype=bool)
        for i in range(len(q)):
            a, b = q[i], q[(i + 1) % len(q)]
            d = b - a
            L = np.hypot(*d)
            e = sgn * (d[0] * (P[:, 1] - a[1]) - d[1] * (P[:, 0] - a[0])) / L
            inside &= e > 0
            # distance to the edge segment
            tt = np.clip(((P - a) @ d) / (L * L), 0, 1)
            dmin = np.minimum(dmin, np.hypot(*(P - (a + tt[:, None] * d)).T))
        count += inside
    return count, dmin


@pytest.mark.parametrize("seed", range(4))
def test_rasteriser_matches_float64(o, seed):
    rng = np.random.default_rng(seed)
    W, H = 40, 24
    fc = frame(W, H, jitter=tuple(rng.uniform(-0.5, 0.5, 2)))
    n = 60
    z = rng.uniform(-1.0, 5.0, (n, 3))
    z[: n // 6] = rng.uniform(-3.0, 0.4, (n // 6, 3))            # wholly behind the near plane
    xy = rng.uniform(-1.2, 1.2, (n, 3, 2)) * np.maximum(np.abs(z), 0.5)[..., None]
    tris = np.concatenate([xy, z[..., None]], -1).astype(np.float32)
    assert ((tris[..., 2] >= 0.5).any(1) & (tris[..., 2] < 0.5).any(1)).sum() > 10        # crossing the near plane
    got = np.zeros(W * H, dtype=np.uint32)
    o.orc_raster_world_tris(ptr(tris), n, C.byref(fc), 0, H, 1, 0, ptr(got))
    want, dmin = coverage_f64(tris, W, H, fc)
    ok = dmin >= 1e-5
    assert ok.mean() > 0.9
    assert (got[ok] == want[ok]).all(), np.flatnonzero(ok & (got != want))
    # a row range rasterises those rows only
    part = np.zeros(W * H, dtype=np.uint32)
    o.orc_raster_world_tris(ptr(tris), n, C.byref(fc), 5, 13, 1, 0, ptr(part))
    rows = np.arange(W * H) // W
    assert (part[(rows >= 5) & (rows < 13)] == got[(rows >= 5) & (rows < 13)]).all() and (part[(rows < 5) | (rows >= 13)] == 0).all()


def grid_tris(xs, ys, flip):
    out = []
    for j in range(len(ys) - 1):
        for i in range(len(xs) - 1):
            a, b, c, d = (xs[i], ys[j]), (xs[i + 1], ys[j]), (xs[i + 1], ys[j + 1]), (xs[i], ys[j + 1])
            out += [a, b, c, a, c, d] if (i + j + flip) % 2 else [a, b, d, b, c, d]
    return np.array(out, dtype=np.float32).reshape(-1, 6)


@pytest.mark.parametrize("flip", [0, 1])
def test_top_left_rule_covers_a_tiling_once(o, flip):
    W, H = 36, 24
    # vertices on pixel centres: every edge family (vertical, horizontal, both diagonals) runs through centres
    xs = 0.5 + 3.0 * np.arange(-1, 14)
    ys = 0.5 + 3.0 * np.arange(-1, 10)
    tris = grid_tris(xs, ys, flip)
    tris[::2] = tris[::2].reshape(-1, 3, 2)[:, ::-1].reshape(-1, 6)        # both windings
    cnt = np.zeros(W * H, dtype=np.uint32)
    o.orc_raster_pixel_tris(ptr(tris), len(tris), W, H, ptr(cnt))
    assert (cnt == 1).all(), np.unique(cnt, return_counts=True)
    # a jittered mesh through the camera: shared vertices project once, so the tiling still covers each pixel once
    rng = np.random.default_rng(flip)
    fc = frame(W, H, jitter=(0.25, -0.375))
    gx, gy = np.linspace(-2.0, 2.0, 13), np.linspace(-1.4, 1.4, 9)
    V = np.stack(np.meshgrid(gx, gy), -1) + rng.uniform(-0.1, 0.1, (9, 13, 2))
    Z = rng.uniform(1.0, 1.3, (9, 13))
    P = np.concatenate([V, Z[..., None]], -1).astype(np.float32)
    tw = []
    for j in range(8):
        for i in range(12):
            a, b, c, d = P[j, i], P[j, i + 1], P[j + 1, i + 1], P[j + 1, i]
            tw += [a, b, c, a, c, d] if (i + j + flip) % 2 else [a, b, d, b, c, d]
    tw = np.array(tw, dtype=np.float32)
    cnt = np.zeros(W * H, dtype=np.uint32)
    o.orc_raster_world_tris(ptr(tw), len(tw) // 3, C.byref(fc), 0, H, 1, 0, ptr(cnt))
    assert (cnt == 1).all(), np.unique(cnt, return_counts=True)


def outline_numpy(mask, W, H, y0, y1, img):
    out = img.copy().reshape(H, W)
    m = mask.reshape(H, W).astype(np.int64)
    pad = np.zeros((H + 2, W + 2), dtype=np.int64)
    pad[1:-1, 1:-1] = m
    colour = np.uint32(sum(int(v) << (8 * i) for i, v in enumerate(srgb8(OUTLINE))) | 0xff000000)
    hit = np.zeros((H, W), dtype=bool)
    for k in range(32):
        b = (pad >> k) & 1
        t = lambda dy, dx: b[1 + dy:H + 1 + dy, 1 + dx:W + 1 + dx].astype(np.float64)   # noqa: E731
        nb = sum(t(dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)) > 0
        gx = -t(-1, -1) - 2 * t(0, -1) - t(1, -1) + t(-1, 1) + 2 * t(0, 1) + t(1, 1)
        gy = t(-1, -1) + 2 * t(-1, 0) + t(-1, 1) - t(1, -1) - 2 * t(1, 0) - t(1, 1)
        hit |= nb & (np.sqrt(gx * gx + gy * gy) * (0.2126 + 0.7152 + 0.0722) > 0)
    hit[:y0] = hit[y1:] = False
    out[hit] = colour
    return out.ravel()


@pytest.mark.parametrize("seed", range(3))
def test_outline_matches_numpy(o, seed):
    rng = np.random.default_rng(seed)
    W, H = 29, 17
    mask = np.zeros(W * H, dtype=np.uint32)
    for k in rng.choice(32, 5, replace=False):
        blob = rng.random(W * H) < rng.uniform(0.05, 0.6)
        mask |= (blob.astype(np.uint32) << np.uint32(k))
    mask[:W] |= np.uint32(1)                # a bit set along the frame's edge rows
    img = rng.integers(0, 2 ** 32, W * H, dtype=np.uint64).astype(np.uint32)
    for y0, y1 in ((0, H), (3, 9), (0, 1), (H - 1, H)):
        got = img.copy()
        o.orc_outline(ptr(mask), W, H, y0, y1, ptr(got))
        assert (got == outline_numpy(mask, W, H, y0, y1, img)).all(), (y0, y1)
    full = np.full(W * H, 0xffffffff, dtype=np.uint32)        # every bit everywhere: only the frame's border is an outline
    got = img.copy()
    o.orc_outline(ptr(full), W, H, 0, H, ptr(got))
    border = np.zeros((H, W), dtype=bool)
    border[0], border[-1], border[:, 0], border[:, -1] = True, True, True, True
    assert ((got != img) == border.ravel()).all()
