"""ORACLE -- test infrastructure. An independent float64 estimate of the sky-view LUT, written from the single-scattering model of
Hillaire (2020, "A Scalable and Production Ready Sky and Atmosphere Rendering Technique") rather than from the reference shaders:

    L(x, v) = E_sun sum_i T(x, p_i) [sigma_s,R rho_R(p_i) P_R(mu) + sigma_s,M rho_M(p_i) P_M(mu)] T_sun(p_i) dt

over the view ray from a viewer 0.2 km above the ground to the top of the atmosphere or to the ground. Media: Rayleigh scattering
with density exp(-h / 8 km), Mie scattering and absorption with exp(-h / 1.2 km), ozone absorption with a tent 1 - |h - 25| / 15
(clamped at 0); P_R(mu) = 3 (1 + mu^2) / (16 pi), P_M the Schlick approximation of Henyey-Greenstein (Blasi et al. 1993) with
k = 1.55 g - 0.55 g^3. The quadrature is the one the product uses, so that a comparison isolates float32 and storage error: 32
segments of the view ray sampled at their midpoints, T(x, p_i) accumulated through the end of segment i, and T_sun by 8 midpoint
segments towards the sun up to the top of the atmosphere (the planet does not shadow them). Directions follow the LUT's mapping:
longitude phi = 2 pi x / W measured clockwise from +x about +y, latitude theta = pi/2 +- 2 pi (y / H - 1/2)^2 from +y."""
import numpy as np


def _atmosphere(fc):
    sr = np.array(fc.RayleighSigmaSColor[:], dtype=np.float64) * fc.RayleighSigmaSScale
    so = np.array(fc.OzoneSigmaAColor[:], dtype=np.float64) * fc.OzoneSigmaAScale
    return sr, float(fc.MieSigmaS), float(fc.MieSigmaS) + float(fc.MieSigmaA), so


def _densities(p, radius):
    h = np.linalg.norm(p, axis=-1) - radius
    return (np.exp(-np.maximum(h, 0) / 8.0), np.exp(-np.maximum(h, 0) / 1.2), np.maximum(0.0, 1 - np.abs(h - 25.0) / 15.0))


def _exit_distance(o, d, radius):
    """Distance along unit d from o (inside the sphere) to the sphere of `radius` about the planet's centre."""
    b = np.sum(o * d, axis=-1)
    return -b + np.sqrt(b * b - np.sum(o * o, axis=-1) + radius * radius)


def _ground_distance(o, d, radius):
    """Distance to the ground, or nan where the ray misses it or the hit lies behind."""
    b = np.sum(o * d, axis=-1)
    disc = b * b - np.sum(o * o, axis=-1) + radius * radius
    with np.errstate(invalid="ignore"):
        t = -b - np.sqrt(disc)
    return np.where((disc >= 0) & (t >= 0), t, np.nan)


def sky_view_lut(fc, w, h):
    """float64 radiance of every LUT texel before storage, shape (h, w, 3)."""
    R, top = float(fc.PlanetRadius), float(fc.PlanetRadius) + float(fc.AtmosphereAltitude)
    sr, ssm, stm, so = _atmosphere(fc)
    sun = -np.array(fc.SunDir[:], dtype=np.float64)          # towards the sun
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    phi = 2 * np.pi * xs / w
    v = ys / h
    theta = np.pi / 2 + np.sign(v - 0.5 + 1e-300) * 2 * np.pi * (v - 0.5) ** 2
    d = np.stack([np.sin(theta) * np.cos(phi), np.cos(theta), -np.sin(theta) * np.sin(phi)], axis=-1)
    o = np.broadcast_to(np.array([0.0, R + 0.2, 0.0]), d.shape)
    t_ground = _ground_distance(o, d, R)
    t = np.where(np.isnan(t_ground), _exit_distance(o, d, top), t_ground)
    dt = t / 32
    tau = np.zeros(d.shape)
    lr, lm = np.zeros(d.shape), np.zeros(d.shape)
    for i in range(32):
        p = o + ((i + 0.5) * dt)[..., None] * d
        rho_r, rho_m, rho_o = _densities(p, R)
        tau += (sr * rho_r[..., None] + stm * rho_m[..., None] + so * rho_o[..., None]) * dt[..., None]
        # the sun's light reaching p
        ts = _exit_distance(p, np.broadcast_to(sun, p.shape), top)
        ds = ts / 8
        tau_s = np.zeros(d.shape)
        for j in range(8):
            q = p + ((j + 0.5) * ds)[..., None] * sun
            qr, qm, qo = _densities(q, R)
            tau_s += sr * qr[..., None] + stm * qm[..., None] + so * qo[..., None]
        t_sun = np.where((ts <= 1e-5)[..., None], 1.0, np.exp(-tau_s * ds[..., None]))
        tr = np.exp(-tau) * t_sun
        lr += tr * rho_r[..., None]
        lm += tr * rho_m[..., None]
    mu = np.sum(d * sun, axis=-1)
    g = float(fc.g)
    k = 1.55 * g - 0.55 * g ** 3
    p_r = 3 * (1 + mu * mu) / (16 * np.pi)
    p_m = (1 - k * k) / (4 * np.pi * (1 - k * mu) ** 2)
    L = (lr * sr * p_r[..., None] + lm * ssm * p_m[..., None]) * dt[..., None]
    return np.maximum(L * float(fc.SunIlluminance), 0.0)
