"""ORACLE -- test infrastructure, not product code.

Independent float64 radiometric truth for scenes made of axis-aligned rectangles (tests/scene_util.py TRUTH_SCENES): what a
pixel's direct lighting IS, computed without the oracle library (oracle/liborc.so), tests/orc.py or any device source. Its only
inputs are the scene description (rectangles + make_material keyword arguments), the pinned packers of zetaray_b200/scene.py (to
quantise Le exactly as the emissive record and the material store it), the frame-constant camera values and oracle/indep_bsdf.py
for f. It shares no code with the estimators it checks: no light sampling, no pdfs, no MIS, no RIS, no ray offsets.

Semantics taken from the reference (cited, not copied):
  * an emitter triangle emits towards n_L = cross(v1 - v0, v2 - v0); a double-sided one towards both sides
    (Common/LightSource.hlsli:111-130). A surface point receives light from a one-sided emitter only where dot(n_L, -wi) > 0
    (DirectLighting/Emissive/ReSTIR_DI_Temporal.hlsl:79 for BSDF-sampled and :158 for light-sampled candidates).
  * a camera ray that hits an emissive surface shows its Le whichever side it sees (GBuffer/GBufferRT.hlsli:264-279 stores the
    emission without a facing test; ReSTIR_DI_Temporal.hlsl:288-292 writes it as the pixel's DirectLighting value).
  * DirectLighting output 0 at a non-emissive pixel is L_dir(x, wo) = sum over emitters of the integral of
    f(wo, wi) Le V cos' / r^2 dA, with f = BSDF::Unified's value, which has n.wi folded in (indep_bsdf.unified does the same).

Quadrature: each emitter rectangle is cut into G x G cells with a 4 x 4 Gauss-Legendre rule per cell. The value at G and 2G is
compared; the error estimate is their difference and G doubles (up to G_MAX) until that is <= 1e-4 of the pixel's total. Pixels
that do not converge -- the narrow highlights of a glossy floor close to a light's mirror image -- and every pixel that sees an
emitter partly occluded (penumbra, found by a visibility test on a dense grid of the emitter, partly_visible) are flagged, and
the tests leave them out.

Visibility is tested against every rectangle of the scene (the union of a rectangle's triangles is the rectangle, so a
ray-parallelogram test is the brute-force test against both of its triangles); camera rays use the same test."""
import numpy as np

import indep_bsdf

REL_TOL = 1e-4
G_MAX = 32
GL_X, GL_W = np.polynomial.legendre.leggauss(4)
GL_X = 0.5 * (GL_X + 1.0); GL_W = 0.5 * GL_W
DEFAULT_ETA_MAT, DEFAULT_ETA_COAT = 1.5, 1.6      # ShadingData defaults for an opaque material / coat (BSDF.hlsli)


class Rect:
    def __init__(self, d):
        from zetaray_b200 import scene as zscene
        self.name = d["name"]
        self.p0, self.eu, self.ev = (np.asarray(d[k], dtype=np.float64) for k in ("p0", "eu", "ev"))
        c = np.cross(self.eu, self.ev)
        self.area = np.linalg.norm(c)
        self.n = c / self.area
        m = dict(d["mat"])
        self.mat = m
        rgb = zscene.rgb8(m.get("emissive_factor", (0, 0, 0)))
        strength = np.float64(zscene.half_bits(m.get("emissive_strength", 1.0)).view(np.float16))
        self.le = np.array([(rgb >> s) & 0xff for s in (0, 8, 16)], dtype=np.float64) / 255.0 * strength
        self.emissive = bool(rgb)
        self.double_sided = bool(m.get("double_sided", False))

    def point(self, s, t):
        return self.p0 + s[..., None] * self.eu + t[..., None] * self.ev


def rects(desc):
    return [Rect(d) for d in desc]


def intersect(rs, o, d, tmin, tmax):
    """Closest hit of rays o + t d, t in (tmin, tmax), against every rectangle: (t, rect index or -1, (s, t) on the rectangle)."""
    o = np.asarray(o, dtype=np.float64); d = np.asarray(d, dtype=np.float64)
    best = np.full(o.shape[:-1], np.inf); idx = np.full(o.shape[:-1], -1); st = np.zeros(o.shape[:-1] + (2,))
    for k, r in enumerate(rs):
        # Moller-Trumbore against the parallelogram p0 + s eu + t ev
        p = np.cross(d, r.ev)
        det = p @ r.eu
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = 1.0 / det
            tv = o - r.p0
            s = np.sum(tv * p, axis=-1) * inv
            q = np.cross(tv, r.eu)
            t = np.sum(d * q, axis=-1) * inv
            th = (q @ r.ev) * inv
        hit = (det != 0) & (s >= 0) & (s <= 1) & (t >= 0) & (t <= 1) & (th > tmin) & (th < tmax) & (th < best)
        best = np.where(hit, th, best); idx = np.where(hit, k, idx)
        st = np.where(hit[..., None], np.stack([s, t], axis=-1), st)
    return best, idx, st


def occluded(rs, x, y, skip):
    """Segment x -> y (exclusive of both ends) crosses a rectangle other than rs[skip]."""
    d = y - x
    blocked = np.zeros(np.broadcast_shapes(x.shape, y.shape)[:-1], dtype=bool)
    for k, r in enumerate(rs):
        if k == skip:
            continue
        t, i, _ = intersect([r], x, d, 1e-7, 1.0 - 1e-7)
        blocked |= i >= 0
    return blocked


def camera_rays(w, h, fc):
    """Pinhole rays through pixel centres (no jitter): origins, unit directions, and the world-space direction that advances one
    unit of view-space depth (o + z * dview is the point at view depth z)."""
    x, y = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    u = (x.reshape(-1) + 0.5) / w; v = (y.reshape(-1) + 0.5) / h
    ndc_x, ndc_y = 2.0 * u - 1.0, 1.0 - 2.0 * v
    t = float(fc.TanHalfFOV); a = float(fc.AspectRatio)
    R = np.array([[fc.CurrViewInv[4 * r + c] for c in range(3)] for r in range(3)], dtype=np.float64)
    dcam = np.stack([ndc_x * a * t, ndc_y * t, np.ones_like(ndc_x)], axis=-1)
    dview = dcam @ R.T
    d = dview / np.linalg.norm(dview, axis=-1, keepdims=True)
    o = np.broadcast_to(np.array([fc.CameraPos[0], fc.CameraPos[1], fc.CameraPos[2]], dtype=np.float64), d.shape)
    return o, d, dview


class Primary:
    def __init__(self, rs, w, h, fc):
        self.o, self.d, self.dview = camera_rays(w, h, fc)
        self.t, self.rect, st = intersect(rs, self.o, self.d, 0.0, np.inf)
        self.valid = self.rect >= 0
        self.pos = self.o + np.where(self.valid, self.t, 0.0)[:, None] * self.d
        # distance of the hit from the nearest rectangle edge, in world units: hits within rounding of an edge are ambiguous
        ext = np.array([[np.linalg.norm(r.eu), np.linalg.norm(r.ev)] for r in rs])
        e = np.minimum(st, 1.0 - st) * ext[np.maximum(self.rect, 0)]
        self.edge_dist = np.where(self.valid, e.min(axis=-1), np.inf)
        self.emissive = self.valid & np.array([r.emissive for r in rs])[np.maximum(self.rect, 0)]


def _surface_params(rs, rect_idx):
    """indep_bsdf.unified's material arguments per pixel, from the description (opaque classes only)."""
    P = len(rect_idx)
    out = dict(metallic=np.zeros(P, bool), roughness=np.zeros(P), base=np.zeros((P, 3)), coat_w=np.zeros(P),
               coat_col=np.zeros((P, 3)), coat_rough=np.zeros(P), coat_ior=np.full(P, DEFAULT_ETA_COAT))
    for k, r in enumerate(rs):
        m = rect_idx == k
        if not m.any():
            continue
        mat = r.mat
        assert not mat.get("transmission", 0) and not mat.get("thin_walled", False)
        out["metallic"][m] = mat.get("metallic", 0.0) >= 0.9
        out["roughness"][m] = mat.get("roughness", 0.3)
        out["base"][m] = mat.get("base_color", (1, 1, 1))[:3]
        cw = mat.get("coat_weight", 0.0)
        out["coat_w"][m] = cw
        if cw:
            out["coat_col"][m] = mat.get("coat_color", (0.8, 0.8, 0.8))
            out["coat_rough"][m] = mat.get("coat_roughness", 0.0)
            out["coat_ior"][m] = mat.get("coat_ior", 1.6)
    return out


def _emitter_integral(rs, k, x, nrm, wo, sp, rho, G):
    """sum over cells of the emitter rs[k] of f Le V cos' / r^2 dA at the points x (P, 3), G x G cells, 4 x 4 nodes per cell."""
    r = rs[k]
    c = (np.arange(G, dtype=np.float64)[:, None] + GL_X[None, :]).reshape(-1) / G
    wq = np.tile(GL_W, G) / G
    S, T = np.meshgrid(c, c, indexing="ij")
    W = np.outer(wq, wq).reshape(-1) * r.area
    y = r.point(S.reshape(-1), T.reshape(-1))                      # (K, 3)
    P, K = len(x), len(y)
    out = np.zeros((P, 3))
    chunk = max(1, 400000 // K)
    for a in range(0, P, chunk):
        xs = x[a:a + chunk]
        dv = y[None, :, :] - xs[:, None, :]
        d2 = np.sum(dv * dv, axis=-1)
        wi = dv / np.sqrt(d2)[..., None]
        cos_l = -(wi @ r.n)
        cos_l = np.abs(cos_l) if r.double_sided else np.maximum(cos_l, 0.0)
        g = cos_l / d2 * W[None, :]
        live = g > 0
        live &= ~occluded(rs, np.broadcast_to(xs[:, None, :], dv.shape), np.broadcast_to(y[None, :, :], dv.shape), k)
        pi, qi = np.nonzero(live)
        if pi.size == 0:
            continue
        pix = pi + a
        f, _ = indep_bsdf.unified(rho, nrm[pix], wo[pix], wi[pi, qi], sp["metallic"][pix], sp["roughness"][pix], sp["base"][pix],
                                  np.ones(pi.size), np.full(pi.size, DEFAULT_ETA_MAT), np.zeros(pi.size, bool), np.zeros(pi.size),
                                  np.zeros(pi.size), sp["coat_w"][pix], sp["coat_col"][pix], sp["coat_rough"][pix], sp["coat_ior"][pix])
        contrib = f * g[pi, qi][:, None]
        for ch in range(3):
            out[a:a + len(xs), ch] += np.bincount(pi, weights=contrib[:, ch], minlength=len(xs))
    return out * r.le[None, :]


def direct(rs, prim, rho, pixels=None):
    """L_dir at the primary hits (non-emissive pixels; `pixels` restricts to a subset). Returns (L (P, 3), err (P, 3),
    converged (P,)): err is |L(G) - L(G/2)| of the last refinement, converged means err <= REL_TOL x max(L) per pixel."""
    P = len(prim.t)
    sel = np.nonzero(prim.valid & ~prim.emissive)[0] if pixels is None else np.asarray(pixels)
    x = prim.pos[sel]
    ridx = prim.rect[sel]
    nrm = np.array([rs[k].n for k in ridx])
    wo = -prim.d[sel]
    nrm = np.where((np.sum(nrm * wo, axis=-1) < 0)[:, None], -nrm, nrm)        # double-sided surfaces face the viewer
    sp = _surface_params(rs, ridx)
    L = np.zeros((P, 3)); E = np.full((P, 3), np.inf); conv = np.zeros(P, bool)
    em = [k for k, r in enumerate(rs) if r.emissive]
    coarse = {k: _emitter_integral(rs, k, x, nrm, wo, sp, rho, 2) for k in em}
    fine = {k: _emitter_integral(rs, k, x, nrm, wo, sp, rho, 4) for k in em}
    err = {k: np.abs(fine[k] - coarse[k]) for k in em}
    scale = np.maximum(np.max(sum(fine.values()), axis=1), 1e-30)
    for k in em:
        G = 4
        # refine each emitter with headroom (a quarter of the tolerance) against the pixel's total
        todo = np.nonzero(np.max(err[k], axis=1) > 0.25 * REL_TOL * scale)[0]
        while todo.size and G < G_MAX:
            G *= 2
            cur = _emitter_integral(rs, k, x[todo], nrm[todo], wo[todo], {key: v[todo] for key, v in sp.items()}, rho, G)
            err[k][todo] = np.abs(cur - fine[k][todo]); fine[k][todo] = cur
            todo = todo[np.max(err[k][todo], axis=1) > 0.25 * REL_TOL * scale[todo]]
    Lsel = sum(fine.values()); Esel = sum(err.values())
    L[sel] = Lsel; E[sel] = Esel
    ok = np.max(Esel, axis=1) <= REL_TOL * np.maximum(np.max(Lsel, axis=1), 1e-30)
    for k in em:
        ok[ok] &= ~partly_visible(rs, k, x[ok])
    conv[sel] = ok
    return L, E, conv


def partly_visible(rs, k, x, n_edge=128, n_inner=16):
    """Points x that see part, but not all, of the emitter rs[k]. Matching n and 2n Gauss-Legendre values do not prove a
    penumbra pixel converged: a sliver of the emitter seen past an occluder's edge can lie between the nodes of both rules. The
    shadow of a convex occluder on the emitter's plane is convex, so testing the emitter's boundary at 1 / 128 of its edges
    (corners included) and its interior at 1 / 16 finds every mixed case but slivers of <= 1e-4 of the emitter's area."""
    r = rs[k]
    e = np.linspace(0.0, 1.0, n_edge + 1)
    z, o = np.zeros_like(e), np.ones_like(e)
    g = np.linspace(0.0, 1.0, n_inner + 1)
    S, T = np.meshgrid(g, g, indexing="ij")
    s = np.concatenate([e, e, z, o, S.reshape(-1)]); t = np.concatenate([z, o, e, e, T.reshape(-1)])
    y = r.point(s, t)
    out = np.zeros(len(x), dtype=bool)
    chunk = max(1, 400000 // len(y))
    for a in range(0, len(x), chunk):
        xs = x[a:a + chunk]
        xb = np.broadcast_to(xs[:, None, :], (len(xs), len(y), 3)); yb = np.broadcast_to(y[None], xb.shape)
        # points behind a one-sided emitter, or in its plane, receive nothing from it whatever the occluders
        facing = np.abs((xs - r.p0) @ r.n) > 1e-12
        if not r.double_sided:
            facing &= (xs - r.p0) @ r.n > 0
        vis = ~occluded(rs, xb, yb, k)
        out[a:a + chunk] = facing & vis.any(axis=1) & ~vis.all(axis=1)
    return out


def emissive_vertices_f64(em):
    """The three vertices of each packed emissive record, decoded in float64 (octahedral UNORM16 edge directions, half lengths)."""
    def oct_decode(u16):
        u = u16.astype(np.float64) / 65535.0 * 2.0 - 1.0
        n = np.stack([u[:, 0], u[:, 1], 1.0 - np.abs(u[:, 0]) - np.abs(u[:, 1])], axis=-1)
        t = np.clip(-n[:, 2], 0.0, None)
        n[:, 0] -= np.where(n[:, 0] >= 0, t, -t); n[:, 1] -= np.where(n[:, 1] >= 0, t, -t)
        return n / np.linalg.norm(n, axis=-1, keepdims=True)
    v0 = em["Vtx0"].astype(np.float64)
    lens = em["EdgeLengths"].view(np.float16).astype(np.float64)
    v1 = v0 + oct_decode(em["V0V1"]) * lens[:, :1]
    v2 = v0 + oct_decode(em["V0V2"]) * lens[:, 1:]
    return v0, v1, v2
