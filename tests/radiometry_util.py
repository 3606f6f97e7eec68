"""Shared pieces of the radiometric-truth tests (tests/test_radiometry_oracle.py, tests/test_radiometry_gpu.py): the truth of a
TRUTH_SCENES scene at one image size, and the tile statistics that compare R independent replicas with it."""
import functools
import os
import sys
import numpy as np
from scipy import stats

from tests import scene_util
from zetaray_b200.camera import look_at_frame_constants

sys.path.insert(0, os.path.join(scene_util.ROOT, "oracle"))
import indep_bsdf  # noqa: E402
import indep_radiometry as ir  # noqa: E402

TILE = 8
ALPHA = 0.01            # family-wise false-alarm rate of one test file: the chance that a correct estimator fails any comparison
LUM = np.array([0.2126, 0.7152, 0.0722])


class Truth:
    def __init__(self, name, w, h):
        self.flat, self.desc = scene_util.truth_scene(name)
        self.w, self.h = w, h
        self.rs = ir.rects(self.desc)
        self.prim = ir.Primary(self.rs, w, h, look_at_frame_constants(w, h))
        self.L, self.err, self.converged = ir.direct(self.rs, self.prim, indep_bsdf.RhoTable(scene_util.rho_lut()))
        le = np.array([r.le for r in self.rs])
        self.le = np.where(self.prim.emissive[:, None], le[np.maximum(self.prim.rect, 0)], 0.0)
        # pixels whose direct-lighting truth a test may use: a lit surface (not an emitter, not the sky), well inside its rectangle,
        # with a converged quadrature
        self.usable = self.prim.valid & ~self.prim.emissive & self.converged & (self.prim.edge_dist > 1e-3)


@functools.lru_cache(maxsize=None)
def truth(name, w, h):
    return Truth(name, w, h)


def luminance(c):
    return c @ LUM


def num_tiles(w, h, tile=TILE):
    return ((w + tile - 1) // tile) * ((h + tile - 1) // tile)


def threshold(replicas, comparisons, alpha=ALPHA):
    """The |z| a comparison may reach. z uses a standard error estimated from R replica means, so a correct estimator's z follows
    Student's t with R - 1 degrees of freedom; over `comparisons` such tests (Bonferroni) the chance that any exceeds this
    threshold is <= alpha. Never below 5."""
    return max(5.0, float(stats.t.isf(alpha / (2.0 * comparisons), replicas - 1)))


def _z(mean, truth, sigma):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(sigma > 0, (mean - truth) / sigma, np.where(mean == truth, 0.0, np.inf))


def tile_stats(replicas, T, thr, tile=TILE):
    """replicas: (R, P, 3) per-replica pixel means of DirectLighting output 0. Each tile averages its usable pixels, per RGB
    channel. The replicas are independent, so a tile's standard error is the spread of its R replica means over sqrt(R),
    combined with the truth's own quadrature error (pixels inside one replica are correlated by reuse and per-group random
    numbers, so they are never treated as independent samples). Returns per-tile arrays: z (tiles, 3) for every channel, and
    `detect`, the relative luminance bias a |z| <= thr test can detect."""
    R = replicas.shape[0]
    ty, tx = np.divmod(np.arange(T.w * T.h), T.w)
    tid = (ty // tile) * ((T.w + tile - 1) // tile) + tx // tile
    m = T.usable
    cnt = np.bincount(tid[m], minlength=num_tiles(T.w, T.h, tile))
    keep = cnt > 0

    def tile_mean(v):       # (usable,) -> (tiles,)
        return (np.bincount(tid[m], weights=v, minlength=len(cnt)) / np.maximum(cnt, 1))[keep]
    per = np.stack([np.stack([tile_mean(replicas[r, m, c]) for c in range(3)], axis=-1) for r in range(R)])   # (R, tiles, 3)
    tr = np.stack([tile_mean(T.L[m, c]) for c in range(3)], axis=-1)
    tr_err = np.stack([tile_mean(T.err[m, c]) for c in range(3)], axis=-1)
    s = dict(count=cnt[keep], replica_means=per, truth=tr, truth_err=tr_err)
    s.update(_compare(per, tr, tr_err, thr))
    return s


def _compare(per, tr, tr_err, thr):
    R = per.shape[0]
    mean = per.mean(axis=0)
    sigma = np.sqrt(per.var(axis=0, ddof=1) / R + tr_err ** 2)
    lum = per @ LUM
    sig_l = np.sqrt(lum.var(axis=0, ddof=1) / R + (tr_err @ LUM) ** 2)
    with np.errstate(divide="ignore", invalid="ignore"):
        detect = thr * sig_l / (tr @ LUM)
        detect_rgb = thr * sigma / tr
    return dict(mean=mean, sigma=sigma, z=_z(mean, tr, sigma), detect=detect, detect_rgb=detect_rgb)


def region_stats(s, region, thr):
    """The same comparison over the union of the tiles in `region`, weighted by their pixel counts (replicas stay the unit)."""
    wgt = s["count"][region] / s["count"][region].sum()
    per = np.einsum("rtc,t->rc", s["replica_means"][:, region], wgt)[:, None, :]
    tr = (wgt @ s["truth"][region])[None, :]
    tr_err = (wgt @ s["truth_err"][region])[None, :]
    g = _compare(per, tr, tr_err, thr)
    return dict(z=g["z"][0], detect=g["detect"][0], detect_rgb=g["detect_rgb"][0])


def asserted_region(s, bound):
    """Tiles that can detect a relative luminance bias of `bound`. Every tile is compared with the truth in every channel; these
    are the ones whose comparison is also a bound on their bias. A test asserts that they cover most of the lit image."""
    return (s["truth"] @ LUM > 0) & (s["detect"] <= bound)


def check(s, region, g, thr, region_bound, label):
    """The assertions both tiers make, and the line they print."""
    lit = s["truth"] @ LUM > 0
    assert region.any(), ("no tile resolves the bias bound", np.abs(s["z"]).max(), thr)
    print("%s: %d tiles (%d asserted), max |z| %.2f of %.2f, detectable luminance bias per asserted tile <= %.2f %% (median %.2f %%); "
          "region z (%.2f, %.2f, %.2f), detectable (%.3f, %.3f, %.3f) %%" % (
              label, len(lit), region.sum(), np.abs(s["z"]).max(), thr, 100 * s["detect"][region].max(),
              100 * np.median(s["detect"][region]), *g["z"], *(100 * g["detect_rgb"])))
    assert region.sum() >= 0.6 * lit.sum(), (region.sum(), lit.sum())
    assert (g["detect_rgb"] <= region_bound).all(), g["detect_rgb"]
    assert np.abs(s["z"]).max() <= thr, (np.abs(s["z"]).max(), thr)
    assert (np.abs(g["z"]) <= thr).all(), g["z"]
