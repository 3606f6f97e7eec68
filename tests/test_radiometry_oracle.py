"""The oracle's ReSTIR DI against an independent float64 radiometric truth (oracle/indep_radiometry.py), CPU only.

Parity tests hold the device to the oracle bit for bit; they cannot see a transcription error the two share. These tests ask what
a pixel's direct lighting should be: the truth integrates f Le V cos' / r^2 over every emitter by quadrature, with its own ray
tests and the independent BSDF evaluator, and each test compares tile means of R independent replicas (fresh temporal state,
frame numbers 1000 apart, so the random numbers differ) with it in every RGB channel. The threshold is Student's t with R - 1
degrees of freedom, Bonferroni-corrected over all comparisons of the file, so a correct oracle fails the file with probability
<= 1 % whatever the seeds. The tiles that can detect a 5 % luminance bias must cover at least 60 % of the lit tiles, and together
they must resolve 1 % in each channel. tests/test_radiometry_gpu.py repeats the comparison on the device with enough frames for a
1 % bound per tile."""
import numpy as np
import pytest

from tests import radiometry_util as ru, rpt_util
from zetaray_b200.camera import FrameSequence

W, H = 64, 40
REPLICAS, FRAMES, WARMUP, PRESAMPLED_EXTRA = 32, 20, 4, 12
SCENES = ["truth_a", "truth_b"]
TILE_BOUND, REGION_BOUND = 0.05, 0.01       # relative bias the test detects: per asserted tile, and over all of them
# every tile x channel and every region channel of the 12 DI cases is one comparison; a correct oracle fails one with
# probability <= ru.ALPHA
THRESHOLD = ru.threshold(REPLICAS, 12 * 3 * (ru.num_tiles(W, H) + 1))


def _replicas(T, di_params=None, presample=None, replicas=REPLICAS, frames=FRAMES):
    out = []
    for r in range(replicas):
        R = rpt_util.OracleRenderer(T.flat, T.w, T.h)
        if presample:
            R.osc.set_presampling(*presample)
        for k, v in (di_params or {}).items():
            setattr(R.di_params, k, v)
        seq = FrameSequence(T.w, T.h, jitter=False, first_frame=1 + 1000 * r)
        acc = np.zeros((T.w * T.h, 3))
        for f in range(frames):
            fc = seq.next(); R.gbuffer(fc); R.rdi(fc)
            if f >= WARMUP:
                acc += R.di_final[:, :3]
        out.append(acc / (frames - WARMUP))
    return np.array(out)


@pytest.mark.parametrize("name", SCENES)
def test_truth_scene_emissive_records_match_the_mesh(name):
    """The light sampler draws from the packed emissive records, the hit tests see the mesh under its quantised instance
    transform (the identity quaternion stores as 1.5e-5 per component, a rotation of ~3e-5 rad). Decoded in float64, the
    records' vertices and areas agree with that mesh to 1e-4 of the edge length, and the mesh with the truth's rectangles to 1e-4
    of the distance from the origin -- far below any bias these tests resolve."""
    from zetaray_b200 import scene as zscene
    T = ru.truth(name, W, H)
    v0, v1, v2 = ru.ir.emissive_vertices_f64(T.flat.emissives)
    pos = T.flat.vertices["pos"].astype(np.float64)
    tris = []
    for inst, ntri in zip(T.flat.instances, T.flat.instance_num_tris):
        if inst["BaseEmissiveTriOffset"] == 0xffffffff:
            continue
        idx = T.flat.indices[inst["BaseIdxOffset"]:inst["BaseIdxOffset"] + 3 * ntri].reshape(-1, 3) + inst["BaseVtxOffset"]
        q = inst["Rotation"].astype(np.float64) / 65535.0 * 2.0 - 1.0
        world = zscene.quat_rotate_np(q / np.linalg.norm(q), pos[idx] * inst["Scale"].view(np.float16).astype(np.float64))
        tris.append(world + inst["Translation"].astype(np.float64))
        assert (np.abs(world - pos[idx]) <= 1e-4 * np.maximum(np.linalg.norm(pos[idx], axis=-1, keepdims=True), 1)).all()
    mesh = np.concatenate(tris)
    size = np.linalg.norm(mesh[:, 1] - mesh[:, 0], axis=1)[:, None]
    for k, v in enumerate((v0, v1, v2)):
        assert (np.abs(v - mesh[:, k]) / size).max() <= 1e-4
    area = lambda a, b, c: 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1)
    assert (np.abs(area(v0, v1, v2) / area(*mesh.transpose(1, 0, 2)) - 1)).max() <= 1e-4
    # the scene covers what it is meant to: a >= 256-triangle emitter and per-triangle powers >= 100x apart (truth_b), a
    # one-sided and a double-sided emitter (truth_a)
    le = np.array([r.le for r in T.rs if r.emissive])
    ds = [r.double_sided for r in T.rs if r.emissive]
    counts = np.diff(np.append(T.flat.instances["BaseEmissiveTriOffset"][T.flat.instances["BaseEmissiveTriOffset"] != 0xffffffff],
                               len(T.flat.emissives)))
    power = ru.luminance(np.repeat(le, counts, axis=0)) * area(v0, v1, v2)
    if name == "truth_b":
        assert counts.max() >= 256 and power.max() / power.min() >= 100
    else:
        assert True in ds and False in ds
    assert zscene.EMISSIVE_TRI.itemsize == 48


@pytest.mark.parametrize("name", SCENES)
def test_truth_primary_hits_match_the_oracle_gbuffer(name):
    """Before any radiance is compared, the truth's camera rays must hit what the oracle's G-buffer saw: the same pixels are
    valid and emissive, and the position decoded from depth + camera lies within 1e-4 of the ray length of the truth's hit's
    plane. (The quantised instance rotation moves the mesh by ~3e-5 of its distance from the origin; along a grazing ray the
    distance to the hit point grows as 1 / |n.d|, so that direction is bounded by its median.)"""
    T = ru.truth(name, W, H)
    R = rpt_util.OracleRenderer(T.flat, W, H)
    core, depth, _, _, _ = R.gbuffer(FrameSequence(W, H, jitter=False).next())
    flags = core[:, 3] & 0xff
    valid, emissive = ((flags >> 2) & 1) == 0, ((flags >> 1) & 1) == 1
    assert (valid == T.prim.valid).all() and (emissive == T.prim.emissive).all()
    v = T.prim.valid
    pos = T.prim.o[v] + depth[v].astype(np.float64)[:, None] * T.prim.dview[v]
    n = np.array([T.rs[k].n for k in T.prim.rect[v]])
    plane = np.abs(np.sum((pos - T.prim.pos[v]) * n, axis=1)) / T.prim.t[v]
    along = np.linalg.norm(pos - T.prim.pos[v], axis=1) / T.prim.t[v]
    assert plane.max() <= 1e-4 and np.median(along) <= 1e-4, (plane.max(), np.median(along), along.max())


@pytest.mark.parametrize("name", SCENES)
def test_truth_quadrature_is_converged_where_used(name):
    """The truth's own error (n vs 2n nodes per axis) is <= 1e-4 of the pixel's value wherever a test uses it; the pixels left
    out (penumbra, the narrow highlight of the glossy floor) are a small part of the lit image. In truth_a the wall above the
    one-sided light sees only its back: it is lit by the double-sided light alone."""
    T = ru.truth(name, W, H)
    lit = T.prim.valid & ~T.prim.emissive
    u = T.usable
    assert (np.max(T.err[u], axis=1) <= 1e-4 * np.max(T.L[u], axis=1)).all()
    assert u.sum() >= 0.9 * lit.sum(), (u.sum(), lit.sum())
    if name == "truth_a":
        wall = [k for k, r in enumerate(T.rs) if r.name == "wall"][0]
        above = u & (T.prim.rect == wall) & (T.prim.pos[:, 1] > 2.05)
        assert above.sum() >= 20
        side = [r for r in T.rs if r.name == "light_side"][0]
        rs_side = [r for r in T.rs if r.name != "light_down"]
        T2 = ru.ir.direct(rs_side, ru.ir.Primary(rs_side, W, H, ru.look_at_frame_constants(W, H)),
                          ru.indep_bsdf.RhoTable(ru.scene_util.rho_lut()), pixels=np.nonzero(above)[0])[0]
        assert side.double_sided and np.allclose(T2[above], T.L[above], rtol=1e-9, atol=0)


@pytest.mark.parametrize("name", SCENES)
def test_emissive_pixels_show_le(name):
    """A camera ray that hits an emitter shows its Le, from either side, exactly up to the R11G11B10 storage of the G-buffer's
    emission (truncation to 6 / 6 / 5 mantissa bits) -- no statistics involved."""
    T = ru.truth(name, W, H)
    img = _replicas(T, replicas=1, frames=WARMUP + 1)[0]
    em = T.prim.emissive
    assert em.sum() >= 10
    rel = (T.le[em] - img[em]) / T.le[em]
    assert (rel >= 0).all() and (rel[:, :2] <= 2.0 ** -6).all() and (rel[:, 2] <= 2.0 ** -5).all(), rel.max(axis=0)


DI_MODES = {"no_reuse": dict(temporal_resample=0, spatial_resample=0), "temporal": dict(temporal_resample=1, spatial_resample=0),
            "temporal_spatial": {}}


@pytest.mark.parametrize("sampling", ["alias", "presampled"])
@pytest.mark.parametrize("mode", list(DI_MODES))
@pytest.mark.parametrize("name", SCENES)
def test_restir_di_matches_radiometric_truth(name, mode, sampling):
    T = ru.truth(name, W, H)
    # a presampled set is shared by an 8 x 8 pixel group, i.e. by a whole tile in one frame: those tiles need more frames
    presampled = sampling == "presampled"
    reps = _replicas(T, DI_MODES[mode], presample=(16, 64) if presampled else None, frames=FRAMES + PRESAMPLED_EXTRA * presampled)
    s = ru.tile_stats(reps, T, THRESHOLD)
    region = ru.asserted_region(s, TILE_BOUND)
    ru.check(s, region, ru.region_stats(s, region, THRESHOLD), THRESHOLD, REGION_BOUND, "%s %s %s" % (name, mode, sampling))
