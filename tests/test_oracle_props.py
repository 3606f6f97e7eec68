"""CPU-only checks of the oracle itself (the reference has no tests for this code, so these are the sanity anchors):
codecs against their stated precision, BSDF sampling self-consistency and energy bounds, ReSTIR PT vs plain PT mean."""
import ctypes as C
import os
import numpy as np
import pytest

from tests.orc import SurfaceDesc, ptr


def surf(roughness=0.5, metallic=0, base=(0.8, 0.8, 0.8), spec_tr=0, coat=0.0, coat_rough=0.1, wo=(0.3, 0.2, 0.93), subsurface=0.0):
    s = SurfaceDesc()
    s.normal[:] = (0, 0, 1)
    w = np.array(wo, dtype=np.float64); w /= np.linalg.norm(w)
    s.wo[:] = tuple(w)
    s.metallic, s.roughness = metallic, roughness
    s.baseColor[:] = base
    s.eta_curr, s.eta_next, s.specTr = 1.0, 1.5, spec_tr
    s.trDepth, s.subsurface, s.coat_weight = 0.0, subsurface, coat
    s.coat_color[:] = (0.9, 0.9, 0.9)
    s.coat_roughness, s.coat_ior = coat_rough, 1.6
    return s


@pytest.fixture(scope="module")
def o(oracle):
    from tests import scene_util
    lut = scene_util.rho_lut()       # process-wide instance: the oracle keeps a bare pointer
    oracle.orc_set_rho_lut(ptr(lut))
    return oracle


def test_octahedral_roundtrip_1e6(o):
    # Tests/TestMath.cpp:485-508: encode/decode of unit vectors round-trips to 1e-6 ... with 16-bit storage the
    # reference's bound for oct32 is looser; check the 2 x UNORM16 precision (angle error < 1e-4 rad)
    rng = np.random.default_rng(1)
    v = rng.normal(size=(20000, 3)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    out = np.zeros_like(v)
    o.orc_oct32_roundtrip(ptr(v), len(v), ptr(out))
    assert np.abs(v.astype(np.float64) - out).max() < 1e-4
    assert np.abs(np.linalg.norm(out, axis=1) - 1).max() < 1e-6


def test_storage_codecs(o):
    out = (C.c_float * 3)()
    for rgb in [(0, 0, 0), (1, 0.5, 0.25), (20, 15.5, 12.3), (65000, 1e-3, 3.3)]:
        p = o.orc_pack_r11g11b10(rgb[0], rgb[1], rgb[2])
        o.orc_unpack_r11g11b10(p, out)
        for a, b, tol in zip(rgb, out, (1 / 64, 1 / 64, 1 / 32)):
            assert b <= a + 1e-12 and (a == 0 or (a - b) / a <= tol + 1e-6)     # truncation, 6/6/5 mantissa bits
    out2 = (C.c_float * 2)()
    for xy in [(0, 0), (0.5, -0.5), (1, -1), (3, -3), (1e-3, -2e-5)]:
        o.orc_unpack_snorm16x2(o.orc_pack_snorm16x2(xy[0], xy[1]), out2)
        for a, b in zip(xy, out2):
            assert abs(np.clip(a, -1, 1) - b) <= 0.5 / 32767 + 1e-9


SURFACES = {
    "rough_diffuse": surf(roughness=1.0),
    "glossy": surf(roughness=0.2),
    "metal": surf(roughness=0.3, metallic=1, base=(0.95, 0.64, 0.54)),
    "coated": surf(roughness=0.6, coat=1.0),
    "glass": surf(roughness=0.15, spec_tr=1, base=(1, 1, 1)),
    "thin": surf(roughness=0.5, subsurface=0.5),
}


@pytest.mark.parametrize("name", list(SURFACES))
def test_sampler_eval_matches_sample(o, name):
    # EvalBSDFSampler must reproduce the joint (lobe, wi) pdf and f / pdf of SampleBSDF for the same 9 uniforms
    # (BSDFSampling.hlsli:548-563) -- the property the random-replay shift relies on
    s = SURFACES[name]
    a = (C.c_float * 12)(); b = (C.c_float * 8)()
    n_ok = 0
    for seed in range(1, 400):
        o.orc_bsdf_sample(C.byref(s), seed, a)
        if a[4] <= 0:
            continue
        wi = (C.c_float * 3)(a[0], a[1], a[2])
        o.orc_bsdf_eval_sampler(C.byref(s), wi, int(a[3]), seed, b)
        assert np.float32(a[11]).tobytes() == np.float32(b[7]).tobytes()      # both consumed exactly 9 uniforms
        # the half vector is re-derived from wi on the eval side: sharp lobes amplify that rounding
        rtol = 5e-3 if name == "glass" else 2e-4
        assert abs(b[0] - a[4]) <= rtol * max(1.0, abs(a[4])), (name, seed, b[0], a[4])
        for k in range(3):
            assert abs(b[1 + k] - a[5 + k]) <= (2e-2 if name == "glass" else 2e-3) * max(1.0, abs(a[5 + k]))
        n_ok += 1
    assert n_ok > 100


@pytest.mark.parametrize("name", ["rough_diffuse", "glossy", "metal", "coated"])
def test_white_furnace_bound(o, name):
    # E[f cos / pdf] is the directional albedo: <= 1 (+ MC noise) for a white base
    s = surf(roughness=SURFACES[name].roughness, metallic=SURFACES[name].metallic, base=(1, 1, 1), coat=SURFACES[name].coat_weight)
    a = (C.c_float * 12)()
    acc = np.zeros(3)
    n = 4000
    for seed in range(1, n + 1):
        o.orc_bsdf_sample(C.byref(s), seed * 7919, a)
        acc += [a[5], a[6], a[7]]
    albedo = acc / n
    assert (albedo < 1.05).all() and (albedo > 0.3).all(), albedo


def test_restir_pt_mean_matches_plain_path_tracing():
    # unbiasedness sanity: ReSTIR PT (temporal + spatial) and plain PT agree on the mean image radiance
    from tests import scene_util, rpt_util
    w, h = 128, 72

    def run(temporal, spatial, nframes=28):
        R = rpt_util.OracleRenderer(scene_util.cornell(), w, h)
        R.params.temporal_resample = temporal
        R.params.num_spatial_passes = spatial
        seq = rpt_util.FrameSequence(w, h)
        acc = np.zeros(3); n = 0
        for fr in range(nframes):
            fc = seq.next(); R.gbuffer(fc); R.rpt(fc)
            if fr >= 4:
                acc += R.final[:, :3].astype(np.float64).mean(axis=0); n += 1
        return acc / n
    pt = run(0, 0)
    rs = run(1, 1)
    assert np.all(np.abs(rs - pt) / pt < 0.12), (pt, rs)


def test_plain_path_tracer_is_the_ground_truth_for_both_restir_integrators():
    """SURVEY 8f-4: the reference's plain path tracer (MIS at every bounce, no reuse) is the in-repo ground truth. ReSTIR PT and
    ReSTIR GI with all their reuse switched on converge to the same image mean. The comparison uses the median of per-frame
    means: ReSTIR GI's light-only NEE after the first bounce (MIS_ALL_BOUNCES 0) has a 1 / t^2 tail, so single fireflies
    move a plain mean by factors."""
    from tests import scene_util, rpt_util
    w, h = 128, 72

    def run(mode, nframes=36):
        R = rpt_util.OracleRenderer(scene_util.cornell(), w, h)
        R.gi_params.stochastic_multi_bounce = 0
        seq = rpt_util.FrameSequence(w, h)
        means = []
        for fr in range(nframes):
            fc = seq.next(); R.gbuffer(fc)
            if mode == "pt":
                R.pt(fc); img = R.gi_final
            elif mode == "gi":
                R.rgi(fc); img = R.gi_final
            else:
                R.rpt(fc); img = R.final
            if fr >= 6:
                means.append(img[:, :3].astype(np.float64).mean(axis=0))
        return np.median(np.array(means), axis=0)
    pt, gi, rs = run("pt"), run("gi"), run("rpt")
    assert np.all(np.abs(rs - pt) / pt < 0.12), (pt, rs)
    assert np.all(np.abs(gi - pt) / pt < 0.2), (pt, gi)


def test_oracle_outputs_are_frozen():
    """The lighting oracle has no external pin; tests/golden/oracle_hashes.json freezes its outputs (tools/make_oracle_hashes.py)
    so that a change to the oracle is a deliberate, visible act."""
    import importlib.util
    import json
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("make_oracle_hashes", os.path.join(root, "tools", "make_oracle_hashes.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    want = json.load(open(os.path.join(root, "tests", "golden", "oracle_hashes.json")))
    for name, kw in m.CASES.items():
        got = m.run(**kw)
        assert got == want[name], "oracle output changed for case %s: %s" % (name, [k for k in got if got[k] != want[name].get(k)])


def test_presampled_sets_follow_the_alias_distribution():
    """PresampleEmissives draws lights in proportion to their power: over many sets the light indices of the oracle's presampled
    records match the alias table's probabilities."""
    import numpy as np
    from tests import scene_util
    osc = scene_util.OracleScene(scene_util.cornell())
    osc.set_presampling(64, 512)
    osc.presample(7)
    idx = osc.sample_sets.reshape(-1, 10)[:64 * 512, 6]
    p = osc.power / osc.power.sum()
    freq = np.bincount(idx, minlength=len(p)) / idx.size
    assert np.abs(freq - p).max() < 0.01, (freq, p)
