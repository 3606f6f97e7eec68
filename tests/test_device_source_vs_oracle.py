"""CPU tier: the DEVICE source of the layered BSDF (zetaray_b200/csrc/zr_bsdf.cuh, compiled for the host by tests/hostsim with the
product's numeric contract: no contraction, explicit fmaf, zr_fpmath transcendentals) against the oracle's restatement
(oracle/orc_bsdf.h), bit for bit, over random surfaces of every material class: sampling (all lobes, incl. the no-diffuse sampler
used by ReSTIR GI's MIS), sampler evaluation, sampler pdfs and the unified evaluation. The GPU tier checks the same code through
whole kernels; this test catches a one-sided edit of either transcription where the driver runs its CPU suite, without a GPU."""
import ctypes as C

import numpy as np
import pytest

from tests import hostsim, orc
from tests.orc import SurfaceDesc, ptr


def random_surface(rng):
    s = SurfaceDesc()
    n = rng.normal(size=3); n /= np.linalg.norm(n)
    wo = rng.normal(size=3); wo /= np.linalg.norm(wo)
    if rng.random() < 0.85 and np.dot(wo, n) < 0:
        wo = -wo                                         # mostly front-facing, some back-facing views
    s.normal[:] = tuple(n.astype(np.float32)); s.wo[:] = tuple(wo.astype(np.float32))
    kind = rng.integers(0, 6)
    s.metallic = int(kind == 1)
    s.roughness = float(np.float32(rng.choice([0.0, 0.02, 0.1, 0.3, 0.6, 1.0]) if rng.random() < 0.5 else rng.random()))
    s.baseColor[:] = tuple(rng.random(3).astype(np.float32))
    s.specTr = int(kind in (2, 3))
    inside = kind == 3 and rng.random() < 0.5
    ior = float(np.float32(1.0 + 1.4 * rng.random()))
    s.eta_curr, s.eta_next = (ior, 1.0) if inside else (1.0, ior)
    s.trDepth = float(np.float32(rng.random())) if kind == 3 else 0.0
    s.subsurface = float(np.float32(rng.random())) if kind == 4 else 0.0
    s.coat_weight = float(np.float32(rng.random())) if kind == 5 or rng.random() < 0.2 else 0.0
    s.coat_color[:] = tuple(rng.random(3).astype(np.float32))
    s.coat_roughness = float(np.float32(rng.choice([0.0, 0.05, 0.3]) if rng.random() < 0.5 else rng.random()))
    s.coat_ior = float(np.float32(1.1 + rng.random()))
    return s


def same(a, b, n):
    return np.frombuffer(a, dtype=np.uint32, count=n).tobytes() == np.frombuffer(b, dtype=np.uint32, count=n).tobytes()


def test_bsdf_device_source_is_bit_identical_to_the_oracle():
    from tests import scene_util
    hs = hostsim.load()
    o = orc.load()
    lut = scene_util.rho_lut()
    o.orc_set_rho_lut(ptr(lut)); hs.hostsim_set_rho_lut(ptr(lut))
    rng = np.random.default_rng(42)
    a = (C.c_float * 12)(); b = (C.c_float * 12)()
    lobes_seen = set()
    n_sampled = 0
    for it in range(6000):
        s = random_surface(rng)
        seed = int(rng.integers(1, 2**32 - 1))
        o.orc_bsdf_sample(C.byref(s), seed, a); hs.hostsim_bsdf_sample(C.byref(s), seed, b)
        assert same(a, b, 12), ("SampleBSDF", it, list(a), list(b))
        lobes_seen.add(int(a[3])); n_sampled += a[4] > 0
        wi = (C.c_float * 3)(a[0], a[1], a[2]) if a[4] > 0 and rng.random() < 0.7 else (C.c_float * 3)(*(lambda v: v / np.linalg.norm(v))(rng.normal(size=3)).astype(np.float32))
        lobe = int(a[3])
        o.orc_bsdf_eval_sampler(C.byref(s), wi, lobe, seed, a); hs.hostsim_bsdf_eval_sampler(C.byref(s), wi, lobe, seed, b)
        assert same(a, b, 8), ("EvalBSDFSampler", it, list(a)[:8], list(b)[:8])
        pa = o.orc_bsdf_sampler_pdf(C.byref(s), wi, seed); pb = hs.hostsim_bsdf_sampler_pdf(C.byref(s), wi, seed)
        assert np.float32(pa).tobytes() == np.float32(pb).tobytes(), ("BSDFSamplerPdf", it, pa, pb)
        o.orc_bsdf_unified(C.byref(s), wi, a); hs.hostsim_bsdf_unified(C.byref(s), wi, b)
        assert same(a, b, 3), ("Unified", it, list(a)[:3], list(b)[:3])
        o.orc_bsdf_sample_nodiffuse(C.byref(s), seed, a); hs.hostsim_bsdf_sample_nodiffuse(C.byref(s), seed, b)
        assert same(a, b, 12), ("SampleBSDF_NoDiffuse", it, list(a), list(b))
        pa = o.orc_bsdf_sampler_pdf_nodiffuse(C.byref(s), wi); pb = hs.hostsim_bsdf_sampler_pdf_nodiffuse(C.byref(s), wi)
        assert np.float32(pa).tobytes() == np.float32(pb).tobytes(), ("BSDFSamplerPdf_NoDiffuse", it, pa, pb)
    assert n_sampled > 4000 and len(lobes_seen) >= 4, (n_sampled, lobes_seen)


def test_storage_codecs_device_source_vs_oracle():
    """G-buffer / reservoir storage codecs of zr_common.cuh (host build) against the oracle's: octahedral normals, R11G11B10F
    emissive colour, SNORM16 motion vectors, halves."""
    hs = hostsim.load()
    o = orc.load()
    rng = np.random.default_rng(9)
    n = 20000
    v = rng.normal(size=(n, 3)); v /= np.linalg.norm(v, axis=1, keepdims=True)
    v = np.ascontiguousarray(v.astype(np.float32))
    a = np.zeros((n, 3), dtype=np.float32); b = np.zeros((n, 3), dtype=np.float32); enc = np.zeros(n, dtype=np.uint32)
    o.orc_oct32_roundtrip(ptr(v), n, ptr(a)); hs.hostsim_oct32_roundtrip(ptr(v), n, ptr(b), ptr(enc))
    assert a.tobytes() == b.tobytes()
    out_a = (C.c_float * 3)(); out_b = (C.c_float * 3)()
    cols = np.concatenate([rng.random((3000, 3)) * rng.choice([1e-3, 1.0, 50.0, 7e4], (3000, 1)), [[0, 0, 0], [65504, 1e-8, 1.0]]]).astype(np.float32)
    for c in cols:
        pa = o.orc_pack_r11g11b10(c[0], c[1], c[2]); pb = hs.hostsim_pack_r11g11b10(c[0], c[1], c[2])
        assert pa == pb, (c, hex(pa), hex(pb))
        o.orc_unpack_r11g11b10(pa, out_a); hs.hostsim_unpack_r11g11b10(pa, out_b)
        assert bytes(out_a) == bytes(out_b)
    mv = np.concatenate([rng.normal(size=(3000, 2)) * 0.3, [[0, 0], [1, -1], [2, -2], [1e-6, -1e-6]]]).astype(np.float32)
    for m in mv:
        pa = o.orc_pack_snorm16x2(m[0], m[1]); pb = hs.hostsim_pack_snorm16x2(m[0], m[1])
        assert pa == pb, (m, hex(pa), hex(pb))
        o.orc_unpack_snorm16x2(pa, out_a); hs.hostsim_unpack_snorm16x2(pa, out_b)
        assert bytes(out_a)[:8] == bytes(out_b)[:8]
    h = np.concatenate([rng.normal(size=4000) * rng.choice([1e-6, 1.0, 300.0, 1e5], 4000), [0.0, -0.0, 65504.0, 65520.0, 1e-8, np.inf]]).astype(np.float32)
    mine = np.array([hs.hostsim_pack_half2(x, -x) for x in h], dtype=np.uint32)
    with np.errstate(over="ignore"):
        want = h.astype(np.float16).view(np.uint16).astype(np.uint32) | ((-h).astype(np.float16).view(np.uint16).astype(np.uint32) << 16)
    assert np.array_equal(mine, want)


@pytest.mark.parametrize("which,detail,nq", [("cornell", None, 3000), ("atrium", 0.5, 1200), ("tunnel", 0.35, 600)])
def test_ray_query_material_and_light_sampling_device_source_vs_oracle(which, detail, nq):
    """zr_rt.cuh on a host-resident scene (the product's BVH from zr_bvh_build_host, the flat buffers as uploaded) against the
    oracle (brute-force ray queries): FindClosest + hit attributes, GetMaterialData (checked through a BSDF sample and a unified
    evaluation on the fetched surface), FindClosestEmissive, both shadow-segment rules, light sampling through the alias table --
    at secondary-path vertices of scenes with tens of thousands of triangles, hundreds of instances and all material classes."""
    from tests import scene_util
    from tests.test_bvh_host import world_tris, build
    from tests.test_bvh_quality import ray_sets
    from zetaray_b200 import procedural
    hs = hostsim.load()
    if which == "cornell":
        flat, cam = scene_util.glass_cornell(), (0.0, 1.2, -4.043)
    else:
        make, cam = procedural.SCENES[which]
        flat = make(detail)
    osc = scene_util.OracleScene(flat)
    o = osc.o
    lut = osc.lut
    hs.hostsim_set_rho_lut(ptr(lut))
    wt, tri_mesh, first = world_tris(flat)
    nodes, order, leaf, info = build(wt)
    keep = [np.ascontiguousarray(x) for x in (flat.vertices, flat.indices, flat.instances, flat.materials, flat.emissives, osc.alias)]
    hsc = hostsim.Scene(*[k.ctypes.data for k in keep], nodes.ctypes.data, leaf.ctypes.data, tri_mesh.ctypes.data, first.ctypes.data,
                    lut.ctypes.data, len(flat.instances), len(flat.emissives), len(wt))

    def closest(rays):
        out = np.zeros((len(rays), 4), dtype=np.float32)
        hs.hostsim_trace(ptr(nodes), ptr(leaf), ptr(tri_mesh), ptr(first), ptr(rays), len(rays), ptr(out), None, None, 8)
        return out
    prim, sec, sh = ray_sets(flat, wt, cam, closest)
    rng = np.random.default_rng(5)
    pick = rng.choice(len(sec), size=min(nq, len(sec)), replace=False)
    a = (C.c_uint32 * 24)(); b = (C.c_uint32 * 24)()
    hits = lights = 0
    for k in pick:
        # a path vertex: position on a surface, its geometric normal (= the direction ray_sets offset along), a sampled direction
        pos = sec[k, 0:3]; wi = sec[k, 4:7]
        nrm = wi / np.linalg.norm(wi)        # any normal with wi in its hemisphere serves the query (only the offset side matters)
        for transmissive in (0.0, 1.0):
            q = np.concatenate([pos, nrm, wi, [transmissive]]).astype(np.float32)
            seed = int(rng.integers(1, 2**32 - 1))
            o.orc_probe_path_vertex(osc.h, ptr(q), seed, a); hs.hostsim_probe_path_vertex(C.byref(hsc), ptr(q), seed, b)
            assert bytes(a) == bytes(b), (which, int(k), list(a), list(b))
            hits += a[0]
            o.orc_probe_emissive_and_visibility(osc.h, ptr(q), a); hs.hostsim_probe_emissive_and_visibility(C.byref(hsc), ptr(q), b)
            assert bytes(a)[:48] == bytes(b)[:48], (which, int(k), list(a)[:12], list(b)[:12])
            lights += a[4] != 0xffffffff and a[0] != 0
        # back-facing direction (transmission through the surface, or an early out when not transmissive)
        q = np.concatenate([pos, -nrm, wi, [1.0]]).astype(np.float32)
        o.orc_probe_path_vertex(osc.h, ptr(q), 7, a); hs.hostsim_probe_path_vertex(C.byref(hsc), ptr(q), 7, b)
        assert bytes(a) == bytes(b)
        seed = int(rng.integers(1, 2**32 - 1))
        p3 = pos.astype(np.float32)
        o.orc_probe_sample_light(osc.h, ptr(p3), 0, seed, 0, a); hs.hostsim_probe_sample_light(C.byref(hsc), ptr(p3), 0, seed, 0, b)
        assert bytes(a)[:64] == bytes(b)[:64], (which, int(k), list(a)[:16], list(b)[:16])
    # the degenerate query the path tracer issues after a failed BSDF sample on a transmissive surface: wi = 0 -> no hit, on both sides
    q = np.concatenate([sec[pick[0], 0:3], [0, 0, 1], [0, 0, 0], [1.0]]).astype(np.float32)
    o.orc_probe_emissive_and_visibility(osc.h, ptr(q), a); hs.hostsim_probe_emissive_and_visibility(C.byref(hsc), ptr(q), b)
    assert bytes(a)[:48] == bytes(b)[:48] and a[0] == 0
    assert hits > len(pick) // 4     # a good share of the queries hit something (the Cornell box is open at the front)
    assert lights > 0                # and some BSDF-direction queries end on a light


@pytest.mark.parametrize("which", ["glossy", "glass", "tunnel"])
def test_restir_pt_reservoir_record_codec(which):
    """RPT::Reservoir of zr_rpt.cuh (host build) against the oracle's on real reservoirs: every 64-byte record an oracle frame
    sequence produces (all reconnection cases k = 2 / k > 2, lobes, light types, empty reservoirs) is loaded and written back
    (full write with the M clamp, and the partial WriteReservoirData) by both; the bytes must agree."""
    from tests import scene_util, rpt_util
    hs = hostsim.load()
    w, h = 128, 72
    R = rpt_util.OracleRenderer(scene_util.SCENES[which](), w, h)
    cam = scene_util.CAMERAS.get(which)
    seq = rpt_util.FrameSequence(w, h, cam_path=(lambda f: cam) if cam else None)
    seen_k = set()
    for fr in range(3):
        fc = seq.next()
        R.gbuffer(fc); R.rpt(fc)
        res = np.ascontiguousarray(R.curr_reservoirs())
        n = len(res)
        seen_k |= set(np.unique(res["meta"] & 0xf).tolist())
        for m_max in (0, 4, 10):
            oa = np.zeros(n, dtype=rpt_util.RES); ob = np.zeros(n, dtype=rpt_util.RES)
            da = np.zeros(n, dtype=rpt_util.RES); db = np.zeros(n, dtype=rpt_util.RES)
            R.o.orc_probe_rpt_reservoir(ptr(res), n, m_max, ptr(oa), ptr(ob))
            hs.hostsim_probe_rpt_reservoir(ptr(res), n, m_max, ptr(da), ptr(db))
            assert oa.tobytes() == da.tobytes(), (which, fr, m_max, int((oa != da).sum()))
            assert ob.tobytes() == db.tobytes(), (which, fr, m_max)
    assert 0 in seen_k and 15 in seen_k


@pytest.mark.parametrize("which", ["glossy", "glass", "tunnel"])
def test_restir_pt_hybrid_shift(which):
    """The heart of ReSTIR PT on the CPU tier: random replay (k > 2) + reconnection shift of zr_rpt.cuh, run as a block of one
    thread on a host-resident scene, against the oracle's Replay_kGt2 / Shift2. Paths come from real reservoirs of an oracle
    frame sequence, destinations are first hits of camera rays through OTHER pixels (as spatial reuse does), so all three
    reconnection cases, replayed prefixes through glossy / transmissive lobes, failed replays and occluded reconnections occur."""
    from tests import scene_util, rpt_util
    from tests.test_bvh_host import world_tris, build
    from tests.test_procedural_scenes import _camera_rays
    hs = hostsim.load()
    w, h = 96, 54
    flat = scene_util.SCENES[which]()
    R = rpt_util.OracleRenderer(flat, w, h)
    osc = R.osc
    hs.hostsim_set_rho_lut(ptr(osc.lut))
    cam = scene_util.CAMERAS.get(which, (0.0, 1.2, -4.043))
    seq = rpt_util.FrameSequence(w, h, cam_path=lambda f: cam)
    for fr in range(3):
        fc = seq.next()
        R.gbuffer(fc); R.rpt(fc)
    res = np.ascontiguousarray(R.curr_reservoirs())
    wt, tri_mesh, first = world_tris(flat)
    nodes, order, leaf, info = build(wt)
    keep = [np.ascontiguousarray(x) for x in (flat.vertices, flat.indices, flat.instances, flat.materials, flat.emissives, osc.alias)]
    hsc = hostsim.Scene(*[k.ctypes.data for k in keep], nodes.ctypes.data, leaf.ctypes.data, tri_mesh.ctypes.data, first.ctypes.data,
                    osc.lut.ctypes.data, len(flat.instances), len(flat.emissives), len(wt))
    rays = _camera_rays(np.array(cam, dtype=np.float32), w, h)
    rng = np.random.default_rng(17)
    nonempty = np.nonzero((res["meta"] & 0xf) != 15)[0]
    a = (C.c_uint32 * 8)(); b = (C.c_uint32 * 8)()
    stats = dict(valid=0, kgt2=0, nonzero=0, replay_ok=0)
    alpha_min = float(np.float32(0.175) * np.float32(0.175))
    for it in range(2500):
        src = int(nonempty[rng.integers(0, len(nonempty))])
        sx, sy = src % w, src // w
        dx, dy = rng.integers(-6, 7, 2)
        px = int(np.clip(sx + dx, 0, w - 1)); py = int(np.clip(sy + dy, 0, h - 1))
        ray = np.concatenate([rays[py * w + px, 0:3], rays[py * w + px, 4:7]]).astype(np.float32)
        rec = res[src:src + 1]
        R.o.orc_probe_rpt_shift(osc.h, ptr(ray), ptr(rec), alpha_min, a)
        hs.hostsim_probe_rpt_shift(C.byref(hsc), ptr(ray), ptr(rec), alpha_min, b)
        assert bytes(a) == bytes(b), (which, it, src, (px, py), list(a), list(b))
        stats["valid"] += a[0]; stats["kgt2"] += a[6] > 2
        stats["nonzero"] += (a[1] | a[2] | a[3]) != 0
        stats["replay_ok"] += a[7] != 0
    print(which, stats)
    assert stats["valid"] > 500 and stats["nonzero"] > 150, stats
    assert stats["kgt2"] > 10 and stats["replay_ok"] > 3, stats          # replayed prefixes occur and some replays succeed


@pytest.mark.parametrize("which,dof", [("glossy", False), ("glass", True), ("atrium", False)])
def test_load_pixel_reconstruction(which, dof):
    """LoadPixel of zr_pixel.cuh -- depth -> world position (pinhole and thin lens, current and previous camera), normal / material
    decode, coat plane, the ShadingData every lighting kernel starts from (checked through a BSDF sample) -- against the oracle's,
    over whole G-buffers the oracle rendered."""
    from tests import scene_util, rpt_util
    hs = hostsim.load()
    w, h = 160, 90
    flat = scene_util.SCENES[which]()
    R = rpt_util.OracleRenderer(flat, w, h)
    osc = R.osc
    hs.hostsim_set_rho_lut(ptr(osc.lut))
    cam = scene_util.CAMERAS.get(which, (0.0, 1.2, -4.043))
    seq = rpt_util.FrameSequence(w, h, cam_path=lambda f: (cam[0] + 0.03 * f, cam[1], cam[2] + 0.02 * f))
    hsc = hostsim.Scene()
    hsc.rho = osc.lut.ctypes.data
    for fr in range(2):
        fc = seq.next()
        if dof:
            fc.DoF, fc.FocusDepth, fc.LensRadius = 1, 4.0, 0.02
        core, depth, me, coat, _ = R.gbuffer(fc)
        for prev in (0, 1):
            a = np.zeros((w * h, 16), dtype=np.uint32); b = np.zeros((w * h, 16), dtype=np.uint32)
            R.o.orc_probe_load_pixels(osc.h, C.byref(fc), ptr(core), ptr(coat), prev, ptr(a))
            hs.hostsim_probe_load_pixels(C.byref(hsc), C.byref(fc), ptr(core), ptr(coat), prev, ptr(b))
            assert a.tobytes() == b.tobytes(), (which, fr, prev, int((a != b).any(axis=1).sum()))
            assert (a[:, 0] != 0xffffffff).mean() > 0.5


def test_presampled_sets_and_light_voxel_grid_consumers():
    """Light::SampleLight's presampled-set branch (40-byte records, with and without the RNG advance the path tracer asks for) and
    LVG::Sample (jittered position -> voxel -> one of its 64 records) of zr_rt.cuh against the oracle, on the sets and the grid the
    oracle built for the many-lights atrium (>= 13107 emissive triangles, the reference's defaults 128 x 512 and 32 x 8 x 40)."""
    from tests import scene_util, rpt_util
    hs = hostsim.load()
    w, h = 96, 54
    flat = scene_util.atrium_many_lights()
    R = rpt_util.OracleRenderer(flat, w, h)
    osc = R.osc
    osc.set_presampling(128, 512)
    osc.set_light_voxel_grid((32, 8, 40), (0.6, 0.45, 0.6), 0.1)
    cam = scene_util.CAMERAS["atrium_lights"]
    fc = rpt_util.FrameSequence(w, h, cam_path=lambda f: cam).next()
    core, depth, me, coat, _ = R.gbuffer(fc)          # runs presampling and the grid build for this frame
    hsc = hostsim.Scene()
    keep = [np.ascontiguousarray(x) for x in (flat.emissives, osc.alias)]
    hsc.emissives, hsc.aliasTable = keep[0].ctypes.data, keep[1].ctypes.data
    hsc.numEmissives = len(flat.emissives)
    hsc.rho = osc.lut.ctypes.data
    hsc.sampleSets, hsc.numSampleSets, hsc.sampleSetSize = osc.sample_sets.ctypes.data, 128, 512
    hsc.lvg = osc.lvg.ctypes.data
    hsc.lvgDim[:] = (32, 8, 40); hsc.lvgExtents[:] = (0.6, 0.45, 0.6); hsc.lvgOffsetY = 0.1
    # positions: the primary hits of this frame (LoadPixel reconstruction) plus points far outside the grid
    px = np.zeros((w * h, 16), dtype=np.uint32)
    R.o.orc_probe_load_pixels(osc.h, C.byref(fc), ptr(core), ptr(coat), 0, ptr(px))
    pos = px[px[:, 0] != 0xffffffff][:, 3:6].copy().view(np.float32)
    rng = np.random.default_rng(23)
    a = (C.c_uint32 * 16)(); b = (C.c_uint32 * 16)()
    inside = 0
    for k in range(3000):
        p3 = pos[rng.integers(0, len(pos))].copy() if k % 10 else (rng.normal(size=3) * 40).astype(np.float32)
        seed = int(rng.integers(1, 2**32 - 1)); sset = int(rng.integers(0, 128))
        for adv in (0, 1):
            R.o.orc_probe_sample_light(osc.h, ptr(p3), sset, seed, adv, a); hs.hostsim_probe_sample_light(C.byref(hsc), ptr(p3), sset, seed, adv, b)
            assert bytes(a) == bytes(b), ("SampleLight presampled", k, adv, list(a), list(b))
        R.o.orc_probe_lvg_sample(osc.h, C.byref(fc), ptr(p3), seed, a); hs.hostsim_probe_lvg_sample(C.byref(hsc), C.byref(fc), ptr(p3), seed, b)
        assert bytes(a)[:52] == bytes(b)[:52], ("LVG::Sample", k, list(a)[:13], list(b)[:13])
        inside += a[0]
    assert 1500 < inside < 3000          # most positions fall into the grid, the far ones do not


@pytest.mark.parametrize("which,dof", [("glossy", False), ("glass", False), ("atrium", False), ("glossy", True)])
def test_restir_gi_temporal_reuse(which, dof):
    """ReSTIR GI's temporal reuse of zr_rgi.cuh (candidate search in the previous frame, target function at the temporal pixel with its
    visibility test, reconnection Jacobians, one- and two-candidate resampling, reservoir record codec) against the oracle's, pixel
    by pixel: the initial reservoirs of frame n (an oracle render with reuse switched off) are resampled against the oracle's
    frame n-1 reservoirs and G-buffer, with a translating camera so that reprojection is not the identity."""
    from tests import scene_util, rpt_util
    from tests.test_bvh_host import world_tris, build
    hs = hostsim.load()
    w, h = 128, 72
    flat = scene_util.SCENES[which]()
    cam = scene_util.CAMERAS.get(which, (0.0, 1.2, -4.043))
    path = lambda f: (cam[0] + 0.03 * f, cam[1], cam[2] + 0.02 * f)

    def frames(temporal_last):
        R = rpt_util.OracleRenderer(flat, w, h)
        R.gi_params.stochastic_multi_bounce = 0
        seq = rpt_util.FrameSequence(w, h, cam_path=path)
        out = []
        for fr in range(3):
            fc = seq.next()
            if dof:
                fc.DoF, fc.FocusDepth, fc.LensRadius = 1, 4.0, 0.02
            if fr == 2:
                R.gi_params.temporal_resample = int(temporal_last)
            gb = R.gbuffer(fc)
            prev_res = R.gi_curr_reservoirs().copy()
            R.rgi(fc)
            out.append((fc, gb, R.gb[R.cur ^ 1], prev_res, R.gi_curr_reservoirs().copy()))
        return R, out
    R, seq_out = frames(temporal_last=False)
    fc, gb, gb_prev, prev_res, initial = seq_out[2]        # frame 3: initial candidates only; prev_res = frame 2's output
    osc = R.osc
    hs.hostsim_set_rho_lut(ptr(osc.lut))
    wt, tri_mesh, first = world_tris(flat)
    nodes, order, leaf, info = build(wt)
    keep = [np.ascontiguousarray(x) for x in (flat.vertices, flat.indices, flat.instances, flat.materials, flat.emissives, osc.alias)]
    hsc = hostsim.Scene()
    (hsc.vertices, hsc.indices, hsc.instances, hsc.materials, hsc.emissives, hsc.aliasTable) = [k.ctypes.data for k in keep]
    hsc.nodes, hsc.leafTris, hsc.triMesh, hsc.meshFirstTri, hsc.rho = nodes.ctypes.data, leaf.ctypes.data, tri_mesh.ctypes.data, first.ctypes.data, osc.lut.ctypes.data
    hsc.numInstances, hsc.numEmissives, hsc.numTris = len(flat.instances), len(flat.emissives), len(wt)
    core, depth, me, coat, _ = gb
    pcore, _, _, pcoat, _ = gb_prev
    prev_res = np.ascontiguousarray(prev_res); initial = np.ascontiguousarray(initial)
    rng = np.random.default_rng(31)
    a = (C.c_uint32 * 17)(); b = (C.c_uint32 * 17)()
    ncand = [0, 0, 0]
    changed = 0
    for k in range(2500):
        x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        seed = int(rng.integers(1, 2**32 - 1))
        ini = initial[y * w + x:y * w + x + 1]
        R.o.orc_probe_rgi_temporal(osc.h, C.byref(fc), ptr(core), ptr(me), ptr(coat), ptr(pcore), ptr(pcoat), ptr(prev_res), ptr(ini), x, y, seed, 10, a)
        hs.hostsim_probe_rgi_temporal(C.byref(hsc), C.byref(fc), ptr(core), ptr(me), ptr(coat), ptr(pcore), ptr(pcoat), ptr(prev_res), ptr(ini), x, y, seed, 10, b)
        assert bytes(a) == bytes(b), (which, k, (x, y), list(a), list(b))
        ncand[min(a[16], 2)] += 1
        changed += bytes(a)[:16] != ini.tobytes()[:16]      # the resampled reservoir picked the temporal sample
    print(which, "candidates 0/1/2:", ncand, "sample replaced:", changed)
    assert ncand[1] + ncand[2] > 1000 and changed > 50, (ncand, changed)


@pytest.mark.parametrize("which,presample", [("cornell", None), ("glossy", None), ("glass", (16, 64)), ("atrium", None)])
def test_restir_di_candidates_and_temporal_reuse(which, presample):
    """ReSTIR DI of zr_rdi.cuh (a block of one thread) against the oracle's, pixel by pixel, as the temporal kernel runs it: RIS over
    1-2 BSDF and 3 light candidates with balance-heuristic MIS (alias table or presampled sets), the temporal candidate (plane /
    roughness / material tests at the reprojected pixel), its resampling with the shift's target re-evaluation and shadow segment,
    the 32-byte reservoir record -- on moving-camera oracle sequences, history = the oracle's previous-frame reservoirs."""
    from tests import scene_util, rpt_util
    from tests.test_bvh_host import world_tris, build
    hs = hostsim.load_di()
    w, h = 128, 72
    flat = scene_util.SCENES[which]()
    cam = scene_util.CAMERAS.get(which, (0.0, 1.2, -4.043))
    R = rpt_util.OracleRenderer(flat, w, h)
    osc = R.osc
    if presample:
        osc.set_presampling(*presample)
    seq = rpt_util.FrameSequence(w, h, cam_path=lambda f: (cam[0] + 0.03 * f, cam[1], cam[2] + 0.02 * f))
    for fr in range(3):
        fc = seq.next()
        gb = R.gbuffer(fc)
        prev_res = np.ascontiguousarray(R.di_curr_reservoirs().copy())      # before this frame's DI pass: last frame's output
        gb_prev = R.gb[R.cur ^ 1]
        R.rdi(fc)
    wt, tri_mesh, first = world_tris(flat)
    if presample:
        osc.set_presampling(*presample)        # world_tris() created a second oracle scene; keep this one's configuration in force
    nodes, order, leaf, info = build(wt)
    keep = [np.ascontiguousarray(x) for x in (flat.vertices, flat.indices, flat.instances, flat.materials, flat.emissives, osc.alias)]
    hsc = hostsim.Scene()
    (hsc.vertices, hsc.indices, hsc.instances, hsc.materials, hsc.emissives, hsc.aliasTable) = [k.ctypes.data for k in keep]
    hsc.nodes, hsc.leafTris, hsc.triMesh, hsc.meshFirstTri, hsc.rho = nodes.ctypes.data, leaf.ctypes.data, tri_mesh.ctypes.data, first.ctypes.data, osc.lut.ctypes.data
    hsc.numInstances, hsc.numEmissives, hsc.numTris = len(flat.instances), len(flat.emissives), len(wt)
    if presample:
        hsc.sampleSets, hsc.numSampleSets, hsc.sampleSetSize = osc.sample_sets.ctypes.data, presample[0], presample[1]
    core, depth, me, coat, _ = gb
    pcore, _, _, pcoat, _ = gb_prev
    rng = np.random.default_rng(41)
    a = (C.c_uint32 * 14)(); b = (C.c_uint32 * 14)()
    stats = dict(shaded=0, temporal_valid=0, lit=0, two_bsdf=0)
    for k in range(2500):
        x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        sset = int(rng.integers(0, presample[0])) if presample else 0
        for temporal in (0, 1):
            R.o.orc_probe_rdi_pixel(osc.h, C.byref(fc), ptr(core), ptr(me), ptr(coat), ptr(pcore), ptr(pcoat), ptr(prev_res), x, y, sset, temporal, 20, a)
            hs.hostsim_probe_rdi_pixel(C.byref(hsc), C.byref(fc), ptr(core), ptr(me), ptr(coat), ptr(pcore), ptr(pcoat), ptr(prev_res), x, y, sset, temporal, 20, b)
            assert bytes(a) == bytes(b), (which, k, (x, y), temporal, list(a), list(b))
        if a[13] != 0xffffffff:
            stats["shaded"] += 1; stats["temporal_valid"] += a[12]; stats["lit"] += a[3] != 0xffffffff; stats["two_bsdf"] += a[13] == 2
    print(which, stats)
    assert stats["shaded"] > 1200 and stats["temporal_valid"] > 600 and stats["lit"] > 600, stats


@pytest.mark.parametrize("which", ["glossy", "atrium"])
def test_restir_di_pairwise_mis(which):
    """PairwiseMIS of zr_rdi.cuh (Stream_Sync with both shift directions: target re-evaluation at the other pixel, the two shadow
    segments, the m_i / m_c weights; End) against the oracle's, for centre pixels with 1-4 neighbours drawn within the spatial
    radius, on the reservoirs and the target plane of an oracle frame sequence."""
    from tests import scene_util, rpt_util
    from tests.test_bvh_host import world_tris, build
    hs = hostsim.load_di()
    w, h = 128, 72
    flat = scene_util.SCENES[which]()
    cam = scene_util.CAMERAS.get(which, (0.0, 1.2, -4.043))
    R = rpt_util.OracleRenderer(flat, w, h)
    osc = R.osc
    seq = rpt_util.FrameSequence(w, h, cam_path=lambda f: cam)
    for fr in range(3):
        fc = seq.next()
        gb = R.gbuffer(fc)
        R.rdi(fc)
    res = np.ascontiguousarray(R.di_curr_reservoirs())
    target = np.ascontiguousarray(R.di_target)
    wt, tri_mesh, first = world_tris(flat)
    nodes, order, leaf, info = build(wt)
    keep = [np.ascontiguousarray(x) for x in (flat.vertices, flat.indices, flat.instances, flat.materials, flat.emissives, osc.alias)]
    hsc = hostsim.Scene()
    (hsc.vertices, hsc.indices, hsc.instances, hsc.materials, hsc.emissives, hsc.aliasTable) = [k.ctypes.data for k in keep]
    hsc.nodes, hsc.leafTris, hsc.triMesh, hsc.meshFirstTri, hsc.rho = nodes.ctypes.data, leaf.ctypes.data, tri_mesh.ctypes.data, first.ctypes.data, osc.lut.ctypes.data
    hsc.numInstances, hsc.numEmissives, hsc.numTris = len(flat.instances), len(flat.emissives), len(wt)
    core, depth, me, coat, _ = gb
    rng = np.random.default_rng(43)
    a = (C.c_uint32 * 14)(); b = (C.c_uint32 * 14)()
    shaded = picked_neighbor = 0
    for k in range(2000):
        x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        n = int(rng.integers(1, 5))
        nx = np.clip(x + rng.integers(-16, 17, n), 0, w - 1).astype(np.int32)
        ny = np.clip(y + rng.integers(-16, 17, n), 0, h - 1).astype(np.int32)
        seed = int(rng.integers(1, 2**32 - 1))
        R.o.orc_probe_rdi_pairwise(osc.h, C.byref(fc), ptr(core), ptr(coat), ptr(res), ptr(target), x, y, ptr(nx), ptr(ny), n, seed, a)
        hs.hostsim_probe_rdi_pairwise(C.byref(hsc), C.byref(fc), ptr(core), ptr(coat), ptr(res), ptr(target), x, y, ptr(nx), ptr(ny), n, seed, b)
        assert bytes(a) == bytes(b), (which, k, (x, y), list(zip(nx, ny)), list(a), list(b))
        if not (a[13] == 0xffffffff and a[0] == 0 and a[11] == 0):
            shaded += 1
            picked_neighbor += a[3] != int(res[y * w + x]["lightIdx"]) or a[0] != int(res[y * w + x]["bary"])
    print(which, "shaded", shaded, "result differs from the centre sample", picked_neighbor)
    assert shaded > 800 and picked_neighbor > 100


def test_oct32_round_trip():
    """The premise of CopyToNextFrame's short cut (zr_rpt_io.cuh): EncodeOct32u(DecodeOct32(c)) == c for EVERY 32-bit code whose two
    UNORM16 halves lie strictly inside (0, 0xffff) -- all 2^32 codes are tried; the codes that do change are aliases on the fold
    lines of the octahedron (one of their halves is 0 or 0xffff), which the short cut does not take."""
    import os
    io = hostsim.load_io()
    boundary = C.c_uint64(0)
    interior_changed = io.hostsim_oct32_round_trip(os.cpu_count() or 1, C.byref(boundary))
    assert interior_changed == 0
    assert 0 < boundary.value <= 4 * 65536


@pytest.mark.parametrize("which", ["glossy", "glass", "tunnel"])
def test_copy_to_next_frame_short_cut(which):
    """CopyToNextFrame (the "reservoir did not change" copy of the merge kernels) moves the reconnection words of a record without
    decoding them when RecordSurvivesRoundTrip says so; the bytes must equal Reservoir::Write(Reservoir::Load(record)) -- on every
    record of oracle frame sequences, and on the same records with fold-line directions, NaN / inf radiance halves and garbage in the
    words their case does not store (those take the slow path or are zeroed)."""
    from tests import scene_util, rpt_util
    io = hostsim.load_io()
    w, h = 128, 72
    R = rpt_util.OracleRenderer(scene_util.SCENES[which](), w, h)
    cam = scene_util.CAMERAS.get(which)
    seq = rpt_util.FrameSequence(w, h, cam_path=(lambda f: cam) if cam else None)
    rng = np.random.default_rng(5)
    fast_total = 0
    for fr in range(3):
        fc = seq.next()
        R.gbuffer(fc); R.rpt(fc)
        res = np.ascontiguousarray(R.curr_reservoirs())
        n = len(res)
        variants = [res]
        v = res.copy()          # hostile variant: boundary directions, special halves, garbage in unused words
        pick = rng.random(n)
        v["w_k"] = np.where(pick < 0.2, v["w_k"] & np.uint32(0xffff0000), v["w_k"])
        v["w_k"] = np.where((pick >= 0.2) & (pick < 0.4), v["w_k"] | np.uint32(0xffff0000), v["w_k"])
        v["L_rg"] = np.where(pick > 0.9, np.uint32(0x7e017c00), v["L_rg"])       # {inf, NaN}
        v["L_b"] = np.where(pick > 0.95, np.uint32(0xfc01), v["L_b"])
        v["L_b"] = v["L_b"] | np.where(pick < 0.1, np.uint32(0xabcd0000), np.uint32(0))
        for f in ("dwdA", "lightPdf"):
            v[f] = np.where(pick < 0.5, v[f], rng.random(n).astype(np.float32))
        for f in ("seed_nee", "meshIdx"):
            v[f] = np.where(pick < 0.5, v[f], rng.integers(0, 2 ** 32, n, dtype=np.uint32))
        variants.append(v)
        for recs in variants:
            recs = np.ascontiguousarray(recs)
            for m_max in (0, 4, 10):
                out = np.zeros(n, dtype=rpt_util.RES); ref = np.zeros(n, dtype=rpt_util.RES)
                fast = C.c_uint32(0)
                io.hostsim_probe_copy_to_next_frame(ptr(recs), n, m_max, ptr(out), ptr(ref), C.byref(fast))
                assert out.tobytes() == ref.tobytes(), (which, fr, m_max)
                fast_total += fast.value
    assert fast_total > 1000        # the short cut is the common case on real records
