"""Loads scene fixtures and builds the oracle-side scene (CPU) for tests, smoke() and bench.py's cpu_baseline."""
import ctypes as C
import os
import numpy as np

from zetaray_b200 import scene as zscene
from zetaray_b200._lib import ALIAS_ENTRY
from tests import orc
from tests.orc import ptr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def cornell():
    return zscene.FlatScene.load(os.path.join(GOLDEN, "cornell_emissive.npz"))


def glossy_cornell():
    """Cornell variant exercising k > 2 reconnections, metals, coat and glass (not a reference asset)."""
    s = cornell()
    m = s.materials.copy()
    # short box: rough metal; tall box: glossy dielectric below alpha_min; back wall: coated
    m[7] = zscene.make_material(base_color=(0.95, 0.64, 0.54, 1), metallic=1.0, roughness=0.25, double_sided=True)
    m[8] = zscene.make_material(base_color=(0.725, 0.71, 0.68, 1), roughness=0.1, double_sided=True)
    m[3] = zscene.make_material(base_color=(0.2, 0.3, 0.7, 1), roughness=0.6, coat_weight=1.0, coat_roughness=0.1,
                                coat_color=(0.9, 0.9, 0.9), double_sided=True)
    s.materials = m
    return s


def glass_cornell():
    """Cornell variant with transmissive materials (not a reference asset): a clear-glass short box (specular
    transmission -> the 4-bounce glossy/transmissive budget, eta tracking, T_MIN_TR_RAY shadow rays), a rough coloured
    glass tall box with a transmission depth (in-medium extinction through zr_logf / zr_expf) and a thin-walled
    translucent back wall (subsurface lobe)."""
    s = cornell()
    m = s.materials.copy()
    m[7] = zscene.make_material(base_color=(1.0, 1.0, 1.0, 1), roughness=0.0, ior=1.5, transmission=1.0, double_sided=True)
    m[8] = zscene.make_material(base_color=(0.6, 0.85, 0.7, 1), roughness=0.3, ior=1.33, transmission=1.0, transmission_depth=0.5,
                                double_sided=True)
    m[3] = zscene.make_material(base_color=(0.8, 0.7, 0.5, 1), roughness=0.5, thin_walled=True, subsurface=0.6, double_sided=True)
    s.materials = m
    return s


def atrium_small():
    """"Sponza-class" procedural atrium (config C4 stand-in) at a size the brute-force oracle traces in seconds."""
    from zetaray_b200 import procedural
    return procedural.atrium(0.12)


def atrium_many_lights():
    """Same hall, coarser, but with finely tessellated lanterns: >= 13107 emissive triangles, the reference's threshold
    for presampled sets (DefaultRendererImpl.h:37-41)."""
    from zetaray_b200 import procedural
    return procedural.atrium(0.08, lamp_tris=224)


def tunnel_small():
    """"Subway-class" procedural station tunnel (config C5 stand-in): glass screens, glossy metal, emissive tubes."""
    from zetaray_b200 import procedural
    return procedural.tunnel(0.1)


SCENES = {"cornell": cornell, "glossy": glossy_cornell, "glass": glass_cornell, "atrium": atrium_small,
          "atrium_lights": atrium_many_lights, "tunnel": tunnel_small}
# static camera per scene (looks down +Z); the Cornell variants use the reference's default camera
CAMERAS = {"atrium": (0.0, 1.7, -13.0), "atrium_lights": (0.0, 1.7, -13.0), "tunnel": (-1.6, 1.7, -4.0)}


# ---- radiometric truth scenes (oracle/indep_radiometry.py) ----------------------------------------------------------------------
# Every surface is an axis-aligned rectangle {p0, eu, ev, nu x nv cells}: a point is p0 + s eu + t ev, s, t in [0, 1], and
# cross(eu, ev) is the side the vertex normals (and an emitter's emission) face. Material parameters are k / 255 so that the
# 8-bit material and G-buffer encodings reproduce them exactly; emitter edges are dyadic and each triangle's two edges from its
# first vertex run along eu and ev, so the emissive record's half-precision lengths are exact.
def _k(v):
    return tuple(float(np.float32(round(x * 255) / 255)) for x in v) if isinstance(v, tuple) else float(np.float32(round(v * 255) / 255))


DIFFUSE = dict(base_color=_k((0.6, 0.6, 0.6)), roughness=1.0, double_sided=True)
GLOSSY_ROUGH = dict(base_color=_k((0.5, 0.6, 0.7)), roughness=_k(0.5), double_sided=True)        # alpha 0.25: above both alpha_min
GLOSSY_MID = dict(base_color=_k((0.7, 0.6, 0.5)), roughness=_k(0.12), double_sided=True)         # alpha (31/255)^2 = 0.0148: DI 0.0025 < alpha < PT 0.0306
METAL = dict(base_color=_k((0.95, 0.64, 0.54)), metallic=1.0, roughness=_k(0.3), double_sided=True)
COATED = dict(base_color=_k((0.2, 0.3, 0.7)), roughness=_k(0.6), coat_weight=1.0, coat_roughness=_k(0.1), coat_color=_k((0.9, 0.9, 0.9)),
              coat_ior=1.6, double_sided=True)


def _emitter(rgb, strength, double_sided=False):
    return dict(base_color=(0, 0, 0), roughness=1.0, emissive_factor=_k(rgb), emissive_strength=strength, double_sided=double_sided)


TRUTH_SCENES = {
    # floor rough diffuse, back wall glossy; a one-sided light facing down (the wall above its plane sees only its back), a
    # double-sided vertical light, and an occluder between the first light and the floor (umbra + penumbra)
    "truth_a": [
        dict(name="floor", p0=(-4, 0, -3), eu=(0, 0, 9), ev=(8, 0, 0), mat=DIFFUSE),
        dict(name="wall", p0=(-4, 0, 3), eu=(0, 4, 0), ev=(8, 0, 0), mat=GLOSSY_ROUGH),
        dict(name="light_down", p0=(-1.25, 2, 0.5), eu=(1, 0, 0), ev=(0, 0, 0.5), mat=_emitter((1.0, 0.9, 0.8), 8.0)),
        dict(name="light_side", p0=(2, 0.5, 1), eu=(0, 0, 1), ev=(0, 1, 0), mat=_emitter((0.6, 0.8, 1.0), 2.0, double_sided=True)),
        dict(name="occluder", p0=(-1.0, 1, 0.25), eu=(0, 0, 1), ev=(0.5, 0, 0), mat=DIFFUSE),
    ],
    # glossy floor (alpha between the two alpha_min), coated back wall, metal side wall; a 256-triangle dim panel and a small
    # strong light: per-triangle powers differ by ~190x, so the alias table is far from uniform
    "truth_b": [
        dict(name="floor", p0=(-4, 0, -3), eu=(0, 0, 9), ev=(8, 0, 0), mat=GLOSSY_MID),
        dict(name="wall", p0=(-4, 0, 3), eu=(0, 4, 0), ev=(8, 0, 0), mat=COATED),
        dict(name="side", p0=(-3, 0, -3), eu=(0, 4, 0), ev=(0, 0, 6), mat=METAL),
        dict(name="panel", p0=(0.5, 2.5, 1), eu=(2, 0, 0), ev=(0, 0, 1), nu=16, nv=8, mat=_emitter((1.0, 1.0, 1.0), 1.0)),
        dict(name="light_small", p0=(-1.5, 1.5, 0), eu=(0.5, 0, 0), ev=(0, 0, 0.5), mat=_emitter((1.0, 0.7, 0.4), 16.0)),
    ],
}


def truth_scene(name):
    """Builds TRUTH_SCENES[name] with SceneBuilder; returns (FlatScene, the description)."""
    desc = TRUTH_SCENES[name]
    b = zscene.SceneBuilder()
    for r in desc:
        p0, eu, ev = (np.asarray(r[k], dtype=np.float64) for k in ("p0", "eu", "ev"))
        nu, nv = r.get("nu", 1), r.get("nv", 1)
        n = np.cross(eu, ev); n /= np.linalg.norm(n)
        s, t = np.meshgrid(np.arange(nu + 1) / nu, np.arange(nv + 1) / nv, indexing="ij")
        pos = p0 + s.reshape(-1, 1) * eu + t.reshape(-1, 1) * ev
        uv = np.stack([s.reshape(-1), t.reshape(-1)], axis=1)
        vid = lambda i, j: i * (nv + 1) + j
        idx = []
        for i in range(nu):
            for j in range(nv):
                # (c00, c10, c01) and (c11, c01, c10): both triangles' edges from vertex 0 run along +-eu / +-ev
                idx += [vid(i, j), vid(i + 1, j), vid(i, j + 1), vid(i + 1, j + 1), vid(i, j + 1), vid(i + 1, j)]
        b.add_mesh(pos, np.tile(n, (len(pos), 1)), uv, idx, b.add_material(zscene.make_material(**r["mat"])))
    return b.finish(), desc


_RHO_LUT = None


def rho_lut():
    """The directional-albedo table, loaded once and kept alive for the life of the process: the oracle holds a bare pointer to it
    (orc_set_rho_lut), so a per-object copy would dangle as soon as a temporary OracleScene is collected."""
    global _RHO_LUT
    if _RHO_LUT is None:
        _RHO_LUT = np.fromfile(os.path.join(ROOT, "zetaray_b200", "assets", "rho_lut.bin"), dtype=np.uint16)
        assert _RHO_LUT.size == 64 * 32 * 16
    return _RHO_LUT


class OracleScene:
    def __init__(self, flat):
        self.o = orc.load()
        self.flat = flat
        self.lut = rho_lut()
        self.o.orc_set_rho_lut(ptr(self.lut))
        self.alias = np.zeros(max(len(flat.emissives), 1), dtype=ALIAS_ENTRY)
        self.h = C.c_void_p(self.o.orc_scene_create(ptr(flat.vertices), ptr(flat.indices), ptr(flat.instances),
                                                    len(flat.instances), ptr(flat.instance_num_tris), ptr(flat.materials),
                                                    ptr(flat.emissives) if len(flat.emissives) else None, len(flat.emissives),
                                                    ptr(self.alias)))
        if len(flat.emissives):
            self.power = np.zeros(len(flat.emissives), dtype=np.float32)
            self.o.orc_estimate_power(self.h, ptr(self.power))
            w = self.power.copy()
            self.o.orc_alias_build_emissive(ptr(w), len(w), 0, ptr(self.alias))

    def set_presampling(self, num_sets, set_size):
        """PresampleEmissives: num_sets x set_size records of 40 bytes; 0, 0 switches back to alias-table sampling."""
        self.num_sets, self.set_size = num_sets, set_size
        self.sample_sets = np.zeros(max(num_sets * set_size, 1) * 10, dtype=np.uint32)      # 40-byte records
        self.o.orc_scene_set_sample_sets(self.h, ptr(self.sample_sets) if num_sets else None, num_sets, set_size)

    def presample(self, frame_num):
        if getattr(self, "num_sets", 0):
            self.o.orc_presample(self.h, frame_num, self.num_sets * self.set_size, ptr(self.sample_sets))

    def set_light_voxel_grid(self, grid_dim, extents, offset_y=0.0):
        self.lvg_dim = tuple(grid_dim)
        n = grid_dim[0] * grid_dim[1] * grid_dim[2]
        self.lvg = np.zeros(max(n, 1) * 64 * 8, dtype=np.uint32)            # 32-byte records
        d = (C.c_uint32 * 3)(*grid_dim)
        e = (C.c_float * 3)(*extents)
        self.o.orc_scene_set_lvg(self.h, ptr(self.lvg) if n else None, d, e, offset_y)

    def build_light_voxel_grid(self, fc):
        if getattr(self, "lvg_dim", None) and self.lvg_dim[0]:
            self.o.orc_build_lvg(self.h, C.byref(fc), ptr(self.lvg))

    def gbuffer(self, fc, tridiff=False, nthreads=8):
        n = fc.RenderWidth * fc.RenderHeight
        core = np.zeros((n, 4), dtype=np.uint32)
        depth = np.zeros(n, dtype=np.float32)
        me = np.zeros((n, 2), dtype=np.uint32)
        coat = np.zeros((n, 2), dtype=np.uint32)
        td = np.zeros((n, 6), dtype=np.uint32) if tridiff else None
        self.o.orc_gbuffer(self.h, C.byref(fc), ptr(core), ptr(depth), ptr(me), ptr(coat), ptr(td) if tridiff else None, nthreads)
        return core, depth, me, coat, td
