"""glTF -> ZetaRay flat scene buffers (offline converter; not on the hot path).

Follows the reference's scene-ingest contract (SURVEY A.8):
  * ZetaCore/Model/glTF.cpp:144-268  positions/normals/tangents (x, y, -z), winding (i0, i2, i1)
  * ZetaCore/Model/glTF.cpp:830-865  node translation (x, y, -z), rotation (-x, -y, z, w)
  * ZetaCore/Core/Vertex.h:8-14      Vertex {pos, uv, oct32 normal, oct32 tangent}
  * ZetaCore/Core/Material.h         32-byte packed material
  * ZetaCore/RayTracing/RtCommon.h   MeshInstance (64 B), EmissiveTriangle (48 B)
  * ZetaCore/Scene/SceneCore.cpp:199-235  emissive triangles baked to world space, ID = PCG3d hash
Textures are not supported in this round: a textured base colour is replaced by the material's
factor (or `texture_fallback`), see DESIGN.md."""
import json
import os
import struct

import numpy as np

VERTEX = np.dtype([("pos", "<f4", 3), ("uv", "<f4", 2), ("normal", "<u2", 2), ("tangent", "<u2", 2)])
MATERIAL = np.dtype([("BaseColorFactor", "<u4"), ("BaseColorTex_Subsurf_CoatWeight", "<u4"), ("NormalTex_TrDepth", "<u4"),
                     ("MRTex_SpecRoughness_CoatRoughness", "<u4"), ("EmissiveFactor_NormalScale", "<u4"),
                     ("EmissiveStrength_IOR", "<u4"), ("EmissiveTex_AlphaCutoff_CoatIOR", "<u4"), ("CoatColor_Flags", "<u4")])
MESH_INSTANCE = np.dtype([("BaseVtxOffset", "<u4"), ("BaseIdxOffset", "<u4"), ("Rotation", "<u2", 4), ("Scale", "<u2", 3),
                          ("MatIdx", "<u2"), ("BaseEmissiveTriOffset", "<u4"), ("Translation", "<f4", 3),
                          ("PrevRotation", "<u2", 4), ("PrevScale", "<u2", 3), ("dTranslation", "<u2", 3),
                          ("BaseColorTex", "<u2"), ("AlphaFactor_Cutoff", "<u2")])
EMISSIVE_TRI = np.dtype([("Vtx0", "<f4", 3), ("V0V1", "<u2", 2), ("V0V2", "<u2", 2), ("EdgeLengths", "<u2", 2),
                         ("ID", "<u4"), ("PackedA", "<u4"), ("PackedB", "<u4"), ("UV0", "<u2", 2), ("UV1", "<u2", 2), ("UV2", "<u2", 2)])
assert VERTEX.itemsize == 28 and MATERIAL.itemsize == 32 and MESH_INSTANCE.itemsize == 64 and EMISSIVE_TRI.itemsize == 48

INVALID_ID = 0xffff
F32 = np.float32


def pcg3d(x, y, z):
    m = 0xffffffff
    x = (x * 1664525 + 1013904223) & m; y = (y * 1664525 + 1013904223) & m; z = (z * 1664525 + 1013904223) & m
    x = (x + y * z) & m; y = (y + z * x) & m; z = (z + x * y) & m
    x ^= x >> 16; y ^= y >> 16; z ^= z >> 16
    x = (x + y * z) & m; y = (y + z * x) & m; z = (z + x * y) & m
    return x, y, z


def _unorm(v, bits):
    """Math::FloatToUNorm8 / FloatToUNorm16 (ZetaCore/Math/Common.h:158-166): (uintN) fmaf(value, 2^N - 1, 0.5f) -- one float32
    rounding of the exact product-sum, then truncation. Pinned against the reference's own code (tests/test_scene_pinning.py)."""
    v = np.asarray(v, dtype=np.float32).astype(np.float64)
    t = (v * float((1 << bits) - 1) + 0.5).astype(np.float32)      # the float64 sum is exact to well below float32 resolution
    return np.clip(t, 0.0, float((1 << bits) - 1)).astype(np.uint32)


def _unorm_rne(v01, bits):
    """The SIMD packers (unorm2 / unorm4::FromNormalized, Vector.h:626-647, 745-769; Float3ToRGB8, Color.h:21-33):
    float32 multiply by 2^N - 1, then _mm_cvtps_epi32 = round to nearest EVEN."""
    t = np.asarray(v01, dtype=np.float32) * np.float32((1 << bits) - 1)
    return np.clip(np.rint(t), 0, (1 << bits) - 1).astype(np.uint32)


def snorm_to_unorm16(v):
    """[-1, 1] -> UNORM16 as unorm2 / unorm4::FromNormalized do it: fmadd(v, 0.5, 0.5) in float32 (v * 0.5 is exact, so one
    rounding), times 65535, round to nearest even."""
    v = np.asarray(v, dtype=np.float32)
    return _unorm_rne(v * np.float32(0.5) + np.float32(0.5), 16)


def oct_encode_unorm16(n):
    """Math::oct32 (ZetaCore/Math/OctahedralVector.h:8-39 over VectorFuncs.h:123-153 encode_octahedral): float32 throughout,
    the abs-sum in hadd_float3's order (|x| + |z|) + |y|, sign(v) = v >= 0 ? 1 : -1 of the INPUT vector, 2 x UNORM16 (RNE).
    Bit-exact with the reference's own code (tests/test_scene_pinning.py)."""
    n = np.asarray(n, dtype=np.float32).reshape(-1, 3)
    a = np.abs(n)
    s = (a[:, 0] + a[:, 2]) + a[:, 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        p = n[:, :2] / s[:, None]
    sgn = np.where(n[:, :2] >= 0, np.float32(1.0), np.float32(-1.0))
    folded = (np.float32(1.0) - np.abs(p[:, ::-1])) * sgn
    enc = np.where((n[:, 2] <= 0)[:, None], folded, p).astype(np.float32)
    return snorm_to_unorm16(enc).astype(np.uint16)


def half_bits(v):
    return np.asarray(v, dtype=np.float32).astype(np.float16).view(np.uint16)


def rgb8(c):
    """Math::Float3ToRGB8 (ZetaCore/Math/Color.h:21-33): float32 * 255, round to nearest even, saturate."""
    u = _unorm_rne(np.asarray(c, dtype=np.float32)[:3], 8)
    return int(u[0]) | (int(u[1]) << 8) | (int(u[2]) << 16)


def rgba8(c):
    """Math::Float4ToRGBA8 (Color.h:35-46)."""
    u = _unorm_rne(np.asarray(c, dtype=np.float32)[:4], 8)
    return int(u[0]) | (int(u[1]) << 8) | (int(u[2]) << 16) | (int(u[3]) << 24)


def make_material(base_color=(1, 1, 1, 1), metallic=0.0, roughness=0.3, ior=1.5, transmission=0.0,
                  emissive_factor=(0, 0, 0), emissive_strength=1.0, coat_weight=0.0, coat_color=(0.8, 0.8, 0.8),
                  coat_roughness=0.0, coat_ior=1.6, double_sided=False, thin_walled=False, subsurface=0.0,
                  transmission_depth=0.0):
    """ZetaCore/Core/Material.h setters (defaults from the constructor, Material.h:69-93)."""
    m = np.zeros(1, dtype=MATERIAL)[0]
    bc = list(base_color) + [1.0] * (4 - len(base_color))
    m["BaseColorFactor"] = rgba8(bc)
    m["BaseColorTex_Subsurf_CoatWeight"] = INVALID_ID | (int(_unorm(subsurface, 8)) << 16) | (int(_unorm(coat_weight, 8)) << 24)
    m["NormalTex_TrDepth"] = INVALID_ID | (int(half_bits(transmission_depth)) << 16)
    m["MRTex_SpecRoughness_CoatRoughness"] = INVALID_ID | (int(_unorm(roughness, 8)) << 16) | (int(_unorm(coat_roughness, 8)) << 24)
    m["EmissiveFactor_NormalScale"] = rgb8(emissive_factor) | (int(_unorm(1.0, 8)) << 24)
    # (ior - MIN_IOR) / (MAX_IOR - MIN_IOR) in float32 (Material.h:160-163, 184-190)
    nior = (np.float32(ior) - np.float32(1.0)) / (np.float32(2.5) - np.float32(1.0))
    ncoat = (np.float32(coat_ior) - np.float32(1.0)) / (np.float32(2.5) - np.float32(1.0))
    m["EmissiveStrength_IOR"] = int(half_bits(emissive_strength)) | (int(_unorm(nior, 16)) << 16)
    m["EmissiveTex_AlphaCutoff_CoatIOR"] = INVALID_ID | (int(_unorm(0.5, 8)) << 16) | (int(_unorm(ncoat, 8)) << 24)
    flags = 0
    if metallic >= 0.9: flags |= 1 << 24
    if double_sided: flags |= 1 << 25
    if transmission >= 0.9: flags |= 1 << 26
    if thin_walled: flags |= 1 << 29
    m["CoatColor_Flags"] = rgb8(coat_color) | flags
    return m


def quat_rotate(q, v):
    q = np.asarray(q, dtype=np.float64); v = np.asarray(v, dtype=np.float64)
    t = np.cross(2.0 * q[:3], v)
    return v + q[3] * t + np.cross(q[:3], t)


def emissive_triangle(v0, v1, v2, uv0, uv1, uv2, factor_rgb8, strength_half_bits, tri_id, double_sided):
    """RT::EmissiveTriangle ctor + StoreVertices (RtCommon.h:72-198)."""
    e = np.zeros(1, dtype=EMISSIVE_TRI)[0]
    v0 = np.asarray(v0, dtype=np.float32); v1 = np.asarray(v1, dtype=np.float32); v2 = np.asarray(v2, dtype=np.float32)
    e["Vtx0"] = v0
    e0 = (v1 - v0).astype(np.float32); e1 = (v2 - v0).astype(np.float32)
    l0 = np.sqrt((e0[0] * e0[0] + e0[1] * e0[1]) + e0[2] * e0[2]); l1 = np.sqrt((e1[0] * e1[0] + e1[1] * e1[1]) + e1[2] * e1[2])
    e["V0V1"] = oct_encode_unorm16(e0 / l0)[0]
    e["V0V2"] = oct_encode_unorm16(e1 / l1)[0]
    e["EdgeLengths"] = half_bits([l0, l1])
    e["ID"] = tri_id
    e["PackedA"] = (factor_rgb8 & 0xffffff) | (1 << 24) | ((1 << 25) if double_sided else 0) | ((int(strength_half_bits) & 0xf) << 28)
    e["PackedB"] = INVALID_ID | (int(strength_half_bits) << 16)
    e["UV0"] = half_bits(uv0); e["UV1"] = half_bits(uv1); e["UV2"] = half_bits(uv2)
    return e


def emissive_triangles(v0, v1, v2, uv0, uv1, uv2, factor_rgb8, strength_half_bits, tri_ids, double_sided):
    """Batch form of emissive_triangle (same arithmetic, n triangles at once)."""
    v0 = np.asarray(v0, dtype=np.float32).reshape(-1, 3); v1 = np.asarray(v1, dtype=np.float32).reshape(-1, 3)
    v2 = np.asarray(v2, dtype=np.float32).reshape(-1, 3)
    n = len(v0)
    e = np.zeros(n, dtype=EMISSIVE_TRI)
    e["Vtx0"] = v0
    e0 = (v1 - v0).astype(np.float32); e1 = (v2 - v0).astype(np.float32)
    l0 = np.sqrt((e0[:, 0] * e0[:, 0] + e0[:, 1] * e0[:, 1]) + e0[:, 2] * e0[:, 2])
    l1 = np.sqrt((e1[:, 0] * e1[:, 0] + e1[:, 1] * e1[:, 1]) + e1[:, 2] * e1[:, 2])
    e["V0V1"] = oct_encode_unorm16(e0 / l0[:, None])
    e["V0V2"] = oct_encode_unorm16(e1 / l1[:, None])
    e["EdgeLengths"] = np.stack([half_bits(l0), half_bits(l1)], axis=1)
    e["ID"] = np.asarray(tri_ids, dtype=np.uint32)
    e["PackedA"] = (factor_rgb8 & 0xffffff) | (1 << 24) | ((1 << 25) if double_sided else 0) | ((int(strength_half_bits) & 0xf) << 28)
    e["PackedB"] = INVALID_ID | (int(strength_half_bits) << 16)
    e["UV0"] = half_bits(uv0).reshape(-1, 2); e["UV1"] = half_bits(uv1).reshape(-1, 2); e["UV2"] = half_bits(uv2).reshape(-1, 2)
    return e


def pcg3d_np(x, y, z):
    """pcg3d over uint32 arrays."""
    x = np.asarray(x, dtype=np.uint64); y = np.asarray(y, dtype=np.uint64); z = np.asarray(z, dtype=np.uint64)
    m = np.uint64(0xffffffff); a = np.uint64(1664525); c = np.uint64(1013904223); s16 = np.uint64(16)
    x = (x * a + c) & m; y = (y * a + c) & m; z = (z * a + c) & m
    x = (x + y * z) & m; y = (y + z * x) & m; z = (z + x * y) & m
    x ^= x >> s16; y ^= y >> s16; z ^= z >> s16
    x = (x + y * z) & m; y = (y + z * x) & m; z = (z + x * y) & m
    return x.astype(np.uint32), y.astype(np.uint32), z.astype(np.uint32)


def quat_rotate_np(q, v):
    q = np.asarray(q, dtype=np.float64); v = np.asarray(v, dtype=np.float64)
    t = np.cross(2.0 * q[:3], v)
    return v + q[3] * t + np.cross(q[:3], t)


class FlatScene:
    """The arrays the renderer publishes by name (ZetaCore/Scene/SceneRenderer.h:15-33)."""

    def __init__(self):
        self.vertices = np.zeros(0, dtype=VERTEX)
        self.indices = np.zeros(0, dtype=np.uint32)
        self.instances = np.zeros(0, dtype=MESH_INSTANCE)
        self.instance_num_tris = np.zeros(0, dtype=np.uint32)
        self.materials = np.zeros(0, dtype=MATERIAL)
        self.emissives = np.zeros(0, dtype=EMISSIVE_TRI)

    def save(self, path):
        np.savez_compressed(path, vertices=self.vertices, indices=self.indices, instances=self.instances,
                            instance_num_tris=self.instance_num_tris, materials=self.materials, emissives=self.emissives)

    @staticmethod
    def load(path):
        z = np.load(path)
        s = FlatScene()
        s.vertices = z["vertices"].view(VERTEX).reshape(-1)
        s.indices = z["indices"].astype(np.uint32)
        s.instances = z["instances"].view(MESH_INSTANCE).reshape(-1)
        s.instance_num_tris = z["instance_num_tris"].astype(np.uint32)
        s.materials = z["materials"].view(MATERIAL).reshape(-1)
        s.emissives = z["emissives"].view(EMISSIVE_TRI).reshape(-1)
        return s

    @property
    def num_triangles(self):
        return int(self.instance_num_tris.sum())


EMISSIVE_A_MATERIAL_BITS = 0xffffff | (1 << 25) | (0xf << 28)     # the PackedA bits emissive_triangle takes from the material


def update_materials(flat, first, materials):
    """zr_scene_update_materials on host arrays: a copy of `flat` whose materials [first, first + len(materials)) are replaced
    and whose emissive triangles of the instances using them carry the re-derived factor, double-sided flag and strength, as
    emissive_triangle stores them. Geometry, instances and the emissive set stay. Raises ValueError where the library refuses
    the edit: a material that becomes emissive while an instance using it has no emissive triangles, or an edit that leaves
    every emissive triangle with zero factor or strength."""
    materials = np.asarray(materials, dtype=MATERIAL).reshape(-1)
    if len(materials) == 0 or first < 0 or first + len(materials) > len(flat.materials):
        raise ValueError("materials [%d, %d) of %d" % (first, first + len(materials), len(flat.materials)))
    out = FlatScene()
    out.vertices, out.indices, out.instances, out.instance_num_tris = flat.vertices, flat.indices, flat.instances, flat.instance_num_tris
    out.materials = flat.materials.copy()
    out.materials[first:first + len(materials)] = materials
    out.emissives = flat.emissives.copy()
    factor = lambda m: int(m["EmissiveFactor_NormalScale"]) & 0xffffff
    strength = lambda m: int(m["EmissiveStrength_IOR"]) & 0xffff
    bits = lambda m: (factor(m) | (int(m["CoatColor_Flags"]) & (1 << 25)) | ((strength(m) & 0xf) << 28), strength(m) << 16)
    powered = lit = False
    for m, (inst, nt) in enumerate(zip(flat.instances, flat.instance_num_tris)):
        mi, base = int(inst["MatIdx"]), int(inst["BaseEmissiveTriOffset"])
        old, new = flat.materials[mi], out.materials[mi]
        if base == 0xffffffff or nt == 0:
            if factor(new) and not factor(old):
                raise ValueError("material %d becomes emissive, but instance %d, which uses it, has no emissive triangles" % (mi, m))
            continue
        lit = True
        powered |= bool(factor(new)) and (strength(new) & 0x7fff) != 0
        if bits(new) != bits(old):      # the library rewrites the triangles of changed lights only
            e = out.emissives[base:base + nt]
            a, b = bits(new)
            e["PackedA"] = (e["PackedA"] & np.uint32(~EMISSIVE_A_MATERIAL_BITS & 0xffffffff)) | np.uint32(a)
            e["PackedB"] = (e["PackedB"] & np.uint32(0xffff)) | np.uint32(b)
    if len(flat.emissives) and lit and not powered:
        raise ValueError("the edit leaves every emissive triangle with zero emissive factor or strength")
    return out


class SceneBuilder:
    """Programmatic scene assembly (also used for the synthetic 'Sponza-class' / 'Subway-class' scenes)."""

    def __init__(self):
        self.v, self.i, self.inst, self.ntris, self.mats, self.em = [], [], [], [], [], []
        self.nv = 0
        self.ni = 0
        self.nem = 0
        self.geo = {}

    def add_material(self, mat):
        self.mats.append(mat)
        return len(self.mats) - 1

    def add_mesh(self, positions, normals, uvs, indices, mat_idx, translation=(0, 0, 0), rotation=(0, 0, 0, 1),
                 scale=(1, 1, 1), tangents=None):
        """positions/normals already in ZetaRay's left-handed space; indices clockwise."""
        positions = np.asarray(positions, dtype=np.float32).reshape(-1, 3)
        normals = np.asarray(normals, dtype=np.float32).reshape(-1, 3)
        uvs = np.asarray(uvs, dtype=np.float32).reshape(-1, 2)
        indices = np.asarray(indices, dtype=np.uint32).reshape(-1)
        n = len(positions)
        vb = np.zeros(n, dtype=VERTEX)
        vb["pos"] = positions
        vb["uv"] = uvs
        vb["normal"] = oct_encode_unorm16(normals)
        vb["tangent"] = oct_encode_unorm16(tangents if tangents is not None else np.tile([1.0, 0, 0], (n, 1)))
        inst = self._instance(self.nv, self.ni, mat_idx, translation, rotation, scale)
        ntri = len(indices) // 3
        geo_idx = len(self.inst)
        self._emit_emissives(inst, mat_idx, positions, uvs, indices, geo_idx)
        self.v.append(vb); self.i.append(indices); self.inst.append(inst); self.ntris.append(ntri)
        self.geo[geo_idx] = (int(inst["BaseVtxOffset"]), int(inst["BaseIdxOffset"]), positions, uvs, indices)
        self.nv += n
        self.ni += len(indices)
        return geo_idx

    def add_instance_of(self, geo_idx, mat_idx, translation=(0, 0, 0), rotation=(0, 0, 0, 1), scale=(1, 1, 1)):
        """Another instance of an already added mesh: same vertex / index range, its own transform and material
        (RT::MeshInstance only stores offsets into the shared buffers, RtCommon.h:47-64)."""
        bv, bi, positions, uvs, indices = self.geo[geo_idx]
        inst = self._instance(bv, bi, mat_idx, translation, rotation, scale)
        new_idx = len(self.inst)
        self._emit_emissives(inst, mat_idx, positions, uvs, indices, new_idx)
        self.inst.append(inst); self.ntris.append(len(indices) // 3)
        return new_idx

    def _instance(self, base_vtx, base_idx, mat_idx, translation, rotation, scale):
        inst = np.zeros(1, dtype=MESH_INSTANCE)[0]
        inst["BaseVtxOffset"] = base_vtx
        inst["BaseIdxOffset"] = base_idx
        q = np.asarray(rotation, dtype=np.float64)
        q = q / np.linalg.norm(q)
        inst["Rotation"] = snorm_to_unorm16(q.astype(np.float32)).astype(np.uint16)       # unorm4::FromNormalized, RtAccelerationStructure.cpp:345
        inst["Scale"] = half_bits(scale)
        inst["MatIdx"] = mat_idx
        inst["Translation"] = np.asarray(translation, dtype=np.float32)
        inst["PrevRotation"] = inst["Rotation"]
        inst["PrevScale"] = inst["Scale"]
        inst["dTranslation"] = half_bits([0, 0, 0])
        inst["BaseColorTex"] = 0xffff
        inst["AlphaFactor_Cutoff"] = 0xffff       # cutoff = 1.0 -> opaque (GBufferRT_Inline.hlsl:41-43)
        return inst

    def _emit_emissives(self, inst, mat_idx, positions, uvs, indices, geo_idx):
        mat = self.mats[mat_idx]
        ef = int(mat["EmissiveFactor_NormalScale"]) & 0xffffff
        if ef == 0:
            inst["BaseEmissiveTriOffset"] = 0xffffffff
            return
        ntri = len(indices) // 3
        inst["BaseEmissiveTriOffset"] = self.nem
        strength = int(mat["EmissiveStrength_IOR"]) & 0xffff
        ds = bool(int(mat["CoatColor_Flags"]) & (1 << 25))
        # same arithmetic the shaders use for world positions: quantised rotation/scale
        qd = (inst["Rotation"].astype(np.float64) / 65535.0) * 2.0 - 1.0
        qd = qd / np.linalg.norm(qd)
        sd = inst["Scale"].view(np.float16).astype(np.float64)
        td = inst["Translation"].astype(np.float64)
        pw = quat_rotate_np(qd, positions.astype(np.float64) * sd) + td
        tri = indices.reshape(-1, 3)
        ids = pcg3d_np(np.full(ntri, geo_idx), np.zeros(ntri), np.arange(ntri))[0]
        self.em.append(emissive_triangles(pw[tri[:, 0]], pw[tri[:, 1]], pw[tri[:, 2]], uvs[tri[:, 0]], uvs[tri[:, 1]],
                                          uvs[tri[:, 2]], ef, strength, ids, ds))
        self.nem += ntri

    def finish(self):
        s = FlatScene()
        s.vertices = np.concatenate(self.v) if self.v else np.zeros(0, dtype=VERTEX)
        s.indices = np.concatenate(self.i).astype(np.uint32) if self.i else np.zeros(0, dtype=np.uint32)
        s.instances = np.array(self.inst, dtype=MESH_INSTANCE)
        s.instance_num_tris = np.array(self.ntris, dtype=np.uint32)
        s.materials = np.array(self.mats, dtype=MATERIAL)
        s.emissives = np.concatenate(self.em) if self.em else np.zeros(0, dtype=EMISSIVE_TRI)
        return s


_CT = {5120: "b", 5121: "B", 5122: "h", 5123: "H", 5125: "I", 5126: "f"}
_NC = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4}


def load_gltf(path, texture_fallback=(0.5, 0.5, 0.5)):
    """Minimal glTF 2.0 reader for the hot path's needs (static meshes, factors only)."""
    g = json.load(open(path))
    base = os.path.dirname(path)
    buffers = [open(os.path.join(base, b["uri"]), "rb").read() for b in g["buffers"]]

    def accessor(idx):
        a = g["accessors"][idx]
        bv = g["bufferViews"][a["bufferView"]]
        fmt = _CT[a["componentType"]]
        nc = _NC[a["type"]]
        off = bv.get("byteOffset", 0) + a.get("byteOffset", 0)
        arr = np.frombuffer(buffers[bv["buffer"]], dtype=np.dtype(fmt).newbyteorder("<"), count=a["count"] * nc, offset=off)
        return arr.reshape(a["count"], nc) if nc > 1 else arr

    b = SceneBuilder()
    for m in g.get("materials", []):
        pbr = m.get("pbrMetallicRoughness", {})
        bc = pbr.get("baseColorFactor", [1, 1, 1, 1])
        if "baseColorTexture" in pbr:
            bc = list(texture_fallback) + [1.0]
        ext = m.get("extensions", {})
        strength = ext.get("KHR_materials_emissive_strength", {}).get("emissiveStrength", 1.0)
        ior = ext.get("KHR_materials_ior", {}).get("ior", 1.5)
        tr = ext.get("KHR_materials_transmission", {}).get("transmissionFactor", 0.0)
        cc = ext.get("KHR_materials_clearcoat", {})
        b.add_material(make_material(base_color=bc, metallic=pbr.get("metallicFactor", 1.0),
                                     roughness=pbr.get("roughnessFactor", 1.0), ior=ior, transmission=tr,
                                     emissive_factor=m.get("emissiveFactor", [0, 0, 0]), emissive_strength=strength,
                                     coat_weight=cc.get("clearcoatFactor", 0.0),
                                     coat_roughness=cc.get("clearcoatRoughnessFactor", 0.0),
                                     double_sided=m.get("doubleSided", False)))
    flip = np.array([1, 1, -1], dtype=np.float32)

    def visit(node_idx):
        node = g["nodes"][node_idx]
        if "mesh" in node:
            t = np.array(node.get("translation", [0, 0, 0]), dtype=np.float32) * flip
            r = node.get("rotation", [0, 0, 0, 1])
            r = (-r[0], -r[1], r[2], r[3])
            s = node.get("scale", [1, 1, 1])
            for prim in g["meshes"][node["mesh"]]["primitives"]:
                at = prim["attributes"]
                pos = accessor(at["POSITION"]).astype(np.float32) * flip
                nrm = accessor(at["NORMAL"]).astype(np.float32) * flip
                uv = accessor(at["TEXCOORD_0"]).astype(np.float32) if "TEXCOORD_0" in at else np.zeros((len(pos), 2), np.float32)
                tan = accessor(at["TANGENT"]).astype(np.float32)[:, :3] * flip if "TANGENT" in at else None
                idx = accessor(prim["indices"]).astype(np.uint32).reshape(-1, 3)[:, [0, 2, 1]].reshape(-1)
                b.add_mesh(pos, nrm, uv, idx, prim["material"], t, r, s, tan)
        for c in node.get("children", []):
            visit(c)

    for n in g["scenes"][g.get("scene", 0)]["nodes"]:
        visit(n)
    return b.finish()
