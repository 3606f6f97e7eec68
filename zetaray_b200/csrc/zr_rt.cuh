// zr_rt.cuh -- ray conventions, hit attributes, material fetch and emissive-light helpers on the device.
//   ZetaRenderPass/Common/RayQuery.hlsli   Hit::FindClosest :15-144, Hit_Emissive :146-299,
//                                          Visibility_Segment :337-406, GetMaterialData :452-524
//   ZetaRenderPass/Common/RT.hlsli:245-262 OffsetRayRTG
//   ZetaRenderPass/Common/LightSource.hlsli emissive triangle decode / sample / Le :46-137, 202-224
// Traversal runs over the library's own 8-wide BVH (zr_scene.cuh). Shadow segments use the
// order-independent rule "occluded iff some triangle other than the target is hit in (tmin, tmax)".
// No textures / alpha test in this build (DESIGN.md scope).
#pragma once
#include "zr_scene.cuh"
#include "zr_bsdf.cuh"

namespace zr
{
constexpr uint32_t UINT32_MAX_ = 0xffffffffu;

namespace RTU
{
    // RT.hlsli:245-262
    ZR_D float3 OffsetRayRTG(float3 pos, float3 geometricNormal)
    {
        const float origin = 1.0f / 32.0f;
        const float float_scale = 1.0f / 65536.0f;
        const float int_scale = 256.0f;
        int ofx = (int)(int_scale * geometricNormal.x), ofy = (int)(int_scale * geometricNormal.y), ofz = (int)(int_scale * geometricNormal.z);
        auto adj = [](float p, int of) { return asfloat((uint32_t)((int)asuint(p) + ((p < 0) ? -of : of))); };
        float3 p_i = f3(adj(pos.x, ofx), adj(pos.y, ofy), adj(pos.z, ofz));
        return f3(fabsf(pos.x) < origin ? pos.x + float_scale * geometricNormal.x : p_i.x,
                  fabsf(pos.y) < origin ? pos.y + float_scale * geometricNormal.y : p_i.y,
                  fabsf(pos.z) < origin ? pos.z + float_scale * geometricNormal.z : p_i.z);
    }
}

constexpr float T_MIN_REFL_RAY = 1e-6f;
constexpr float T_MIN_TR_RAY = 5e-5f;

struct Hit
{
    bool hit; float t; float2 uv; float3 normal; uint32_t ID; uint32_t meshIdx; uint32_t matIdx;
};

struct HitEmissive
{
    bool hit; float t; uint32_t geoIdx, primIdx, emissiveTriIdx; float2 bary; float3 lightPos;
    ZR_D bool HitWasEmissive() const { return emissiveTriIdx != UINT32_MAX_; }
};

// RayQuery.hlsli:213-299 (ToHitInfo) == the attribute part of Hit::FindClosest
ZR_D Hit HitAttributes(const SceneDev& sc, uint32_t meshIdx, uint32_t primIdx, float2 bary, float t)
{
    Hit ret;
    const zr_mesh_instance meshData = LoadInstance(sc, meshIdx);
    ret.hit = true;
    ret.t = t;
    ret.matIdx = meshData.MatIdx;
    ret.meshIdx = meshIdx;
    uint32_t tri = primIdx * 3 + meshData.BaseIdxOffset;
    const VertexD V0 = LoadVertex(sc, __ldg(&sc.indices[tri]) + meshData.BaseVtxOffset);
    const VertexD V1 = LoadVertex(sc, __ldg(&sc.indices[tri + 1]) + meshData.BaseVtxOffset);
    const VertexD V2 = LoadVertex(sc, __ldg(&sc.indices[tri + 2]) + meshData.BaseVtxOffset);
    float4 q = normalize(Math::DecodeNormalized4(meshData.Rotation));
    float3 s = h3(meshData.Scale);
    float tmp = 1 - bary.x - bary.y;
    float2 uv = f2(mad(bary.y, V2.uv.x, tmp * V0.uv.x), mad(bary.y, V2.uv.y, tmp * V0.uv.y));
    uv = f2(mad(bary.x, V1.uv.x, uv.x), mad(bary.x, V1.uv.y, uv.y));
    ret.uv = uv;
    float3 v0_n = Math::DecodeOct32(V0.normal);
    float3 v1_n = Math::DecodeOct32(V1.normal);
    float3 v2_n = Math::DecodeOct32(V2.normal);
    float3 hitNormal = mad(bary.y, v2_n, tmp * v0_n);
    hitNormal = mad(bary.x, v1_n, hitNormal);
    const float3 scaleInv = 1.0f / s;
    hitNormal *= scaleInv;
    hitNormal = Math::RotateVector(hitNormal, q);
    hitNormal = normalize(hitNormal);
    ret.normal = hitNormal;
    ret.ID = RNG::PCG3d(make_uint3(meshIdx, 0u, primIdx)).x;
    return ret;
}

// Hit_Emissive::FindClosest (RayQuery.hlsli:148-205)
ZR_D HitEmissive FindClosestEmissive(const SceneDev& sc, float3 pos, float3 normal, float3 wi, bool transmissive)
{
    HitEmissive ret;
    ret.hit = false;
    ret.emissiveTriIdx = UINT32_MAX_;
    ret.t = 0; ret.geoIdx = 0; ret.primIdx = 0; ret.bary = f2(0, 0); ret.lightPos = f3(0);
    bool wiBackface = dot(normal, wi) <= 0;
    if (wiBackface)
    {
        if (transmissive) normal = -normal;
        else return ret;
    }
    const float3 adjustedOrigin = RTU::OffsetRayRTG(pos, normal);
    RayHit h = TraceClosest(sc, adjustedOrigin, wi, wiBackface ? T_MIN_TR_RAY : T_MIN_REFL_RAY, FLT_MAX_);
    if (h.hit)
    {
        ret.hit = true;
        ret.bary = h.bary;
        ret.t = h.t;
        ret.geoIdx = __ldg(&sc.triMesh[h.tri]);
        ret.primIdx = h.tri - __ldg(&sc.meshFirstTri[ret.geoIdx]);
        const uint32_t baseEmissive = __ldg(&sc.instances[ret.geoIdx].BaseEmissiveTriOffset);
        if (baseEmissive == UINT32_MAX_)
            return ret;
        ret.emissiveTriIdx = baseEmissive + ret.primIdx;
        ret.lightPos = mad(h.t, wi, adjustedOrigin);
    }
    return ret;
}

// Hit::FindClosest<ID, Curr> (RayQuery.hlsli:17-131)
ZR_D Hit FindClosest(const SceneDev& sc, float3 pos, float3 normal, float3 wi, bool transmissive)
{
    Hit ret;
    ret.hit = false;
    ret.ID = UINT32_MAX_;
    ret.t = 0; ret.uv = f2(0, 0); ret.normal = f3(0); ret.meshIdx = 0; ret.matIdx = 0;
    float ndotwi = dot(normal, wi);
    if (ndotwi == 0)
        return ret;
    bool wiBackface = ndotwi < 0;
    if (wiBackface)
    {
        if (!transmissive) return ret;
        normal = -normal;
    }
    const float3 adjustedOrigin = RTU::OffsetRayRTG(pos, normal);
    RayHit h = TraceClosest(sc, adjustedOrigin, wi, wiBackface ? T_MIN_TR_RAY : T_MIN_REFL_RAY, FLT_MAX_);
    if (h.hit)
        {
        const uint32_t mesh = __ldg(&sc.triMesh[h.tri]);
        ret = HitAttributes(sc, mesh, h.tri - __ldg(&sc.meshFirstTri[mesh]), h.bary, h.t);
    }
    return ret;
}

// RayQuery.hlsli:337-406 with APPROXIMATE_EMISSIVE_SHADOW_RAY == 1
ZR_D bool Visibility_Segment(const SceneDev& sc, float3 origin, float3 wi, float rayT, float3 normal, uint32_t triID,
    bool transmissive)
{
    if (triID == UINT32_MAX_) return false;
    if (rayT < 1e-6f) return false;
    float ndotwi = dot(normal, wi);
    if (ndotwi == 0) return false;
    bool wiBackface = ndotwi < 0;
    if (wiBackface)
    {
        if (transmissive) normal = -normal;
        else return false;
    }
    const float3 adjustedOrigin = RTU::OffsetRayRTG(origin, normal);
    const float tMin = 3e-6f;
    const float tMax = Math::PrevFloat32(rayT * 0.999f - Math::NextFloat32(tMin));
    return !TraceAnyExcept(sc, adjustedOrigin, wi, tMin, tMax, triID);
}

// RayQuery.hlsli:337-406 with APPROXIMATE_EMISSIVE_SHADOW_RAY == 0 (the plain path tracer, PathTracer/Params.hlsli:27):
// tMax = rayT, the committed hit is the closest one; visible iff nothing is hit or the closest hit is the light itself.
ZR_D bool Visibility_Segment_Precise(const SceneDev& sc, float3 origin, float3 wi, float rayT, float3 normal, uint32_t triID,
    bool transmissive)
{
    if (triID == UINT32_MAX_) return false;
    if (rayT < 1e-6f) return false;
    float ndotwi = dot(normal, wi);
    if (ndotwi == 0) return false;
    bool wiBackface = ndotwi < 0;
    if (wiBackface)
    {
        if (transmissive) normal = -normal;
        else return false;
    }
    const float3 adjustedOrigin = RTU::OffsetRayRTG(origin, normal);
    const RayHit h = TraceClosest(sc, adjustedOrigin, wi, 3e-6f, rayT);
    if (h.hit)
        return triID == TriID(sc, h.tri);
    return true;
}

// GetMaterialData (RayQuery.hlsli:452-510), textures unsupported (factors only)
template<class SD>
ZR_D bool GetMaterialData(const SceneDev& sc, float3 wo, float eta_curr, Hit& hitInfo, SD& surface, float& eta)
{
    const zr_material mat = LoadMaterial(sc, hitInfo.matIdx);
    const bool hitBackface = dot(wo, hitInfo.normal) < 0;
    eta = BSDF::DEFAULT_ETA_MAT;
    if (!Mat::DoubleSided(mat) && hitBackface)
        return false;
    if (Mat::DoubleSided(mat) && hitBackface)
        hitInfo.normal = -hitInfo.normal;
    float3 baseColor = Mat::GetBaseColorFactor(mat);
    float metallic = Mat::Metallic(mat) ? 1.0f : 0.0f;
    float roughness = Mat::GetSpecularRoughness(mat);
    bool tr = Mat::Transmissive(mat);
    eta = Mat::GetSpecularIOR(mat);
    float trDepth = tr ? Mat::GetTransmissionDepth(mat) : 0;
    float eta_next = eta_curr == BSDF::ETA_AIR ? eta : BSDF::ETA_AIR;
    float subsurface = Mat::ThinWalled(mat) ? to_half(Mat::GetSubsurface(mat)) : 0;
    float coat_weight = Mat::GetCoatWeight(mat);
    float3 coat_color = Mat::GetCoatColor(mat);
    float coat_roughness = Mat::GetCoatRoughness(mat);
    float coat_ior = Mat::GetCoatIOR(mat);
    surface = SD::Init(hitInfo.normal, wo, metallic >= 0.9f, roughness, baseColor, eta_curr, eta_next, tr,
        trDepth, subsurface, coat_weight, coat_color, coat_roughness, coat_ior, sc.rho);
    return true;
}

namespace Light
{
    enum TYPE : uint32_t { NONE = 0, SUN = 1, SKY = 2, EMISSIVE = 3 };
    ZR_D TYPE TypeFromValue(uint32_t x) { return x <= 2 ? (TYPE)x : EMISSIVE; }

    ZR_D float3 DecodeEmissiveTriV1(const zr_emissive_tri& tri)
    {
        float2 v = f2((float)tri.V0V1[0] / 65535.0f, (float)tri.V0V1[1] / 65535.0f);
        float3 decoded = Math::DecodeUnitVector(v);
        return mad(decoded, zr_f16_to_f32(tri.EdgeLengths[0]), f3(tri.Vtx0[0], tri.Vtx0[1], tri.Vtx0[2]));
    }
    ZR_D float3 DecodeEmissiveTriV2(const zr_emissive_tri& tri)
    {
        float2 v = f2((float)tri.V0V2[0] / 65535.0f, (float)tri.V0V2[1] / 65535.0f);
        float3 decoded = Math::DecodeUnitVector(v);
        return mad(decoded, zr_f16_to_f32(tri.EdgeLengths[1]), f3(tri.Vtx0[0], tri.Vtx0[1], tri.Vtx0[2]));
    }
    ZR_D bool IsDoubleSided(const zr_emissive_tri& tri) { return tri.PackedA & (1u << 25); }
    ZR_D float3 Vtx0(const zr_emissive_tri& tri) { return f3(tri.Vtx0[0], tri.Vtx0[1], tri.Vtx0[2]); }

    // Le_EmissiveTriangle (LightSource.hlsli:202-224), no emissive textures
    ZR_D float3 Le_EmissiveTriangle(const zr_emissive_tri& tri)
    {
        const float3 emissiveFactor = Math::UnpackRGB8(tri.PackedA);
        const float emissiveStrength = zr_f16_to_f32((uint16_t)(tri.PackedB >> 16));
        float3 le = emissiveFactor * emissiveStrength;
        if (Math::Luminance(le) == 0)
            return f3(0.0f);
        return le;
    }

    struct AliasTableSample { uint32_t idx; float pdf; };
    ZR_D AliasTableSample SampleAlias(const zr_alias_entry* table, uint32_t numEmissiveTriangles, RNG& rng)
    {
        AliasTableSample ret;
        uint32_t u0 = rng.UniformUintBounded(numEmissiveTriangles);
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(table + u0));
        zr_alias_entry s; s.CachedP_Orig = asfloat(raw.x); s.CachedP_Alias = asfloat(raw.y); s.P_Curr = asfloat(raw.z); s.Alias = raw.w;
        if (rng.Uniform() < s.P_Curr) { ret.pdf = s.CachedP_Orig; ret.idx = u0; return ret; }
        ret.pdf = s.CachedP_Alias;
        ret.idx = s.Alias;
        return ret;
    }

    // One light sample for next-event estimation, from either source (ReSTIR_PT_NEE.hlsli:217-248 /
    // ReSTIR_DI_Temporal.hlsl:119-147): a presampled set of this thread group, or alias table + uniform point on the triangle.
    struct LightSample { float3 pos, normal, le; float2 bary; float pdf; uint32_t idx, ID; bool twoSided; };
    struct EmissiveTriSample { float3 pos, normal; float2 bary; float pdf; };
    ZR_D EmissiveTriSample SampleEmissiveTri(float3 pos, const zr_emissive_tri& tri, RNG& rng, bool reverseNormalIfTwoSided = true)
    {
        EmissiveTriSample ret;
        float2 u = rng.Uniform2D();
        ret.bary = Sampling::UniformSampleTriangle(u);
        const float3 vtx0 = Vtx0(tri);
        const float3 vtx1 = DecodeEmissiveTriV1(tri);
        const float3 vtx2 = DecodeEmissiveTriV2(tri);
        ret.pos = (1.0f - ret.bary.x - ret.bary.y) * vtx0 + ret.bary.x * vtx1 + ret.bary.y * vtx2;
        ret.normal = cross(vtx1 - vtx0, vtx2 - vtx0);
        bool normalIs0 = dot(ret.normal, ret.normal) == 0;
        float twoArea = length(ret.normal);
        ret.pdf = normalIs0 ? 0.0f : 2.0f / twoArea;
        ret.normal = normalIs0 ? ret.normal : ret.normal / twoArea;
        ret.normal = reverseNormalIfTwoSided && IsDoubleSided(tri) && dot(pos - ret.pos, ret.normal) < 0 ? -ret.normal : ret.normal;
        return ret;
    }

    // advanceRng: the path tracer keeps the RNG stream identical with and without presampled sets (":235 Deterministic RNG
    // state regardless of USE_PRESAMPLED_SETS"); ReSTIR DI does not.
    ZR_D LightSample SampleLight(const SceneDev& sc, float3 pos, uint32_t sampleSetIdx, RNG& rng, bool advanceRng)
    {
        LightSample ls;
        if (sc.sampleSetSize > 0)
        {
            const uint32_t u = rng.UniformUintBounded_Faster(sc.sampleSetSize);
            const zr_presampled_tri* p = sc.sampleSets + (size_t)sampleSetIdx * sc.sampleSetSize + u;
            // 40-byte records are 8-byte aligned: five 64-bit loads
            const uint2* q = reinterpret_cast<const uint2*>(p);
            const uint2 q0 = __ldg(q), q1 = __ldg(q + 1), q2 = __ldg(q + 2), q3 = __ldg(q + 3), c = __ldg(q + 4);
            const uint4 a = make_uint4(q0.x, q0.y, q1.x, q1.y);                  // pos.xyz, normal
            const uint4 b = make_uint4(q2.x, q2.y, q3.x, q3.y);                  // pdf, ID, idx, bary; c = le.xyz (half), twoSided
            ls.pos = f3(asfloat(a.x), asfloat(a.y), asfloat(a.z));
            ls.normal = Math::DecodeOct32(a.w);
            ls.bary = Math::DecodeUNorm2(b.w);
            ls.le = f3(zr_f16_to_f32((uint16_t)(c.x & 0xffff)), zr_f16_to_f32((uint16_t)(c.x >> 16)), zr_f16_to_f32((uint16_t)(c.y & 0xffff)));
            ls.pdf = asfloat(b.x); ls.ID = b.y; ls.idx = b.z;
            ls.twoSided = (c.y >> 16) != 0;
            if (ls.twoSided && dot(pos - ls.pos, ls.normal) < 0)
                ls.normal = -ls.normal;
            if (advanceRng)
                rng.Uniform3D();
        }
        else
        {
            AliasTableSample entry = SampleAlias(sc.aliasTable, sc.numEmissives, rng);
            const zr_emissive_tri& tri = sc.emissives[entry.idx];
            const EmissiveTriSample ts = SampleEmissiveTri(pos, tri, rng);
            ls.pos = ts.pos; ls.normal = ts.normal; ls.bary = ts.bary;
            ls.le = Le_EmissiveTriangle(tri);
            ls.pdf = entry.pdf * ts.pdf; ls.idx = entry.idx; ls.ID = tri.ID; ls.twoSided = IsDoubleSided(tri);
        }
        return ls;
    }
}
// Common/LightVoxelGrid.hlsli:8-69
namespace LVG
{
    ZR_D uint32_t FlattenVoxelIndex(uint32_t x, uint32_t y, uint32_t z, uint32_t dx, uint32_t dy) { return z * dx * dy + y * dx + x; }

    ZR_D float3 VoxelCenter(int vx, int vy, int vz, int dx, int dy, int dz, float3 voxelExtents, const float viewInv[3][4], float offset_y)
    {
        const int hx = dx >> 1, hy = dy >> 1, hz = dz >> 1;
        int cx = vx - hx, cy = vy - hy, cz = vz - hz;
        cx += vx < hx ? 1 : 0; cy += vy < hy ? 1 : 0; cz += vz < hz ? 1 : 0;
        cy *= -1;       // voxel space Y points in the opposite direction of camera space Y
        const float3 corner = f3((float)(cx * 2), (float)(cy * 2), (float)(cz * 2)) * voxelExtents;
        const float3 s = f3(Math::SignNotZero((float)cx), Math::SignNotZero((float)cy), Math::SignNotZero((float)cz));
        float3 centerV = corner + voxelExtents * s;
        centerV.y += offset_y;
        return Math::mul3x4(viewInv, centerV);
    }

    ZR_D bool MapPosToVoxel(float3 pos, int dx, int dy, int dz, float3 voxelExtents, const float view[3][4], int& ox, int& oy, int& oz, float offset_y)
    {
        float3 posV = Math::mul3x4(view, pos);
        posV.y -= offset_y;
        const int hx = dx >> 1, hy = dy >> 1, hz = dz >> 1;
        float3 voxel = f3(floorf(fabsf(posV.x) / (2 * voxelExtents.x)), floorf(fabsf(posV.y) / (2 * voxelExtents.y)), floorf(fabsf(posV.z) / (2 * voxelExtents.z)));
        if (voxel.x >= (float)hx || voxel.y >= (float)hy || voxel.z >= (float)hz)
            return false;
        voxel = voxel * f3(Math::SignNotZero(posV.x), Math::SignNotZero(posV.y), Math::SignNotZero(posV.z));
        voxel.y *= -1;
        ox = (int)voxel.x + hx - (posV.x < 0 ? 1 : 0);
        oy = (int)voxel.y + hy - (posV.y >= 0 ? 1 : 0);
        oz = (int)voxel.z + hz - (posV.z < 0 ? 1 : 0);
        return true;
    }
}

namespace LVG
{
    // LightVoxelGrid.hlsli:54-68 (32-byte records, 16-byte aligned: two 128-bit loads)
    struct VoxelLight { float3 pos, normal, le; float pdf; uint32_t ID; bool twoSided; };
    ZR_D bool Sample(const SceneDev& sc, float3 pos, float3 voxelExtents, float offset_y, const float view[3][4], VoxelLight& out, RNG& rng)
    {
        const float3 u = rng.Uniform3D();
        const float3 posJittered = pos + (u * 2.0f - 1.0f) * voxelExtents;
        int vx, vy, vz;
        if (!MapPosToVoxel(posJittered, (int)sc.lvgDim[0], (int)sc.lvgDim[1], (int)sc.lvgDim[2], voxelExtents, view, vx, vy, vz, offset_y))
            return false;
        const uint32_t start = FlattenVoxelIndex((uint32_t)vx, (uint32_t)vy, (uint32_t)vz, sc.lvgDim[0], sc.lvgDim[1]) * 64u;
        const uint32_t k = rng.UniformUintBounded_Faster(64u);
        const uint4* q = reinterpret_cast<const uint4*>(sc.lvg + start + k);
        const uint4 a = __ldg(q), b = __ldg(q + 1);
        out.pos = f3(asfloat(a.x), asfloat(a.y), asfloat(a.z));
        out.normal = Math::DecodeOct32(a.w);
        out.pdf = asfloat(b.x); out.ID = b.y;
        out.le = f3(zr_f16_to_f32((uint16_t)(b.z & 0xffff)), zr_f16_to_f32((uint16_t)(b.z >> 16)), zr_f16_to_f32((uint16_t)(b.w & 0xffff)));
        out.twoSided = (b.w >> 16) != 0;
        return true;
    }
}
} // namespace zr
