// zr_scene.cuh -- device-side scene access and ray traversal.
//
// The reference traces against a driver-built DXR TLAS with inline RayQuery
// (ZetaRenderPass/Common/RayQuery.hlsli:42-53). Here the acceleration structure is ours: an 8-wide
// BVH with child boxes quantised to 8 bits per plane relative to the node's origin/exponent
// (80-byte nodes, 5 x 128-bit loads), leaves of <= 3 world-space triangles stored as 3 x float4
// {v0 | triGlobal, e1, e2}. No OptiX, no RT cores.
//
// Hit rule (shared with the oracle's brute force): Moller-Trumbore on (v0, e1, e2), accept
// tmin < t < tmax, closest t wins, ties go to the lowest global triangle index -- so the result is
// independent of traversal order.
#pragma once
#include "zr_common.cuh"
#include "zr_bvh.h"

namespace zr
{
struct SceneDev
{
    const zr_vertex* vertices;
    const uint32_t* indices;
    const zr_mesh_instance* instances;
    const zr_material* materials;
    const zr_emissive_tri* emissives;
    const zr_alias_entry* aliasTable;
    const uint4* nodes;         // BVH8Node as 5 x uint4
    const float4* tris;         // 3 x float4 per triangle, BVH leaf order
    const uint32_t* triMesh;    // mesh (instance) index per global triangle
    const uint32_t* meshFirstTri;
    const uint16_t* rho;        // 64 x 32 x 16 R16_UNORM directional-albedo table
    uint32_t numInstances;
    uint32_t numEmissives;
    uint32_t numTris;
    // presampled emissive sets (PresampleEmissives.hlsl); sampleSetSize == 0: lights are sampled through the alias table
    const zr_presampled_tri* sampleSets;
    uint32_t numSampleSets, sampleSetSize;
    // light voxel grid (BuildLightVoxelGrid.hlsl); lvg == nullptr: off
    const zr_voxel_sample* lvg;
    uint32_t lvgDim[3];
    float lvgExtents[3];
    float lvgOffsetY;
};

struct RayHit { bool hit; float t; float2 bary; uint32_t tri; };

ZR_D bool TriHit(float3 o, float3 d, float3 v0, float3 e1, float3 e2, float tmin, float tmax, float& t, float& u, float& v)
{
    float3 pvec = cross(d, e2);
    float det = dot(e1, pvec);
    if (det == 0.0f) return false;
    float inv = 1.0f / det;
    float3 tvec = o - v0;
    u = dot(tvec, pvec) * inv;
    if (!(u >= 0.0f) || u > 1.0f) return false;
    float3 qvec = cross(tvec, e1);
    v = dot(d, qvec) * inv;
    if (!(v >= 0.0f) || u + v > 1.0f) return false;
    t = dot(e2, qvec) * inv;
    return t > tmin && t < tmax;
}

ZR_D uint32_t TriPrim(const SceneDev& sc, uint32_t tri) { return tri - __ldg(&sc.meshFirstTri[__ldg(&sc.triMesh[tri])]); }
ZR_D uint32_t TriID(const SceneDev& sc, uint32_t tri)
{
    const uint32_t mesh = __ldg(&sc.triMesh[tri]);
    return RNG::PCG3d(make_uint3(mesh, 0u, tri - __ldg(&sc.meshFirstTri[mesh]))).x;
}

// Mode: 0 = closest hit, 1 = any hit whose ID differs from ignoreID (UINT32_MAX = none ignored)
template<int Mode>
ZR_F1 RayHit Traverse(const SceneDev& sc, float3 o, float3 d, float tmin, float tmax, uint32_t ignoreID)
{
    RayHit best;
    best.hit = false; best.t = tmax; best.bary = f2(0, 0); best.tri = 0xffffffffu;
    // Degenerate rays hit nothing under the hit rule (a zero direction makes every determinant 0, a NaN direction or origin makes
    // every barycentric NaN), but they pass every slab test below (0 * inf and NaN drop out of fminf / fmaxf), i.e. they would
    // sweep the whole tree: one such ray per ~1500 pixels comes out of the path tracer's BSDF-sampled emissive-hit query on
    // transmissive surfaces (wi = 0 when the sampler returns pdf 0), and such a ray holds its whole 1024-thread block
    // for a full sweep of the tree. They start with an empty stack. One translation
    // unit, rgi.cu, opts out (ZR_NO_DEGENERATE_RAY_EARLY_OUT): with this cut compiled in -- as an empty stack or as an early return,
    // both tried -- k_rgi runs with half the active lanes per warp (see rgi.cu).
    const bool degenerate = (d.x == 0.0f && d.y == 0.0f && d.z == 0.0f) || d.x != d.x || d.y != d.y || d.z != d.z ||
        o.x != o.x || o.y != o.y || o.z != o.z;
#if defined(ZR_DEGENERATE_RAY_RETURN)          /* A/B switches for measurements only */
    if (degenerate) return best;
#endif
    const float3 invd = f3(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
    uint32_t stack[BVH_STACK_ENTRIES];
    int sp = 0;
    stack[sp++] = 0;
#if !defined(ZR_NO_DEGENERATE_RAY_EARLY_OUT) && !defined(ZR_DEGENERATE_RAY_RETURN)
    sp = degenerate ? 0 : sp;
#endif
    while (sp > 0)
    {
        const uint32_t nodeIdx = stack[--sp];
#ifdef ZR_TRAVERSE_STATS        /* host test builds only (tests/hostsim): node visits / triangle tests per ray */
        ZR_TRAVERSE_STATS.nodes++;
#endif
        const uint4* np = sc.nodes + (size_t)nodeIdx * 5;
        const uint4 n0 = __ldg(np + 0);
        const uint4 n1 = __ldg(np + 1);
        const uint4 n2 = __ldg(np + 2);
        const uint4 n3 = __ldg(np + 3);
        const uint4 n4 = __ldg(np + 4);
        const float3 p = f3(asfloat(n0.x), asfloat(n0.y), asfloat(n0.z));
        const float sx = asfloat((n0.w & 0xffu) << 23), sy = asfloat(((n0.w >> 8) & 0xffu) << 23), sz = asfloat(((n0.w >> 16) & 0xffu) << 23);
        const uint32_t childBase = n1.x, triBase = n1.y;
        const uint32_t metaLo = n1.z, metaHi = n1.w;
        // qlo[0] = n2.xy, qlo[1] = n2.zw, qlo[2] = n3.xy, qhi[0] = n3.zw, qhi[1] = n4.xy, qhi[2] = n4.zw
        const uint32_t q[12] = { n2.x, n2.y, n2.z, n2.w, n3.x, n3.y, n3.z, n3.w, n4.x, n4.y, n4.z, n4.w };
        // children are visited far-to-near pushed, so near ones pop first
        float childT[8];
        uint32_t childNode[8];
        int nPush = 0;
#pragma unroll
        for (int c = 0; c < 8; c++)
        {
            const uint32_t meta = ((c < 4 ? metaLo : metaHi) >> ((c & 3) * 8)) & 0xffu;
            if (meta == 0) continue;
            const int w = c >> 2, sh = (c & 3) * 8;
            const float lox = fmaf((float)((q[0 + w] >> sh) & 0xffu), sx, p.x);
            const float loy = fmaf((float)((q[2 + w] >> sh) & 0xffu), sy, p.y);
            const float loz = fmaf((float)((q[4 + w] >> sh) & 0xffu), sz, p.z);
            const float hix = fmaf((float)((q[6 + w] >> sh) & 0xffu), sx, p.x);
            const float hiy = fmaf((float)((q[8 + w] >> sh) & 0xffu), sy, p.y);
            const float hiz = fmaf((float)((q[10 + w] >> sh) & 0xffu), sz, p.z);
            const float tx0 = (lox - o.x) * invd.x, tx1 = (hix - o.x) * invd.x;
            const float ty0 = (loy - o.y) * invd.y, ty1 = (hiy - o.y) * invd.y;
            const float tz0 = (loz - o.z) * invd.z, tz1 = (hiz - o.z) * invd.z;
            const float tn = fmaxf(fmaxf(fminf(tx0, tx1), fminf(ty0, ty1)), fmaxf(fminf(tz0, tz1), tmin));
            const float tf = fminf(fminf(fmaxf(tx0, tx1), fmaxf(ty0, ty1)), fminf(fmaxf(tz0, tz1), best.t)) * 1.0000005f;
            if (!(tn <= tf)) continue;
            if (meta & 0x20u)
            {
                childT[nPush] = tn;
                childNode[nPush] = childBase + (meta & 0x1fu);
                nPush++;
            }
            else
            {
                const uint32_t nt = meta >> 6;
                const uint32_t first = triBase + (meta & 0x1fu);
                for (uint32_t k = 0; k < nt; k++)
                {
                    const float4* tp = sc.tris + (size_t)(first + k) * 3;
                    const float4 a = __ldg(tp), b = __ldg(tp + 1), cc = __ldg(tp + 2);
                    float t, u, v;
#ifdef ZR_TRAVERSE_STATS
                    ZR_TRAVERSE_STATS.tris++;
#endif
                    if (TriHit(o, d, f3(a.x, a.y, a.z), f3(b.x, b.y, b.z), f3(cc.x, cc.y, cc.z), tmin, tmax, t, u, v))
                    {
                        const uint32_t triGlobal = asuint(a.w);
                        if (Mode == 1)
                        {
                            if (ignoreID == 0xffffffffu || TriID(sc, triGlobal) != ignoreID)
                            {
                                best.hit = true; best.t = t; best.bary = f2(u, v); best.tri = triGlobal;
                                return best;
                            }
                        }
                        else if (!best.hit || t < best.t || (t == best.t && triGlobal < best.tri))
                        {
                            best.hit = true; best.t = t; best.bary = f2(u, v); best.tri = triGlobal;
                        }
                    }
                }
            }
        }
        // push far-to-near (insertion sort, <= 8 entries)
        for (int i = 1; i < nPush; i++)
        {
            float kt = childT[i]; uint32_t kn = childNode[i];
            int j = i - 1;
            while (j >= 0 && childT[j] < kt) { childT[j + 1] = childT[j]; childNode[j + 1] = childNode[j]; j--; }
            childT[j + 1] = kt; childNode[j + 1] = kn;
        }
        for (int i = 0; i < nPush; i++)
            if (sp < BVH_STACK_ENTRIES) stack[sp++] = childNode[i];      // never drops: scene creation checked BvhBuild::maxStack
    }
    return best;
}

ZR_D RayHit TraceClosest(const SceneDev& sc, float3 o, float3 d, float tmin, float tmax)
{
    return Traverse<0>(sc, o, d, tmin, tmax, 0xffffffffu);
}
ZR_D bool TraceAnyExcept(const SceneDev& sc, float3 o, float3 d, float tmin, float tmax, uint32_t ignoreID)
{
    return Traverse<1>(sc, o, d, tmin, tmax, ignoreID).hit;
}

// ---- material getters (ZetaCore/Core/Material.h:296-427) ----
namespace Mat
{
    ZR_D bool DoubleSided(const zr_material& m) { return m.CoatColor_Flags & (1u << 25); }
    ZR_D bool Metallic(const zr_material& m) { return m.CoatColor_Flags & (1u << 24); }
    ZR_D bool Transmissive(const zr_material& m) { return m.CoatColor_Flags & (1u << 26); }
    ZR_D bool ThinWalled(const zr_material& m) { return m.CoatColor_Flags & (1u << 29); }
    ZR_D float3 GetBaseColorFactor(const zr_material& m) { return Math::UnpackRGB8(m.BaseColorFactor); }
    ZR_D float3 GetCoatColor(const zr_material& m) { return Math::UnpackRGB8(m.CoatColor_Flags); }
    ZR_D float3 GetEmissiveFactor(const zr_material& m) { return Math::UnpackRGB8(m.EmissiveFactor_NormalScale); }
    ZR_D float GetCoatIOR(const zr_material& m) { return mad(1.5f / 255.0f, (float)((m.EmissiveTex_AlphaCutoff_CoatIOR >> 24) & 0xff), 1.0f); }
    ZR_D float GetSpecularRoughness(const zr_material& m) { return Math::UNorm8ToFloat((m.MRTex_SpecRoughness_CoatRoughness >> 16) & 0xff); }
    ZR_D float GetCoatRoughness(const zr_material& m) { return Math::UNorm8ToFloat((m.MRTex_SpecRoughness_CoatRoughness >> 24) & 0xff); }
    ZR_D float GetEmissiveStrength(const zr_material& m) { return zr_f16_to_f32((uint16_t)(m.EmissiveStrength_IOR & 0xffff)); }
    ZR_D float GetSpecularIOR(const zr_material& m) { return mad(1.5f / 65535.0f, (float)(m.EmissiveStrength_IOR >> 16), 1.0f); }
    ZR_D float GetTransmissionDepth(const zr_material& m) { return zr_f16_to_f32((uint16_t)(m.NormalTex_TrDepth >> 16)); }
    ZR_D float GetSubsurface(const zr_material& m) { return Math::UNorm8ToFloat((m.BaseColorTex_Subsurf_CoatWeight >> 16) & 0xff); }
    ZR_D float GetCoatWeight(const zr_material& m) { return Math::UNorm8ToFloat((m.BaseColorTex_Subsurf_CoatWeight >> 24) & 0xff); }
}

ZR_D zr_material LoadMaterial(const SceneDev& sc, uint32_t idx)
{
    const uint4* p = reinterpret_cast<const uint4*>(sc.materials + idx);
    const uint4 a = __ldg(p), b = __ldg(p + 1);
    zr_material m;
    m.BaseColorFactor = a.x; m.BaseColorTex_Subsurf_CoatWeight = a.y; m.NormalTex_TrDepth = a.z; m.MRTex_SpecRoughness_CoatRoughness = a.w;
    m.EmissiveFactor_NormalScale = b.x; m.EmissiveStrength_IOR = b.y; m.EmissiveTex_AlphaCutoff_CoatIOR = b.z; m.CoatColor_Flags = b.w;
    return m;
}

ZR_D zr_mesh_instance LoadInstance(const SceneDev& sc, uint32_t idx)
{
    const uint4* p = reinterpret_cast<const uint4*>(sc.instances + idx);
    uint4 v[4] = { __ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3) };
    zr_mesh_instance m;
    memcpy(&m, v, sizeof(m));
    return m;
}

ZR_D float3 h3(const uint16_t h[3]) { return f3(zr_f16_to_f32(h[0]), zr_f16_to_f32(h[1]), zr_f16_to_f32(h[2])); }

struct VertexD { float3 pos; float2 uv; uint32_t normal; uint32_t tangent; };
ZR_D VertexD LoadVertex(const SceneDev& sc, uint32_t idx)
{
    const uint32_t* p = reinterpret_cast<const uint32_t*>(sc.vertices + idx);
    VertexD v;
    v.pos = f3(asfloat(__ldg(p)), asfloat(__ldg(p + 1)), asfloat(__ldg(p + 2)));
    v.uv = f2(asfloat(__ldg(p + 3)), asfloat(__ldg(p + 4)));
    v.normal = __ldg(p + 5);
    v.tangent = __ldg(p + 6);
    return v;
}

// host side (scene.cu)
struct SceneHostInfo { uint32_t numNodes, numTris, maxDepth, bytes, maxStack; };
} // namespace zr

struct zr_scene
{
    zr::SceneDev dev{};
    zr::SceneHostInfo info{};
    void* allocs[16] = { 0 };
    int numAllocs = 0;
    zr_alias_entry* d_alias = nullptr;
    float* d_power = nullptr;
    uint32_t* d_aliasScratch = nullptr;
    bool aliasBuilt = false;
    zr_presampled_tri* d_sampleSets = nullptr;
    bool samplesValid = false;      // zr_presample_emissives ran since the sets were (re)configured
    zr_voxel_sample* d_lvg = nullptr;
    bool lvgValid = false;          // zr_build_light_voxel_grid ran since the grid was (re)configured
};
