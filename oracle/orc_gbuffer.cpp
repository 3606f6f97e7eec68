// ORACLE -- test infrastructure, not product code (see orc_math.h header).
//
// CPU restatement of the G-buffer pass (SURVEY 8a-7):
//   ZetaRenderPass/GBuffer/GBufferRT_Inline.hlsl  TracePrimaryHit :72-198, main :205-287
//   ZetaRenderPass/GBuffer/GBufferRT.hlsli        ApplyTextureMaps :178-282, WriteToGBuffers :102-176
//   ZetaRenderPass/Common/GBuffers.hlsli          EncodeMetallic :52-68
// Parity unpinned (no reference tests). No textures / alpha test (DESIGN.md scope).
#include "orc_api.h"
#include "orc_scene.h"
#include <thread>
#include <functional>

using namespace orc;

RhoLUT orc::g_rho;

namespace
{
    void parallel_rows(uint32_t H, int nthreads, const std::function<void(uint32_t, uint32_t)>& fn)
    {
        if (nthreads <= 1) { fn(0, H); return; }
        std::vector<std::thread> th;
        uint32_t per = (H + nthreads - 1) / nthreads;
        for (int i = 0; i < nthreads; i++)
        {
            uint32_t y0 = i * per, y1 = y0 + per > H ? H : y0 + per;
            if (y0 >= y1) break;
            th.emplace_back(fn, y0, y1);
        }
        for (auto& t : th) t.join();
    }
}

extern "C"
{
    void orc_set_rho_lut(const uint16_t* data) { g_rho.data = data; }

    void* orc_scene_create(const zr_vertex* v, const uint32_t* idx, const zr_mesh_instance* inst, uint32_t numInst,
        const uint32_t* instNumTris, const zr_material* mats, const zr_emissive_tri* em, uint32_t numEm,
        const zr_alias_entry* alias)
    {
        Scene* s = new Scene();
        s->vertices = v; s->indices = idx; s->instances = inst; s->numInstances = numInst; s->materials = mats;
        s->emissives = em; s->numEmissives = numEm; s->aliasTable = alias;
        s->Build(instNumTris);
        return s;
    }
    void orc_scene_destroy(void* s) { delete (Scene*)s; }
    uint32_t orc_scene_num_tris(void* s) { return (uint32_t)((Scene*)s)->v0.size(); }
    // world-space triangles as the traversal sees them: 9 floats per triangle (v0, e1, e2)
    void orc_scene_get_tris(void* s_, float* out)
    {
        Scene* s = (Scene*)s_;
        for (size_t i = 0; i < s->v0.size(); i++)
        {
            float3 a = s->v0[i], b = s->e1[i], c = s->e2[i];
            float* o = out + 9 * i;
            o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = b.x; o[4] = b.y; o[5] = b.z; o[6] = c.x; o[7] = c.y; o[8] = c.z;
        }
    }
    // rays: n x {o.xyz, tmin, d.xyz, tmax}; hits: n x {t, u, v, tri(bits)}
    void orc_trace_closest(void* s_, const float* rays, uint32_t n, float* hits)
    {
        Scene* s = (Scene*)s_;
        for (uint32_t i = 0; i < n; i++)
        {
            const float* r = rays + 8 * i;
            RayHit h = s->Closest(f3(r[0], r[1], r[2]), f3(r[4], r[5], r[6]), r[3], r[7]);
            float* o = hits + 4 * i;
            o[0] = h.hit ? h.t : FLT_MAX_; o[1] = h.bary.x; o[2] = h.bary.y; o[3] = asfloat(h.tri);
        }
    }
    void orc_trace_any(void* s_, const float* rays, uint32_t n, uint32_t* flags)
    {
        Scene* s = (Scene*)s_;
        for (uint32_t i = 0; i < n; i++)
        {
            const float* r = rays + 8 * i;
            flags[i] = s->AnyHitExcept(f3(r[0], r[1], r[2]), f3(r[4], r[5], r[6]), r[3], r[7], UINT32_MAX_) ? 1u : 0u;
        }
    }

    // core: uint4[w*h], depth: float[w*h], me: uint2[w*h], coat: uint2[w*h], tridiff: 6 x u32 [w*h] or null
    void orc_gbuffer(void* scene_, const zr_frame_constants* fc, uint32_t* core_, float* depthPlane, uint32_t* me_, uint32_t* coat_,
        uint32_t* tridiff, int nthreads)
    {
        uint4* core = (uint4*)core_;
        uint2* me = (uint2*)me_;
        uint2* coat = (uint2*)coat_;
        const Scene& sc = *(Scene*)scene_;
        const uint32_t W = fc->RenderWidth, H = fc->RenderHeight;
        auto rows = [&](uint32_t y0, uint32_t y1)
        {
            for (uint32_t y = y0; y < y1; y++)
                for (uint32_t x = 0; x < W; x++)
                {
                    const size_t idx = (size_t)y * W + x;
                    float2 lensSample = f2(0, 0);
                    const float2 renderDim = f2((float)W, (float)H);
                    const float2 jitter = f2(fc->CurrCameraJitter[0], fc->CurrCameraJitter[1]);
                    // RT::GeneratePinholeCameraRay_CS (RT.hlsli:234-243)
                    float2 uv = (f2((float)x, (float)y) + 0.5f + jitter) / renderDim;
                    float2 ndc = Math::NDCFromUV(uv);
                    float3 rayDirCS = f3(ndc.x * fc->AspectRatio * fc->TanHalfFOV, ndc.y * fc->TanHalfFOV, 1);
                    float3 rayOrigin = f3(fc->CameraPos[0], fc->CameraPos[1], fc->CameraPos[2]);
                    const float3 bx = f3(fc->CurrView[0][0], fc->CurrView[0][1], fc->CurrView[0][2]);
                    const float3 by = f3(fc->CurrView[1][0], fc->CurrView[1][1], fc->CurrView[1][2]);
                    const float3 bz = f3(fc->CurrView[2][0], fc->CurrView[2][1], fc->CurrView[2][2]);
                    if (fc->DoF)
                    {
                        uint3 h = RNG::PCG3d(uint3{ x, y, x });
                        RNG rng = RNG::Init(h.z, h.y, fc->FrameNum);
                        lensSample = Sampling::UniformSampleDiskConcentric(rng.Uniform2D());
                        lensSample = lensSample * fc->LensRadius;
                        rayOrigin += mad(lensSample.x, bx, lensSample.y * by);
                        float3 focalPoint = fc->FocusDepth * rayDirCS;
                        rayDirCS = focalPoint - f3(lensSample.x, lensSample.y, 0);
                    }
                    float3 rayDir = mad(rayDirCS.x, bx, mad(rayDirCS.y, by, rayDirCS.z * bz));
                    rayDir = normalize(rayDir);

                    RayHit h = sc.Closest(rayOrigin, rayDir, 0.0f, FLT_MAX_);
                    if (!h.hit)
                    {
                        float3 prevCameraPos = f3(fc->PrevViewInv[0][3], fc->PrevViewInv[1][3], fc->PrevViewInv[2][3]);
                        float3 motion = f3(fc->CameraPos[0], fc->CameraPos[1], fc->CameraPos[2]) - prevCameraPos;
                        float2 motionNDC = motion.z > 0 ? f2(motion.x, motion.y) / (motion.z * fc->TanHalfFOV) : f2(0, 0);
                        motionNDC.x /= fc->AspectRatio;
                        float2 motionUV = Math::UVFromNDC(motionNDC);
                        core[idx] = uint4{ asuint(FLT_MAX_), 0u, 0u, 4u };
                        depthPlane[idx] = FLT_MAX_;
                        me[idx] = uint2{ pack_snorm16x2(motionUV), 0u };
                        coat[idx] = uint2{ 0u, 0u };
                        if (tridiff) for (int k = 0; k < 6; k++) tridiff[idx * 6 + k] = 0;
                        continue;
                    }
                    const uint32_t meshIdx = sc.triMesh[h.tri], primIdx = sc.triPrim[h.tri];
                    const zr_mesh_instance& meshData = sc.instances[meshIdx];
                    const float2 bary = h.bary;
                    uint32_t tri = primIdx * 3 + meshData.BaseIdxOffset;
                    const zr_vertex& V0 = sc.vertices[sc.indices[tri] + meshData.BaseVtxOffset];
                    const zr_vertex& V1 = sc.vertices[sc.indices[tri + 1] + meshData.BaseVtxOffset];
                    const zr_vertex& V2 = sc.vertices[sc.indices[tri + 2] + meshData.BaseVtxOffset];
                    float4 q = normalize(Math::DecodeNormalized4(meshData.Rotation));
                    const float3 scale = Scene::h3(meshData.Scale);
                    const float3 translation = f3(meshData.Translation[0], meshData.Translation[1], meshData.Translation[2]);
                    const float2 uv0 = f2(V0.uv[0], V0.uv[1]), uv1 = f2(V1.uv[0], V1.uv[1]), uv2 = f2(V2.uv[0], V2.uv[1]);
                    float3 v0_n = Math::DecodeOct32((uint32_t)V0.normal[0] | ((uint32_t)V0.normal[1] << 16));
                    float3 v1_n = Math::DecodeOct32((uint32_t)V1.normal[0] | ((uint32_t)V1.normal[1] << 16));
                    float3 v2_n = Math::DecodeOct32((uint32_t)V2.normal[0] | ((uint32_t)V2.normal[1] << 16));
                    float3 normal = v0_n + bary.x * (v1_n - v0_n) + bary.y * (v2_n - v0_n);
                    const float3 scaleInv = 1.0f / scale;
                    normal *= scaleInv;
                    normal = Math::RotateVector(normal, q);
                    normal = normalize(normal);

                    const float3 p0 = f3(V0.pos[0], V0.pos[1], V0.pos[2]), p1 = f3(V1.pos[0], V1.pos[1], V1.pos[2]), p2 = f3(V2.pos[0], V2.pos[1], V2.pos[2]);
                    float3 v0W = Math::TransformTRS(p0, translation, q, scale);
                    float3 v1W = Math::TransformTRS(p1, translation, q, scale);
                    float3 v2W = Math::TransformTRS(p2, translation, q, scale);
                    float3 n0W = normalize(Math::RotateVector(v0_n * scaleInv, q));
                    float3 n1W = normalize(Math::RotateVector(v1_n * scaleInv, q));
                    float3 n2W = normalize(Math::RotateVector(v2_n * scaleInv, q));
                    Math::TriDifferentials td = Math::TriDifferentials::Compute(v0W, v1W, v2W, n0W, n1W, n2W, uv0, uv1, uv2);

                    // motion vector
                    float3 hitPos = mad(rayDir, h.t, rayOrigin);
                    float3 posL = Math::InverseTransformTRS(hitPos, translation, q, scale);
                    float3 prevTranslation = translation - Scene::h3(meshData.dTranslation);
                    float4 q_prev = normalize(Math::DecodeNormalized4(meshData.PrevRotation));
                    float3 pos_prev = Math::TransformTRS(posL, prevTranslation, q_prev, Scene::h3(meshData.PrevScale));
                    float3 posV_prev = Math::mul3x4(fc->PrevView, pos_prev);
                    float2 posNDC_prev = f2(posV_prev.x, posV_prev.y) / (posV_prev.z * fc->TanHalfFOV);
                    posNDC_prev.x /= fc->AspectRatio;

                    float2 currUV = (f2((float)x, (float)y) + 0.5f) / renderDim;
                    float2 prevUV = Math::UVFromNDC(posNDC_prev) - (jitter / renderDim);
                    float2 motionVec = currUV - prevUV;

                    float3 pos = mad(h.t, rayDir, rayOrigin);
                    float3 posV = Math::mul3x4(fc->CurrView, pos);
                    float z = fc->DoF ? h.t : posV.z;
                    float3 wo = rayOrigin - pos;

                    // ApplyTextureMaps (factors only)
                    const zr_material& mat = sc.materials[meshData.MatIdx];
                    float3 baseColor = Mat::GetBaseColorFactor(mat);
                    float3 emissiveColor = Mat::GetEmissiveFactor(mat);
                    float metallic = Mat::Metallic(mat) ? 1.0f : 0.0f;
                    float roughness = Mat::GetSpecularRoughness(mat);
                    float3 shadingNormal = normal;
                    float3 dndu = td.dndu, dndv = td.dndv;
                    if (Mat::DoubleSided(mat) && dot(wo, normal) < 0)
                    {
                        shadingNormal = -shadingNormal;
                        dndu = -dndu; dndv = -dndv;
                    }
                    if (dot(wo, normal) > 0 && dot(wo, shadingNormal) < 0)
                    {
                        float3 won = normalize(wo);
                        shadingNormal = shadingNormal - dot(shadingNormal, won) * won;
                        shadingNormal = 1e-4f * won + shadingNormal;
                        shadingNormal = normalize(shadingNormal);
                    }
                    float emissiveStrength = Mat::GetEmissiveStrength(mat);
                    emissiveColor *= emissiveStrength;
                    bool transmissive = Mat::Transmissive(mat);
                    float ior = Mat::GetSpecularIOR(mat);
                    float trDepth = transmissive ? Mat::GetTransmissionDepth(mat) : 0;
                    float subsurface = Mat::ThinWalled(mat) ? Mat::GetSubsurface(mat) : 0;
                    float coat_weight = Mat::GetCoatWeight(mat);
                    float3 coat_color = Mat::GetCoatColor(mat);
                    float coat_roughness = Mat::GetCoatRoughness(mat);
                    float coat_ior = Mat::GetCoatIOR(mat);
                    // GBuffer::EncodeMetallic
                    bool isMetal = metallic >= 0.9f;
                    bool isEmissive = dot(emissiveColor, emissiveColor) > 0;
                    uint32_t flags = (transmissive ? 1u : 0u) | ((isEmissive ? 1u : 0u) << 1) | ((trDepth > 0 ? 1u : 0u) << 3) |
                        ((subsurface > 0 ? 1u : 0u) << 4) | ((coat_weight > 0 ? 1u : 0u) << 5) | ((isMetal ? 1u : 0u) << 7);

                    // WriteToGBuffers
                    uint32_t bc = unorm8(baseColor.x) | (unorm8(baseColor.y) << 8) | (unorm8(baseColor.z) << 16) |
                        ((subsurface > 0 ? unorm8(subsurface) : 0u) << 24);
                    uint32_t iorE = transmissive ? unorm8(EncodeIOR(ior)) : 0u;
                    core[idx] = uint4{ asuint(z), pack_unorm16x2(Math::EncodeUnitVector(shadingNormal)), bc,
                        flags | (unorm8(roughness) << 8) | (iorE << 16) };
                    depthPlane[idx] = z;
                    uint32_t em = isEmissive ? pack_r11g11b10(max3(emissiveColor, 0.0f)) : 0u;
                    me[idx] = uint2{ pack_snorm16x2(motionVec), em };
                    if (coat_weight > 0)
                    {
                        uint32_t c = Math::Float3ToRGB8(coat_color);
                        uint32_t px = (c & 0xffff);
                        uint32_t py = (c >> 16) | (Math::FloatToUNorm8(coat_weight) << 8);
                        float normalized = EncodeIOR(coat_ior);
                        uint32_t pz = Math::FloatToUNorm8(coat_roughness) | (Math::FloatToUNorm8(normalized) << 8);
                        coat[idx] = uint2{ px | (py << 16), pz };
                    }
                    else
                        coat[idx] = uint2{ 0u, 0u };
                    if (tridiff)
                    {
                        uint32_t* o = tridiff + idx * 6;
                        o[0] = pack_half2(td.dpdu.x, td.dpdu.y);
                        o[1] = pack_half2(td.dpdu.z, td.dpdv.x);
                        o[2] = pack_half2(td.dpdv.y, td.dpdv.z);
                        o[3] = pack_half2(dndu.x, dndu.y);
                        o[4] = pack_half2(dndu.z, dndv.x);
                        o[5] = pack_half2(dndv.y, dndv.z);
                    }
                }
        };
        parallel_rows(H, nthreads, rows);
    }
}

extern "C"
{
    // PresampleEmissives.hlsl:19-44
    void orc_presample(void* scene_, uint32_t frameNum, uint32_t numTotal, zr_presampled_tri* out)
    {
        const Scene& sc = *(Scene*)scene_;
        for (uint32_t i = 0; i < numTotal; i++)
        {
            RNG rng = RNG::InitIdx(i, frameNum);
            Light::AliasTableSample entry = Light::SampleAlias(sc.aliasTable, sc.numEmissives, rng);
            const zr_emissive_tri& tri = sc.emissives[entry.idx];
            Light::EmissiveTriSample ls = Light::SampleEmissiveTri(f3(0.0f), tri, rng, false);
            const float3 le = Light::Le_EmissiveTriangle(tri);
            zr_presampled_tri s;
            s.pos[0] = ls.pos.x; s.pos[1] = ls.pos.y; s.pos[2] = ls.pos.z;
            s.normal = Math::EncodeOct32u(ls.normal);
            s.pdf = entry.pdf * ls.pdf;
            s.ID = tri.ID;
            s.idx = entry.idx;
            s.bary = Math::EncodeUNorm2(ls.bary);
            s.le[0] = zr_f32_to_f16(le.x); s.le[1] = zr_f32_to_f16(le.y); s.le[2] = zr_f32_to_f16(le.z);
            s.twoSided = Light::IsDoubleSided(tri) ? 1 : 0;
            out[i] = s;
        }
    }
    void orc_scene_set_sample_sets(void* scene_, const zr_presampled_tri* sets, uint32_t numSets, uint32_t setSize)
    {
        Scene& sc = *(Scene*)scene_;
        sc.sampleSets = sets; sc.numSampleSets = numSets; sc.sampleSetSize = setSize;
    }
    void orc_scene_set_lvg(void* scene_, const zr_voxel_sample* lvg, const uint32_t dim[3], const float extents[3], float offset_y)
    {
        Scene& sc = *(Scene*)scene_;
        sc.lvg = lvg;
        for (int i = 0; i < 3; i++) { sc.lvgDim[i] = lvg ? dim[i] : 0; sc.lvgExtents[i] = lvg ? extents[i] : 0; }
        sc.lvgOffsetY = offset_y;
    }
    // BuildLightVoxelGrid.hlsl:56-162: one group of 64 threads per voxel; the two wave sums of a group add up in any order
    // (zeros elsewhere), each 32-lane wave sum in the xor-butterfly order
    void orc_build_lvg(void* scene_, const zr_frame_constants* fc, zr_voxel_sample* out)
    {
        const Scene& sc = *(Scene*)scene_;
        const uint32_t dx = sc.lvgDim[0], dy = sc.lvgDim[1], dz = sc.lvgDim[2];
        const float3 extents = f3(sc.lvgExtents[0], sc.lvgExtents[1], sc.lvgExtents[2]);
        for (uint32_t gz = 0; gz < dz; gz++) for (uint32_t gy = 0; gy < dy; gy++) for (uint32_t gx = 0; gx < dx; gx++)
        {
            const uint32_t gridStart = LVG::FlattenVoxelIndex(gx, gy, gz, dx, dy);
            const float3 voxelCenter = LVG::VoxelCenter((int)gx, (int)gy, (int)gz, (int)dx, (int)dy, (int)dz, extents, fc->CurrViewInv, sc.lvgOffsetY);
            float3 corners[8];
            for (int i = 0; i < 8; i++)
                corners[i] = voxelCenter + f3((i & 4) ? 1.0f : -1.0f, (i & 2) ? 1.0f : -1.0f, (i & 1) ? 1.0f : -1.0f) * extents;
            float w_sum[64], target_z[64]; uint32_t numLights[64];
            zr_voxel_sample r[64];
            for (uint32_t Gidx = 0; Gidx < 64; Gidx++)
            {
                RNG rng = RNG::InitIdx(gridStart * 64 + Gidx, fc->FrameNum);
                zr_voxel_sample& s = r[Gidx];
                s.pos[0] = s.pos[1] = s.pos[2] = FLT_MAX_; s.normal = 0; s.le[0] = s.le[1] = s.le[2] = 0; s.pdf = 0; s.twoSided = 0; s.ID = 0xffffffffu;
                w_sum[Gidx] = 0; target_z[Gidx] = 0; numLights[Gidx] = 0;
                for (int i = 0; i < 6; i++)
                {
                    Light::AliasTableSample entry = Light::SampleAlias(sc.aliasTable, sc.numEmissives, rng);
                    const zr_emissive_tri& tri = sc.emissives[entry.idx];
                    Light::EmissiveTriSample lightSample = Light::SampleEmissiveTri(voxelCenter, tri, rng, false);
                    const float3 le = Light::Le_EmissiveTriangle(tri);
                    // AdjustLightPos: snap lights inside the voxel to its boundary planes
                    const float3 d = f3(fabsf(lightSample.pos.x - voxelCenter.x), fabsf(lightSample.pos.y - voxelCenter.y), fabsf(lightSample.pos.z - voxelCenter.z));
                    const bool inside = d.x <= extents.x && d.y <= extents.y && d.z <= extents.z;
                    float3 lightPos = lightSample.pos;
                    if (inside)
                    {
                        const int maxIdx = d.x >= d.y ? (d.x >= d.z ? 0 : 2) : (d.y >= d.z ? 1 : 2);
                        if (maxIdx == 0) lightPos.x = extents.x; else if (maxIdx == 1) lightPos.y = extents.y; else lightPos.z = extents.z;
                    }
                    if (!inside && !Light::IsDoubleSided(tri))
                    {
                        bool backfacing = false;
                        for (int c = 0; c < 8; c++)
                            if (dot(corners[c] - lightSample.pos, lightSample.normal) <= 0) { backfacing = true; break; }
                        if (backfacing)
                            continue;
                    }
                    const float t = length(lightPos - voxelCenter);
                    const float target = Math::Luminance(le) / fmaxf(t * t, 1e-6f);
                    const float lightPdf = entry.pdf * lightSample.pdf;
                    const float w = target / fmaxf(lightPdf, 1e-6f);
                    w_sum[Gidx] += w;
                    if (rng.Uniform() < w / fmaxf(w_sum[Gidx], 1e-6f))
                    {
                        s.pos[0] = lightSample.pos.x; s.pos[1] = lightSample.pos.y; s.pos[2] = lightSample.pos.z;
                        s.normal = Math::EncodeOct32u(lightSample.normal);
                        s.le[0] = zr_f32_to_f16(le.x); s.le[1] = zr_f32_to_f16(le.y); s.le[2] = zr_f32_to_f16(le.z);
                        s.twoSided = Light::IsDoubleSided(tri) ? 1 : 0;
                        s.ID = tri.ID;
                        target_z[Gidx] = target;
                    }
                    numLights[Gidx]++;
                }
            }
            float waveSum[2]; uint32_t waveLights[2];
            for (int wv = 0; wv < 2; wv++)
            {
                float a[32];
                for (int i = 0; i < 32; i++) a[i] = w_sum[wv * 32 + i];
                for (int off = 16; off >= 1; off >>= 1)
                {
                    float b[32];
                    for (int i = 0; i < 32; i++) b[i] = a[i] + a[i ^ off];
                    for (int i = 0; i < 32; i++) a[i] = b[i];
                }
                waveSum[wv] = a[0];
                waveLights[wv] = 0;
                for (int i = 0; i < 32; i++) waveLights[wv] += numLights[wv * 32 + i];
            }
            float w_sum_group = waveSum[0] + waveSum[1];
            const uint32_t numLightsGroup = (waveLights[0] + waveLights[1]) & 0xffffu;
            w_sum_group /= (float)numLightsGroup;
            for (uint32_t Gidx = 0; Gidx < 64; Gidx++)
            {
                r[Gidx].pdf = target_z[Gidx] / fmaxf(w_sum_group, 1e-6f);
                out[gridStart * 64 + Gidx] = r[Gidx];
            }
        }
    }
    // EstimateTriEmissivePower.hlsl:30-79 without emissive textures
    void orc_estimate_power(void* scene_, float* power)
    {
        const Scene& sc = *(Scene*)scene_;
        for (uint32_t i = 0; i < sc.numEmissives; i++)
        {
            const zr_emissive_tri& tri = sc.emissives[i];
            float3 p = f3(64.0f);
            const float3 emissiveFactor = Math::UnpackRGB8(tri.PackedA);
            const float emissiveStrength = zr_f16_to_f32((uint16_t)(tri.PackedB >> 16));
            p = p * emissiveFactor * emissiveStrength;
            const float3 vtx0 = Light::Vtx0(tri);
            const float3 vtx1 = Light::DecodeEmissiveTriV1(tri);
            const float3 vtx2 = Light::DecodeEmissiveTriV2(tri);
            const float surfaceArea = 0.5f * length(cross(vtx1 - vtx0, vtx2 - vtx0));
            const float pdf = surfaceArea > 0 ? 1.0f / surfaceArea : 0;
            power[i] = pdf > 0 ? Math::Luminance(p) * PI / (pdf * 64.0f) : 0;
        }
    }
}
