// gbuffer.cu -- primary-hit G-buffer pass and the pre-lighting node.
//
// Replaces GBuffer/GBufferRT_Inline.hlsl:72-287 + GBufferRT.hlsli:102-282 (host: GBufferRT.cpp:99-160)
// and PreLighting/EstimateTriEmissivePower.hlsl:30-79 (+ the alias-table protocol of
// PreLighting.cpp:317-429, 512-585 -- now entirely on the device, alias.cu).
// Output layout: include/zr_abi.h zr_gbuffer (one 16-byte record + 4-byte depth + 8-byte
// motion/emissive per pixel, written with 128/64-bit stores).
#include "zr_rt.cuh"        // scene + emissive-light helpers
#include "zr_planes.h"

namespace zr
{
zr_status alias_table_build(float* d_weights, uint32_t n, zr_alias_entry* d_table, uint32_t* d_scratch, cudaStream_t stream);

namespace
{
    ZR_D uint32_t unorm8(float f) { return (uint32_t)mad(saturate(f), 255.0f, 0.5f); }
    ZR_D float EncodeIOR(float ior) { return (ior - 1.0f) / (2.5f - 1.0f); }

    // 14 blocks of 64 per SM is the residency its 72 registers give; stating it keeps the pick arguments from raising that count
    __global__ void __launch_bounds__(64, 14) k_gbuffer(SceneDev sc, zr_frame_constants fc, uint4* __restrict__ core,
        float* __restrict__ depthPlane, uint2* __restrict__ me, uint2* __restrict__ coat, uint2* __restrict__ tridiff,
        uint32_t rowBegin, uint32_t rowEnd, uint32_t* __restrict__ pickOut, uint32_t pickIdx)
    {
        // 8x8 groups like GBUFFER_RT_GROUP_DIM (GBufferRT_Common.h:6-7); rows [rowBegin, rowEnd) of the frame
        const uint32_t x = blockIdx.x * 8 + (threadIdx.x & 7);
        const uint32_t y = rowBegin + blockIdx.y * 8 + (threadIdx.x >> 3);
        const uint32_t W = fc.RenderWidth, H = fc.RenderHeight;
        if (x >= W || y >= H || y >= rowEnd) return;
        const size_t idx = (size_t)y * W + x;

        float2 lensSample = f2(0, 0);
        const float2 renderDim = f2((float)W, (float)H);
        const float2 jitter = f2(fc.CurrCameraJitter[0], fc.CurrCameraJitter[1]);
        float2 uv = (f2((float)x, (float)y) + 0.5f + jitter) / renderDim;
        float2 ndc = Math::NDCFromUV(uv);
        float3 rayDirCS = f3(ndc.x * fc.AspectRatio * fc.TanHalfFOV, ndc.y * fc.TanHalfFOV, 1);
        float3 rayOrigin = f3(fc.CameraPos[0], fc.CameraPos[1], fc.CameraPos[2]);
        const float3 bx = f3(fc.CurrView[0][0], fc.CurrView[0][1], fc.CurrView[0][2]);
        const float3 by = f3(fc.CurrView[1][0], fc.CurrView[1][1], fc.CurrView[1][2]);
        const float3 bz = f3(fc.CurrView[2][0], fc.CurrView[2][1], fc.CurrView[2][2]);
        if (fc.DoF)
        {
            const uint3 h = RNG::PCG3d(make_uint3(x, y, x));
            RNG rng = RNG::Init(h.z, h.y, fc.FrameNum);
            lensSample = Sampling::UniformSampleDiskConcentric(rng.Uniform2D());
            lensSample = lensSample * fc.LensRadius;
            rayOrigin += mad(lensSample.x, bx, lensSample.y * by);
            const float3 focalPoint = fc.FocusDepth * rayDirCS;
            rayDirCS = focalPoint - f3(lensSample.x, lensSample.y, 0);
        }
        float3 rayDir = mad(rayDirCS.x, bx, mad(rayDirCS.y, by, rayDirCS.z * bz));
        rayDir = normalize(rayDir);

        const RayHit h = TraceClosest(sc, rayOrigin, rayDir, 0.0f, FLT_MAX_);
        if (!h.hit)
        {
            const float3 prevCameraPos = f3(fc.PrevViewInv[0][3], fc.PrevViewInv[1][3], fc.PrevViewInv[2][3]);
            const float3 motion = f3(fc.CameraPos[0], fc.CameraPos[1], fc.CameraPos[2]) - prevCameraPos;
            float2 motionNDC = motion.z > 0 ? f2(motion.x, motion.y) / (motion.z * fc.TanHalfFOV) : f2(0, 0);
            motionNDC.x /= fc.AspectRatio;
            const float2 motionUV = Math::UVFromNDC(motionNDC);
            core[idx] = make_uint4(asuint(FLT_MAX_), 0u, 0u, 4u);
            depthPlane[idx] = FLT_MAX_;
            me[idx] = make_uint2(pack_snorm16x2(motionUV), 0u);
            coat[idx] = make_uint2(0u, 0u);
            if (tridiff) { tridiff[idx * 3] = make_uint2(0, 0); tridiff[idx * 3 + 1] = make_uint2(0, 0); tridiff[idx * 3 + 2] = make_uint2(0, 0); }
            if ((uint32_t)idx == pickIdx) *pickOut = 0xffffffffu;
            return;
        }
        const uint32_t meshIdx = __ldg(&sc.triMesh[h.tri]);
        const uint32_t primIdx = h.tri - __ldg(&sc.meshFirstTri[meshIdx]);
        const zr_mesh_instance meshData = LoadInstance(sc, meshIdx);
        const float2 bary = h.bary;
        const uint32_t tri = primIdx * 3 + meshData.BaseIdxOffset;
        const VertexD V0 = LoadVertex(sc, __ldg(&sc.indices[tri]) + meshData.BaseVtxOffset);
        const VertexD V1 = LoadVertex(sc, __ldg(&sc.indices[tri + 1]) + meshData.BaseVtxOffset);
        const VertexD V2 = LoadVertex(sc, __ldg(&sc.indices[tri + 2]) + meshData.BaseVtxOffset);
        const float4 q = normalize(Math::DecodeNormalized4(meshData.Rotation));
        const float3 scale = h3(meshData.Scale);
        const float3 translation = f3(meshData.Translation[0], meshData.Translation[1], meshData.Translation[2]);
        const float3 v0_n = Math::DecodeOct32(V0.normal);
        const float3 v1_n = Math::DecodeOct32(V1.normal);
        const float3 v2_n = Math::DecodeOct32(V2.normal);
        float3 normal = v0_n + bary.x * (v1_n - v0_n) + bary.y * (v2_n - v0_n);
        const float3 scaleInv = 1.0f / scale;
        normal *= scaleInv;
        normal = Math::RotateVector(normal, q);
        normal = normalize(normal);

        Math::TriDifferentials td;
        td.dpdu = td.dpdv = td.dndu = td.dndv = f3(0);
        if (tridiff)
        {
            const float3 v0W = Math::TransformTRS(V0.pos, translation, q, scale);
            const float3 v1W = Math::TransformTRS(V1.pos, translation, q, scale);
            const float3 v2W = Math::TransformTRS(V2.pos, translation, q, scale);
            const float3 n0W = normalize(Math::RotateVector(v0_n * scaleInv, q));
            const float3 n1W = normalize(Math::RotateVector(v1_n * scaleInv, q));
            const float3 n2W = normalize(Math::RotateVector(v2_n * scaleInv, q));
            td = Math::TriDifferentials::Compute(v0W, v1W, v2W, n0W, n1W, n2W, V0.uv, V1.uv, V2.uv);
        }

        // motion vector
        const float3 hitPos = mad(rayDir, h.t, rayOrigin);
        const float3 posL = Math::InverseTransformTRS(hitPos, translation, q, scale);
        const float3 prevTranslation = translation - h3(meshData.dTranslation);
        const float4 q_prev = normalize(Math::DecodeNormalized4(meshData.PrevRotation));
        const float3 pos_prev = Math::TransformTRS(posL, prevTranslation, q_prev, h3(meshData.PrevScale));
        const float3 posV_prev = Math::mul3x4(fc.PrevView, pos_prev);
        float2 posNDC_prev = f2(posV_prev.x, posV_prev.y) / (posV_prev.z * fc.TanHalfFOV);
        posNDC_prev.x /= fc.AspectRatio;
        const float2 currUV = (f2((float)x, (float)y) + 0.5f) / renderDim;
        const float2 prevUV = Math::UVFromNDC(posNDC_prev) - (jitter / renderDim);
        const float2 motionVec = currUV - prevUV;

        const float3 pos = mad(h.t, rayDir, rayOrigin);
        const float3 posV = Math::mul3x4(fc.CurrView, pos);
        const float z = fc.DoF ? h.t : posV.z;
        const float3 wo = rayOrigin - pos;

        const zr_material mat = LoadMaterial(sc, meshData.MatIdx);
        const float3 baseColor = Mat::GetBaseColorFactor(mat);
        float3 emissiveColor = Mat::GetEmissiveFactor(mat);
        const float metallic = Mat::Metallic(mat) ? 1.0f : 0.0f;
        const float roughness = Mat::GetSpecularRoughness(mat);
        float3 shadingNormal = normal;
        float3 dndu = td.dndu, dndv = td.dndv;
        if (Mat::DoubleSided(mat) && dot(wo, normal) < 0)
        {
            shadingNormal = -shadingNormal;
            dndu = -dndu; dndv = -dndv;
        }
        if (dot(wo, normal) > 0 && dot(wo, shadingNormal) < 0)
        {
            const float3 won = normalize(wo);
            shadingNormal = shadingNormal - dot(shadingNormal, won) * won;
            shadingNormal = 1e-4f * won + shadingNormal;
            shadingNormal = normalize(shadingNormal);
        }
        emissiveColor *= Mat::GetEmissiveStrength(mat);
        const bool transmissive = Mat::Transmissive(mat);
        const float ior = Mat::GetSpecularIOR(mat);
        const float trDepth = transmissive ? Mat::GetTransmissionDepth(mat) : 0;
        const float subsurface = Mat::ThinWalled(mat) ? Mat::GetSubsurface(mat) : 0;
        const float coat_weight = Mat::GetCoatWeight(mat);
        const bool isMetal = metallic >= 0.9f;
        const bool isEmissive = dot(emissiveColor, emissiveColor) > 0;
        const uint32_t flags = (transmissive ? 1u : 0u) | ((isEmissive ? 1u : 0u) << 1) | ((trDepth > 0 ? 1u : 0u) << 3) |
            ((subsurface > 0 ? 1u : 0u) << 4) | ((coat_weight > 0 ? 1u : 0u) << 5) | ((isMetal ? 1u : 0u) << 7);

        const uint32_t bc = unorm8(baseColor.x) | (unorm8(baseColor.y) << 8) | (unorm8(baseColor.z) << 16) |
            ((subsurface > 0 ? unorm8(subsurface) : 0u) << 24);
        const uint32_t iorE = transmissive ? unorm8(EncodeIOR(ior)) : 0u;
        if ((uint32_t)idx == pickIdx) *pickOut = meshIdx;       // GBufferRT_Inline.hlsl:241-242 (hitMeshIdx)
        core[idx] = make_uint4(asuint(z), Math::EncodeUNorm2(Math::EncodeUnitVector(shadingNormal)), bc,
            flags | (unorm8(roughness) << 8) | (iorE << 16));
        depthPlane[idx] = z;
        const uint32_t em = isEmissive ? pack_r11g11b10(max3(emissiveColor, 0.0f)) : 0u;
        me[idx] = make_uint2(pack_snorm16x2(motionVec), em);
        if (coat_weight > 0)
        {
            const uint32_t c = Math::Float3ToRGB8(Mat::GetCoatColor(mat));
            const uint32_t px = (c & 0xffff);
            const uint32_t py = (c >> 16) | (Math::FloatToUNorm8(coat_weight) << 8);
            const float normalized = EncodeIOR(Mat::GetCoatIOR(mat));
            const uint32_t pz = Math::FloatToUNorm8(Mat::GetCoatRoughness(mat)) | (Math::FloatToUNorm8(normalized) << 8);
            coat[idx] = make_uint2(px | (py << 16), pz);
        }
        else
            coat[idx] = make_uint2(0u, 0u);
        if (tridiff)
        {
            tridiff[idx * 3 + 0] = make_uint2(pack_half2(td.dpdu.x, td.dpdu.y), pack_half2(td.dpdu.z, td.dpdv.x));
            tridiff[idx * 3 + 1] = make_uint2(pack_half2(td.dpdv.y, td.dpdv.z), pack_half2(dndu.x, dndu.y));
            tridiff[idx * 3 + 2] = make_uint2(pack_half2(dndu.z, dndv.x), pack_half2(dndv.y, dndv.z));
        }
    }

    // one thread per emissive triangle (no emissive textures in this build, so the 64 Halton taps
    // of the reference collapse to the constant 64)
    // PresampleEmissives.hlsl:19-44: one power-proportional light sample per thread, packed to 40 bytes
    __global__ void __launch_bounds__(64) k_presample(SceneDev sc, uint32_t frameNum, uint32_t numTotal, zr_presampled_tri* __restrict__ out)
    {
        const uint32_t i = blockIdx.x * 64 + threadIdx.x;
        if (i >= numTotal) return;
        RNG rng = RNG::InitIdx(i, frameNum);
        const Light::AliasTableSample entry = Light::SampleAlias(sc.aliasTable, sc.numEmissives, rng);
        const zr_emissive_tri& tri = sc.emissives[entry.idx];
        const Light::EmissiveTriSample ls = Light::SampleEmissiveTri(f3(0), tri, rng, false);
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
        uint2 v[5];
        memcpy(v, &s, 40);
        uint2* q = reinterpret_cast<uint2*>(out + i);
        for (int k = 0; k < 5; k++) q[k] = v[k];
    }

    // BuildLightVoxelGrid.hlsl:56-162: one 64-thread group per voxel, RIS over 6 alias-table candidates per thread
    __global__ void __launch_bounds__(64) k_build_lvg(SceneDev sc, zr_frame_constants fc, zr_voxel_sample* __restrict__ out)
    {
        __shared__ float s_waveSum[2];
        __shared__ uint32_t s_waveLights[2];
        const uint32_t dx = sc.lvgDim[0], dy = sc.lvgDim[1], dz = sc.lvgDim[2];
        const uint32_t Gidx = threadIdx.x;
        const uint32_t gridStart = LVG::FlattenVoxelIndex(blockIdx.x, blockIdx.y, blockIdx.z, dx, dy);
        const float3 extents = f3(sc.lvgExtents[0], sc.lvgExtents[1], sc.lvgExtents[2]);
        RNG rng = RNG::InitIdx(gridStart * 64 + Gidx, fc.FrameNum);
        const float3 voxelCenter = LVG::VoxelCenter((int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z, (int)dx, (int)dy, (int)dz, extents, fc.CurrViewInv,
            sc.lvgOffsetY);
        zr_voxel_sample r;
        r.pos[0] = r.pos[1] = r.pos[2] = FLT_MAX_; r.normal = 0; r.le[0] = r.le[1] = r.le[2] = 0; r.pdf = 0; r.twoSided = 0; r.ID = 0xffffffffu;
        float w_sum = 0, target_z = 0;
        uint32_t numLights = 0;
        for (int i = 0; i < 6; i++)
        {
            const Light::AliasTableSample entry = Light::SampleAlias(sc.aliasTable, sc.numEmissives, rng);
            const zr_emissive_tri& tri = sc.emissives[entry.idx];
            const Light::EmissiveTriSample lightSample = Light::SampleEmissiveTri(voxelCenter, tri, rng, false);
            const float3 le = Light::Le_EmissiveTriangle(tri);
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
                {
                    const float3 corner = voxelCenter + f3((c & 4) ? 1.0f : -1.0f, (c & 2) ? 1.0f : -1.0f, (c & 1) ? 1.0f : -1.0f) * extents;
                    if (dot(corner - lightSample.pos, lightSample.normal) <= 0) backfacing = true;
                }
                if (backfacing)
                    continue;
            }
            const float t = length(lightPos - voxelCenter);
            const float target = Math::Luminance(le) / fmaxf(t * t, 1e-6f);
            const float lightPdf = entry.pdf * lightSample.pdf;
            const float w = target / fmaxf(lightPdf, 1e-6f);
            w_sum += w;
            if (rng.Uniform() < w / fmaxf(w_sum, 1e-6f))
            {
                r.pos[0] = lightSample.pos.x; r.pos[1] = lightSample.pos.y; r.pos[2] = lightSample.pos.z;
                r.normal = Math::EncodeOct32u(lightSample.normal);
                r.le[0] = zr_f32_to_f16(le.x); r.le[1] = zr_f32_to_f16(le.y); r.le[2] = zr_f32_to_f16(le.z);
                r.twoSided = Light::IsDoubleSided(tri) ? 1 : 0;
                r.ID = tri.ID;
                target_z = target;
            }
            numLights++;
        }
        const float waveSum = WaveSum32(w_sum);
        uint32_t waveLights = numLights;
        for (int off = 16; off >= 1; off >>= 1) waveLights += __shfl_xor_sync(0xffffffffu, waveLights, off);
        if ((Gidx & 31) == 0) { s_waveSum[Gidx >> 5] = waveSum; s_waveLights[Gidx >> 5] = waveLights; }
        __syncthreads();
        float w_sum_group = s_waveSum[0] + s_waveSum[1];
        const uint32_t numLightsGroup = (s_waveLights[0] + s_waveLights[1]) & 0xffffu;
        w_sum_group /= (float)numLightsGroup;
        r.pdf = target_z / fmaxf(w_sum_group, 1e-6f);
        uint4 v[2];
        memcpy(v, &r, 32);
        uint4* q = reinterpret_cast<uint4*>(out + gridStart * 64 + Gidx);
        q[0] = v[0]; q[1] = v[1];
    }

    __global__ void k_emissive_power(SceneDev sc, float* __restrict__ power)
    {
        const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= sc.numEmissives) return;
        const zr_emissive_tri tri = sc.emissives[i];
        float3 p = f3(64.0f);
        const float3 emissiveFactor = Math::UnpackRGB8(tri.PackedA);
        const float emissiveStrength = zr_f16_to_f32((uint16_t)(tri.PackedB >> 16));
        p = p * emissiveFactor * emissiveStrength;
        const float3 vtx0 = f3(tri.Vtx0[0], tri.Vtx0[1], tri.Vtx0[2]);
        const float3 d1 = Math::DecodeUnitVector(f2((float)tri.V0V1[0] / 65535.0f, (float)tri.V0V1[1] / 65535.0f));
        const float3 d2 = Math::DecodeUnitVector(f2((float)tri.V0V2[0] / 65535.0f, (float)tri.V0V2[1] / 65535.0f));
        const float3 vtx1 = mad(d1, zr_f16_to_f32(tri.EdgeLengths[0]), vtx0);
        const float3 vtx2 = mad(d2, zr_f16_to_f32(tri.EdgeLengths[1]), vtx0);
        const float surfaceArea = 0.5f * length(cross(vtx1 - vtx0, vtx2 - vtx0));
        const float pdf = surfaceArea > 0 ? 1.0f / surfaceArea : 0;
        power[i] = pdf > 0 ? Math::Luminance(p) * PI / (pdf * 64.0f) : 0;
    }
}
} // namespace zr

struct zr_gbuffer_pass
{
    // GBufferRT (GBuffer/GBufferRT.h): the renderer owns the G-buffers (ZetaRenderer/Default/DefaultRendererImpl.h:111-121); the
    // pass holds only the picked-instance word that the caller reads back after a picking render
    uint32_t rowBegin = 0, rowEnd = 0xffffffffu;    // rows this device renders (strip-sharded frames); all by default
    zr::Planes planes{ "zr_gbuffer_pass" };
    uint32_t* d_pick = nullptr;                     // instance index under the last picked pixel, 0xffffffff for none
    bool pickArmed = false;
    uint32_t pickX = 0, pickY = 0;

    zr_status Setup()
    {
        ZR_TRY(planes.Alloc(d_pick, 1, false));
        ZR_CLEAR_BEGIN();
        ZR_CUDA(cudaMemset(d_pick, 0xff, sizeof(uint32_t)));
        ZR_CLEAR_END();
        return ZR_OK;
    }
    zr_status Render(const zr_frame_inputs* in, cudaStream_t stream)
    {
        using namespace zr;
        if (!in || !in->scene || !in->curr.d_core || !in->curr.d_depth || !in->curr.d_motion_emissive || !in->curr.d_coat)
        {
            set_error("zr_gbuffer_pass_render: missing scene or G-buffer planes");
            return ZR_ERR_INVALID_ARG;
        }
        const uint32_t W = in->frame.RenderWidth, H = in->frame.RenderHeight;
        if (!W || !H) { set_error("zr_gbuffer_pass_render: zero render size"); return ZR_ERR_INVALID_ARG; }
        const uint32_t y1 = rowEnd < H ? rowEnd : H;
        if (rowBegin >= y1) { set_error("zr_gbuffer_pass_render: empty row range"); return ZR_ERR_INVALID_ARG; }
        // GBufferRT::PickPixel is one-shot: this render answers it. A pixel the kernel does not visit (outside the frame or the
        // pass's rows) answers "none" here.
        uint32_t pickIdx = 0xffffffffu;
        if (pickArmed)
        {
            if (pickX < W && pickY >= rowBegin && pickY < y1)
                pickIdx = pickY * W + pickX;
            else
                ZR_CUDA(cudaMemsetAsync(d_pick, 0xff, sizeof(uint32_t), stream));
        }
        dim3 grid((W + 7) / 8, (y1 - rowBegin + 7) / 8);
        ZR_PROF("k_gbuffer", stream);
        k_gbuffer<<<grid, 64, 0, stream>>>(in->scene->dev, in->frame, (uint4*)in->curr.d_core, (float*)in->curr.d_depth,
            (uint2*)in->curr.d_motion_emissive, (uint2*)in->curr.d_coat, (uint2*)in->curr.d_tridiff, rowBegin, y1, d_pick, pickIdx);
        ZR_LAUNCH_CHECK();
        pickArmed = false;
        return ZR_OK;
    }
};

extern "C"
{
    zr_status zr_gbuffer_alloc(uint32_t width, uint32_t height, int with_tridiff, zr_gbuffer* out)
    {
        if (!out || !width || !height) { zr::set_error("zr_gbuffer_alloc: bad args"); return ZR_ERR_INVALID_ARG; }
        const size_t n = (size_t)width * height;
        memset(out, 0, sizeof(*out));
        cudaError_t e = cudaMalloc(&out->d_core, n * 16);
        if (e == cudaSuccess) e = cudaMalloc(&out->d_depth, n * 4);
        if (e == cudaSuccess) e = cudaMalloc(&out->d_motion_emissive, n * 8);
        if (e == cudaSuccess) e = cudaMalloc(&out->d_coat, n * 8);
        if (e == cudaSuccess && with_tridiff) e = cudaMalloc(&out->d_tridiff, n * 24);
        if (e != cudaSuccess)
        {
            cudaGetLastError();     // the failure is reported here, not by the next launch check
            zr_gbuffer_free(out);
            zr::set_error("zr_gbuffer_alloc: cannot allocate the %ux%u G-buffer (%s)", width, height, cudaGetErrorString(e));
            return e == cudaErrorMemoryAllocation ? ZR_ERR_OUT_OF_MEMORY : ZR_ERR_CUDA;
        }
        ZR_CLEAR_BEGIN();
        ZR_CUDA(cudaMemset(out->d_core, 0, n * 16));
        ZR_CUDA(cudaMemset(out->d_depth, 0, n * 4));
        ZR_CUDA(cudaMemset(out->d_motion_emissive, 0, n * 8));
        ZR_CUDA(cudaMemset(out->d_coat, 0, n * 8));
        ZR_CLEAR_END();
        return ZR_OK;
    }
    void zr_gbuffer_free(zr_gbuffer* g)
    {
        if (!g) return;
        cudaFree(g->d_core); cudaFree(g->d_depth); cudaFree(g->d_motion_emissive); cudaFree(g->d_coat);
        if (g->d_tridiff) cudaFree(g->d_tridiff);
        memset(g, 0, sizeof(*g));
    }
    zr_status zr_gbuffer_pass_create(zr_gbuffer_pass** out)
    {
        if (!out) return ZR_ERR_INVALID_ARG;
        *out = nullptr;
        std::unique_ptr<zr_gbuffer_pass> p(new zr_gbuffer_pass());
        ZR_TRY(p->Setup());
        *out = p.release();
        return ZR_OK;
    }
    zr_status zr_gbuffer_pass_pick(zr_gbuffer_pass* p, uint32_t x, uint32_t y)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        p->pickArmed = true; p->pickX = x; p->pickY = y;
        return ZR_OK;
    }
    zr_status zr_gbuffer_pass_get_pick(zr_gbuffer_pass* p, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        *out = zr_image2d{ p->d_pick, 1, 1, 4u, 4u };
        return ZR_OK;
    }
    zr_status zr_gbuffer_pass_set_rows(zr_gbuffer_pass* p, uint32_t y0, uint32_t y1)
    {
        if (!p || y0 >= y1) { zr::set_error("zr_gbuffer_pass_set_rows: empty row range"); return ZR_ERR_INVALID_ARG; }
        p->rowBegin = y0; p->rowEnd = y1;
        return ZR_OK;
    }
    zr_status zr_gbuffer_pass_render(zr_gbuffer_pass* p, const zr_frame_inputs* in, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, (cudaStream_t)stream);
    }
    zr_status zr_gbuffer_pass_describe_io(zr_gbuffer_pass* p, zr_resource_use* uses, int* n)
    {
        if (!p || !uses || !n) return ZR_ERR_INVALID_ARG;
        uses[0] = zr_resource_use{ ZR_RES_SCENE_BVH, 0 };
        uses[1] = zr_resource_use{ ZR_RES_GBUFFER_CURR, 1 };
        *n = 2;
        return ZR_OK;
    }
    void zr_gbuffer_pass_destroy(zr_gbuffer_pass* p) { delete p; }

    zr_status zr_estimate_emissive_power(const zr_scene* scene, float* d_power, void* stream)
    {
        if (!scene || !d_power) { zr::set_error("zr_estimate_emissive_power: null argument"); return ZR_ERR_INVALID_ARG; }
        const uint32_t n = scene->dev.numEmissives;
        if (n == 0) return ZR_OK;
        ZR_PROF("k_emissive_power", (cudaStream_t)stream);
        zr::k_emissive_power<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(scene->dev, d_power);
        ZR_LAUNCH_CHECK();
        return ZR_OK;
    }
    zr_status zr_prelighting_render(zr_scene* scene, void* stream)
    {
        if (!scene) return ZR_ERR_INVALID_ARG;
        if (scene->dev.numEmissives == 0) return ZR_OK;
        zr_status s = zr_estimate_emissive_power(scene, scene->d_power, stream);
        if (s != ZR_OK) return s;
        s = zr::alias_table_build(scene->d_power, scene->dev.numEmissives, scene->d_alias, scene->d_aliasScratch, (cudaStream_t)stream);
        if (s == ZR_OK) scene->aliasBuilt = true;
        return s;
    }

    zr_status zr_scene_set_presampling(zr_scene* scene, uint32_t num_sets, uint32_t set_size)
    {
        if (!scene) return ZR_ERR_INVALID_ARG;
        if ((num_sets == 0) != (set_size == 0) || (uint64_t)num_sets * set_size > (1u << 24))
        {
            zr::set_error("zr_scene_set_presampling: num_sets and set_size must both be 0 or both > 0 (at most 2^24 samples)");
            return ZR_ERR_INVALID_ARG;
        }
        if (scene->d_sampleSets) { cudaFree(scene->d_sampleSets); scene->d_sampleSets = nullptr; }
        scene->dev.sampleSets = nullptr; scene->dev.numSampleSets = 0; scene->dev.sampleSetSize = 0;
        scene->samplesValid = false;
        if (num_sets)
        {
            ZR_CUDA(cudaMalloc(&scene->d_sampleSets, (size_t)num_sets * set_size * sizeof(zr_presampled_tri)));
            scene->dev.sampleSets = scene->d_sampleSets; scene->dev.numSampleSets = num_sets; scene->dev.sampleSetSize = set_size;
        }
        return ZR_OK;
    }
    zr_status zr_presample_emissives(zr_scene* scene, uint32_t frame_num, void* stream)
    {
        if (!scene) return ZR_ERR_INVALID_ARG;
        if (!scene->dev.sampleSetSize) return ZR_OK;        // presampling is off: nothing to do (like the reference's render graph)
        if (!scene->aliasBuilt || scene->dev.numEmissives == 0)
        {
            zr::set_error("zr_presample_emissives: needs emissive triangles and zr_prelighting_render first");
            return ZR_ERR_NOT_INITIALIZED;
        }
        const uint32_t total = scene->dev.numSampleSets * scene->dev.sampleSetSize;
        ZR_PROF("k_presample", stream);
        zr::k_presample<<<(total + 63) / 64, 64, 0, (cudaStream_t)stream>>>(scene->dev, frame_num, total, scene->d_sampleSets);
        ZR_LAUNCH_CHECK();
        scene->samplesValid = true;
        return ZR_OK;
    }
    zr_status zr_scene_set_light_voxel_grid(zr_scene* scene, const uint32_t grid_dim[3], const float extents[3], float offset_y)
    {
        if (!scene) return ZR_ERR_INVALID_ARG;
        if (scene->d_lvg) { cudaFree(scene->d_lvg); scene->d_lvg = nullptr; }
        scene->dev.lvg = nullptr; scene->lvgValid = false;
        for (int i = 0; i < 3; i++) { scene->dev.lvgDim[i] = 0; scene->dev.lvgExtents[i] = 0; }
        scene->dev.lvgOffsetY = 0;
        if (!grid_dim || (grid_dim[0] | grid_dim[1] | grid_dim[2]) == 0)
            return ZR_OK;       // off
        const uint64_t voxels = (uint64_t)grid_dim[0] * grid_dim[1] * grid_dim[2];
        if (!extents || !grid_dim[0] || !grid_dim[1] || !grid_dim[2] || voxels > (1u << 20) || !(extents[0] > 0 && extents[1] > 0 && extents[2] > 0))
        {
            zr::set_error("zr_scene_set_light_voxel_grid: need positive dims (<= 2^20 voxels) and extents");
            return ZR_ERR_INVALID_ARG;
        }
        ZR_CUDA(cudaMalloc(&scene->d_lvg, voxels * 64 * sizeof(zr_voxel_sample)));
        scene->dev.lvg = scene->d_lvg;
        for (int i = 0; i < 3; i++) { scene->dev.lvgDim[i] = grid_dim[i]; scene->dev.lvgExtents[i] = extents[i]; }
        scene->dev.lvgOffsetY = offset_y;
        return ZR_OK;
    }
    zr_status zr_build_light_voxel_grid(zr_scene* scene, const zr_frame_constants* frame, void* stream)
    {
        if (!scene || !frame) return ZR_ERR_INVALID_ARG;
        if (!scene->dev.lvg) return ZR_OK;
        if (!scene->aliasBuilt || scene->dev.numEmissives == 0)
        {
            zr::set_error("zr_build_light_voxel_grid: needs emissive triangles and zr_prelighting_render first");
            return ZR_ERR_NOT_INITIALIZED;
        }
        ZR_PROF("k_build_lvg", stream);
        zr::k_build_lvg<<<dim3(scene->dev.lvgDim[0], scene->dev.lvgDim[1], scene->dev.lvgDim[2]), 64, 0, (cudaStream_t)stream>>>(scene->dev, *frame,
            scene->d_lvg);
        ZR_LAUNCH_CHECK();
        scene->lvgValid = true;
        return ZR_OK;
    }
    zr_status zr_scene_get_light_voxel_grid(zr_scene* scene, void** d_samples, uint32_t* num_samples)
    {
        if (!scene || !d_samples || !num_samples) return ZR_ERR_INVALID_ARG;
        *d_samples = scene->d_lvg;
        *num_samples = scene->dev.lvgDim[0] * scene->dev.lvgDim[1] * scene->dev.lvgDim[2] * 64u;
        return ZR_OK;
    }
    zr_status zr_scene_get_sample_sets(zr_scene* scene, void** d_sets, uint32_t* num_sets, uint32_t* set_size)
    {
        if (!scene || !d_sets || !num_sets || !set_size) return ZR_ERR_INVALID_ARG;
        *d_sets = scene->d_sampleSets; *num_sets = scene->dev.numSampleSets; *set_size = scene->dev.sampleSetSize;
        return ZR_OK;
    }
}
