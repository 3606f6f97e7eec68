// ORACLE -- test infrastructure, not product code (see orc_math.h header). PARITY UNPINNED: the reference has no tests,
// golden images or CPU implementation for this shader.
//
// CPU restatement of ReSTIR GI with emissive NEE (the ReSTIR_GI_WoPS / _WPS shader variants):
//   IndirectLighting/ReSTIR_GI/ReSTIR_GI.hlsl        main :64-165
//   IndirectLighting/ReSTIR_GI/Resampling.hlsli      RIS_InitialCandidates :39-113, FindTemporalCandidate :124-233,
//                                                    TargetLumAtTemporalPixel :235-284, JacobianReconnectionShift :288-308,
//                                                    TemporalResample1 :310-371, TemporalResample2 :373-454,
//                                                    SuppressOutlierReservoirs :533-539, EstimateIndirectLighting :541-612
//   IndirectLighting/ReSTIR_GI/PathTracing.hlsli     PathTrace :10-98
//   IndirectLighting/ReSTIR_GI/ReSTIR_GI_NEE.hlsli   NEE_Emissive_MIS :8-121, NEE :195-270 (NEE_EMISSIVE == 1, USE_MIS == 1)
//   IndirectLighting/NEE.hlsli                       NEE_Emissive<1> :152-221
//   IndirectLighting/ReSTIR_GI/Reservoir.hlsli       Reservoir, read/write :9-131
//   host: IndirectLighting.cpp RenderReSTIR_GI :277-368 (ping-pong, flags)
// Not restated: ray differentials (only feed texture LOD; no textures in this build), the sun/sky variant, the disabled
// spatial pass (Resampling.hlsli:603-608 is commented out upstream).
// Wave-scope ops: the Russian-roulette WaveActiveMax inside the bounce loop is evaluated over the lanes of a wave that
// are at the same iteration (lock-step, like the ReSTIR PT restatement); SuppressOutlierReservoirs sums over the lanes
// that reached it, in the xor-butterfly order.
// D3D semantics kept: texture reads outside the image return 0 (FindTemporalCandidate does not reject negative taps).
#include "orc_api.h"
#include "orc_pixel.h"

namespace orc
{
namespace
{
    struct GIParams
    {
        uint32_t maxNonTrBounces, maxGlossyTrBounces, russianRoulette, stochasticMultiBounce, boilingSuppression, M_max;
        uint32_t temporalResample;      // caller-level switch; the pass ANDs it with "previous reservoirs are valid"
    };

    struct GIReservoir
    {
        float3 pos, Lo, normal, target_z;
        float W, w_sum; uint32_t ID; float M;       // M is a half in the reference; small integers are exact
        static GIReservoir Init()
        {
            GIReservoir r;
            r.pos = f3(FLT_MAX_); r.normal = f3(0); r.Lo = f3(0); r.M = 0; r.w_sum = 0; r.W = 0; r.ID = UINT32_MAX_; r.target_z = f3(0);
            return r;
        }
        bool Update(float weight, float3 vtxPos, float3 vtxNormal, uint32_t vtxID, float3 vtxLo, float3 target, RNG& rng)
        {
            if (weight != weight)
                return false;
            w_sum += weight;
            M += 1;
            if (rng.Uniform() < (weight / fmaxf(1e-6f, w_sum)))
            {
                pos = vtxPos; normal = vtxNormal; ID = vtxID; Lo = vtxLo; target_z = target;
                return true;
            }
            return false;
        }
    };

    // zr_rgi_reservoir (48 bytes): A = {pos.xyz, ID}, B = {Lo.rg (half2), Lo.b | M (half2), w_sum, W}, C = {oct32 normal, 0, 0, 0}
    void WriteReservoir(zr_rgi_reservoir& s, const GIReservoir& r, float M_max)
    {
        s.pos[0] = r.pos.x; s.pos[1] = r.pos.y; s.pos[2] = r.pos.z; s.ID = r.ID;
        const float M_clamped = fminf(r.M, M_max);
        s.Lo_rg = (uint32_t)zr_f32_to_f16(r.Lo.x) | ((uint32_t)zr_f32_to_f16(r.Lo.y) << 16);
        s.Lo_b_M = (uint32_t)zr_f32_to_f16(r.Lo.z) | ((uint32_t)zr_f32_to_f16(M_clamped) << 16);
        s.w_sum = r.w_sum; s.W = r.W;
        s.normal = Math::EncodeOct32u(r.normal);
        s.pad[0] = s.pad[1] = s.pad[2] = 0;
    }
    const zr_rgi_reservoir* TexelOrNull(const zr_rgi_reservoir* res, uint32_t W, uint32_t H, int x, int y)
    {
        return (x < 0 || y < 0 || x >= (int)W || y >= (int)H) ? nullptr : &res[(size_t)y * W + x];
    }
    GIReservoir PartialReadReservoir_Reuse(const zr_rgi_reservoir* res, uint32_t W, uint32_t H, int x, int y)
    {
        const zr_rgi_reservoir* s = TexelOrNull(res, W, H, x, y);
        GIReservoir r;
        r.normal = f3(0); r.w_sum = 0; r.W = 0; r.target_z = f3(0);
        if (!s) { r.pos = f3(0); r.ID = 0; r.Lo = f3(0); r.M = 0; return r; }      // out-of-bounds texture read
        r.pos = f3(s->pos[0], s->pos[1], s->pos[2]); r.ID = s->ID;
        r.Lo = f3(zr_f16_to_f32((uint16_t)(s->Lo_rg & 0xffff)), zr_f16_to_f32((uint16_t)(s->Lo_rg >> 16)), zr_f16_to_f32((uint16_t)(s->Lo_b_M & 0xffff)));
        r.M = (float)(uint16_t)zr_f16_to_f32((uint16_t)(s->Lo_b_M >> 16));
        return r;
    }
    void PartialReadReservoir_ReuseRest(const zr_rgi_reservoir* res, uint32_t W, uint32_t H, int x, int y, GIReservoir& r)
    {
        const zr_rgi_reservoir* s = TexelOrNull(res, W, H, x, y);
        r.w_sum = s ? s->w_sum : 0; r.W = s ? s->W : 0;
        r.normal = Math::DecodeOct32(s ? s->normal : 0u);
    }

    // ---- NEE ----
    inline bool IsSpecular(const BSDF::ShadingData& surface)
    {
        return surface.GlossSpecular() && (surface.metallic || surface.specTr) && (!surface.Coated() || surface.CoatSpecular());
    }

    // ReSTIR_GI_NEE.hlsli:8-121 with NumLightSamples = 1. ReSTIR GI compiles it with skipDiffuse = true
    // (MIS_NON_DIFFUSE_BSDF_SAMPLING 1) and approximate shadow rays; the plain path tracer with skipDiffuse = false and
    // APPROXIMATE_EMISSIVE_SHADOW_RAY 0 (PathTracer/Params.hlsli:19-27).
    float3 NEE_Emissive_MIS(const Scene& sc, float3 pos, float3 normal, BSDF::ShadingData surface, uint32_t sampleSetIdx, RNG& rng,
        bool skipDiffuse = true, bool preciseShadow = false)
    {
        float3 ld = f3(0);
        const bool specular = IsSpecular(surface);
        const int numLightSamples = specular ? 0 : 1;
        {
            BSDF::BSDFSample bsdfSample = skipDiffuse ? BSDF::SampleBSDF_NoDiffuse(normal, surface, rng) : BSDF::SampleBSDF(normal, surface, rng);
            float3 wi = bsdfSample.wi;
            float3 f = bsdfSample.f;
            float wiPdf = bsdfSample.pdf;
            HitEmissive hitInfo = FindClosestEmissive(sc, pos, normal, wi, surface.Transmissive());
            if (hitInfo.HitWasEmissive())
            {
                const zr_emissive_tri& emissive = sc.emissives[hitInfo.emissiveTriIdx];
                float3 le = Light::Le_EmissiveTriangle(emissive);
                const float3 vtx0 = Light::Vtx0(emissive);
                const float3 vtx1 = Light::DecodeEmissiveTriV1(emissive);
                const float3 vtx2 = Light::DecodeEmissiveTriV2(emissive);
                float3 lightNormal = cross(vtx1 - vtx0, vtx2 - vtx0);
                float twoArea = length(lightNormal);
                twoArea = fmaxf(twoArea, 1e-6f);
                lightNormal = dot(lightNormal, lightNormal) == 0 ? f3(1.0f) : lightNormal / twoArea;
                lightNormal = Light::IsDoubleSided(emissive) && dot(-wi, lightNormal) < 0 ? -lightNormal : lightNormal;
                const float lightSourcePdf = numLightSamples > 0 ? sc.aliasTable[hitInfo.emissiveTriIdx].CachedP_Orig : 0;
                const float lightPdf = lightSourcePdf * (2.0f / twoArea);
                float dwdA = hitInfo.t > 0 ? saturate(dot(lightNormal, -wi)) / (hitInfo.t * hitInfo.t) : 0;
                wiPdf *= dwdA;
                le *= f * dwdA;
                ld = RT::PowerHeuristic(wiPdf, lightPdf, le, 1, (float)numLightSamples);
            }
        }
        for (int s_l = 0; s_l < numLightSamples; s_l++)
        {
            const Light::LightSample lightSample = Light::SampleLight(sc, pos, sampleSetIdx, rng, false);
            float3 le = lightSample.le;
            const float lightPdf = lightSample.pdf;
            const uint32_t lightID = lightSample.ID;
            const float t = length(lightSample.pos - pos);
            const float3 wi = (lightSample.pos - pos) / t;
            if (dot(lightSample.normal, -wi) > 0)
            {
                const float dwdA = saturate(dot(lightSample.normal, -wi)) / (t * t);
                surface.SetWi(wi, normal);
                le *= BSDF::Unified(surface).f * dwdA;
                if (dot(le, le) > 0)
                    le *= (preciseShadow ? Visibility_Segment_Precise(sc, pos, wi, t, normal, lightID, surface.Transmissive())
                                         : Visibility_Segment(sc, pos, wi, t, normal, lightID, surface.Transmissive())) ? 1.0f : 0.0f;
                float bsdfPdf = skipDiffuse ? BSDF::BSDFSamplerPdf_NoDiffuse(normal, surface, wi) : BSDF::BSDFSamplerPdf(normal, surface, wi, rng);
                bsdfPdf *= dwdA;
                ld += RT::PowerHeuristic(lightPdf, bsdfPdf, le, (float)numLightSamples);
            }
        }
        return ld;
    }

    // NEE.hlsli:152-221 with NumSamples = 1 (only .ld is consumed by the GI path tracer)
    float3 NEE_Emissive_1(const Scene& sc, float3 pos, float3 normal, BSDF::ShadingData surface, uint32_t sampleSetIdx, RNG& rng)
    {
        float3 ret = f3(0);
        const Light::LightSample lightSample = Light::SampleLight(sc, pos, sampleSetIdx, rng, false);
        const float3 le = lightSample.le;
        const float lightPdf = lightSample.pdf;
        const float t = length(lightSample.pos - pos);
        const float3 wi = (lightSample.pos - pos) / t;
        if (dot(lightSample.normal, -wi) > 0)
        {
            const float dwdA = saturate(dot(lightSample.normal, -wi)) / (t * t);
            surface.SetWi(wi, normal);
            float3 ld = le * BSDF::Unified(surface).f * dwdA;
            if (Math::Luminance(ld) > 1e-6f)
                ld *= Visibility_Segment(sc, pos, wi, t, normal, lightSample.ID, surface.Transmissive()) ? 1.0f : 0.0f;
            ret += ld / lightPdf;
        }
        ret = ret / 1.0f;
        return ret;
    }

    // ReSTIR_GI_NEE.hlsli:123-193 with numSamples = 1 (the ReSTIR_GI_LVG variant); extents / offset arrive as halves (ReSTIR_GI.hlsl:52-55)
    float3 NEE_Emissive_LVG(const Scene& sc, const zr_frame_constants& fc, float3 pos, float3 normal, BSDF::ShadingData surface, uint32_t sampleSetIdx, RNG& rng)
    {
        float3 ret = f3(0);
        const float3 extents = f3(to_half(sc.lvgExtents[0]), to_half(sc.lvgExtents[1]), to_half(sc.lvgExtents[2]));
        const float offset_y = to_half(sc.lvgOffsetY);
        zr_voxel_sample s;
        float3 lightPos, lightNormal, le; float lightPdf; uint32_t lightID;
        if (LVG::Sample(sc, pos, extents, offset_y, fc.CurrView, s, rng))
        {
            lightPos = f3(s.pos[0], s.pos[1], s.pos[2]);
            lightNormal = Math::DecodeOct32(s.normal);
            le = f3(zr_f16_to_f32(s.le[0]), zr_f16_to_f32(s.le[1]), zr_f16_to_f32(s.le[2]));
            lightPdf = s.pdf; lightID = s.ID;
            if (s.twoSided && dot(lightNormal, pos - lightPos) < 0)
                lightNormal = -lightNormal;
        }
        else
        {
            const Light::LightSample ls = Light::SampleLight(sc, pos, sampleSetIdx, rng, false);
            lightPos = ls.pos; lightNormal = ls.normal; le = ls.le; lightPdf = ls.pdf; lightID = ls.ID;
        }
        const float t = length(lightPos - pos);
        const float3 wi = (lightPos - pos) / t;
        if (lightID != UINT32_MAX_ && dot(lightNormal, -wi) > 0)
        {
            const float dwdA = saturate(dot(lightNormal, -wi)) / (t * t);
            surface.SetWi(wi, normal);
            le *= BSDF::Unified(surface).f * dwdA;
            if (Math::Luminance(le) > 1e-6f)
                le *= Visibility_Segment(sc, pos, wi, t, normal, lightID, surface.Transmissive()) ? 1.0f : 0.0f;
            ret += le / fmaxf(lightPdf, 1e-6f);
        }
        ret = ret / 1.0f;
        return ret;
    }

    // plainPT: the macro set of IndirectLighting/PathTracer/Params.hlsli -- MIS_ALL_BOUNCES 1, MIS_NON_DIFFUSE_BSDF_SAMPLING 0,
    // APPROXIMATE_EMISSIVE_SHADOW_RAY 0 (ReSTIR_GI_NEE.hlsli:225-238)
    float3 NEE(const Scene& sc, const zr_frame_constants& fc, float3 pos, float3 normal, const BSDF::ShadingData& surface, uint32_t sampleSetIdx, int bounce, RNG& rng,
        bool plainPT = false)
    {
        if (plainPT)
            return NEE_Emissive_MIS(sc, pos, normal, surface, sampleSetIdx, rng, false, true);
        if (bounce == 0)
            return NEE_Emissive_MIS(sc, pos, normal, surface, sampleSetIdx, rng);
        if (sc.lvg && sc.sampleSetSize)
            return NEE_Emissive_LVG(sc, fc, pos, normal, surface, sampleSetIdx, rng);
        return NEE_Emissive_1(sc, pos, normal, surface, sampleSetIdx, rng);
    }

    // ---- the lane of a wave ----
    struct GILane
    {
        bool active = false;        // passed the flags test in main
        bool tracing = false;       // inside PathTrace's loop
        int px = 0, py = 0;
        Pixel p; BSDF::ShadingData surface0;    // primary hit, surface as main builds it (no coat / subsurface / tr depth)
        RNG rngThread, rngGroup;
        int maxNumBounces = 0; uint32_t sampleSetIdx = 0;
        // RIS_InitialCandidates
        BSDF::BSDFSample bsdfSample0; Hit hit0; float3 hitPos0;
        // PathTrace state
        float3 pos, normal, li, throughput; float eta_curr, eta_next; bool inTranslucentMedium; int bounce;
        BSDF::BSDFSample bsdfSample; Hit hitInfo; BSDF::ShadingData surface;
        GIReservoir r;
    };

    // loop top .. Russian-roulette point; false = left the loop
    bool PT_PhaseA(const Scene& sc, const zr_frame_constants& fc, GILane& s, bool plainPT = false)
    {
        const float3 hitPos = mad(s.hitInfo.t, s.bsdfSample.wi, s.pos);
        if (!GetMaterialData(sc, -s.bsdfSample.wi, s.eta_curr, s.hitInfo, s.surface, s.eta_next))
            return false;
        s.li += s.throughput * NEE(sc, fc, hitPos, s.hitInfo.normal, s.surface, s.sampleSetIdx, s.bounce, s.rngThread, plainPT);
        // ACCOUNT_FOR_TRANSMITTANCE == 1 (PathTracing.hlsli:41-48): Beer's law inside a translucent medium
        if (plainPT && s.inTranslucentMedium && (s.surface.trDepth > 0))
        {
            const float3 c = s.surface.baseColor_Fr0_TrCol;
            const float3 extCoeff = f3(-zr_logf(c.x), -zr_logf(c.y), -zr_logf(c.z)) / s.surface.trDepth;
            s.throughput *= f3(zr_expf(-s.hitInfo.t * extCoeff.x), zr_expf(-s.hitInfo.t * extCoeff.y), zr_expf(-s.hitInfo.t * extCoeff.z));
        }
        if (s.bounce >= (s.maxNumBounces - 1))
            return false;
        s.pos = hitPos;
        s.normal = s.hitInfo.normal;
        s.bounce++;
        return true;
    }
    bool PT_PhaseB(const Scene& sc, GILane& s, bool doRR, float waveThroughput)
    {
        if (doRR)
        {
            const float p_terminate = fmaxf(0.05f, 1 - waveThroughput);
            if (s.rngGroup.Uniform() < p_terminate)
                return false;
            s.throughput /= (1 - p_terminate);
        }
        s.bsdfSample = BSDF::BSDFSample::Init();
        if (s.bounce < s.maxNumBounces)
            s.bsdfSample = BSDF::SampleBSDF(s.normal, s.surface, s.rngThread);
        if (Math::Luminance(s.bsdfSample.bsdfOverPdf) == 0)
            return false;
        s.hitInfo = FindClosest(sc, s.pos, s.normal, s.bsdfSample.wi, s.surface.Transmissive());
        if (!s.hitInfo.hit)
            return false;
        s.throughput *= s.bsdfSample.bsdfOverPdf;
        const bool transmitted = dot(s.normal, s.bsdfSample.wi) < 0;
        s.eta_curr = transmitted ? (s.eta_curr == BSDF::ETA_AIR ? s.eta_next : BSDF::ETA_AIR) : s.eta_curr;
        s.inTranslucentMedium = transmitted ? !s.inTranslucentMedium : s.inTranslucentMedium;
        return true;
    }

    // ---- temporal reuse ----
    struct PrevTexel { float depth; GFlags flags; float roughness; float2 normalEnc; float iorEnc; float3 baseColor; };
    PrevTexel LoadPrev(const Frame& f, int x, int y)
    {
        PrevTexel t;
        if (x < 0 || y < 0 || x >= (int)f.W || y >= (int)f.H)
        {
            t.depth = 0; t.flags = DecodeFlags(0); t.roughness = 0; t.normalEnc = f2(0, 0); t.iorEnc = 0; t.baseColor = f3(0);
            return t;
        }
        const GCore g = LoadCore(f.pcore, (size_t)y * f.W + x);
        t.depth = g.depth; t.flags = DecodeFlags(g.flagsByte); t.roughness = g.roughness; t.normalEnc = g.normalEnc; t.iorEnc = g.iorEnc;
        t.baseColor = f3(g.baseColor.x, g.baseColor.y, g.baseColor.z);
        return t;
    }

    struct TemporalSampleData { float3 posW, normal; float roughness; int sx, sy; bool metallic, transmissive; float eta_next; };

    bool PlaneHeuristic(float3 samplePos, float3 currNormal, float3 currPos, float linearDepth, float th)
    {
        return fabsf(dot(currNormal, samplePos - currPos)) <= th * linearDepth;
    }

    float3 PrevCamPos(const zr_frame_constants& fc) { return f3(fc.PrevViewInv[0][3], fc.PrevViewInv[1][3], fc.PrevViewInv[2][3]); }

    int FindTemporalCandidate(const Frame& f, int x, int y, float3 posW, float3 normal, float viewZ, float roughness, bool transmissive,
        float2 prevUV, RNG& rng, TemporalSampleData data[2], bool valid[2])
    {
        const zr_frame_constants& fc = *f.fc;
        valid[0] = valid[1] = false;
        if (prevUV.x < 0.0f || prevUV.y < 0.0f || prevUV.x > 1.0f || prevUV.y > 1.0f)
            return 0;
        const float2 renderDim = f2((float)f.W, (float)f.H);
        const float2 pp = prevUV * renderDim;
        const int prevPixelX = (int)pp.x, prevPixelY = (int)pp.y;
        int curr = 0;
        const float3 prevCamPos = PrevCamPos(fc);
        for (int i = 0; i < 3; i++)
        {
            const float theta = rng.Uniform() * TWO_PI;
            float sinTheta, cosTheta;
            zr_sincosf(theta, &sinTheta, &cosTheta);
            const float2 offset = f2(16.0f * sinTheta, 16.0f * cosTheta);
            const float m = i > 0 ? 1.0f : 0.0f;
            const int sx = (int)((float)prevPixelX + m * offset.x), sy = (int)((float)prevPixelY + m * offset.y);
            if ((float)sx >= renderDim.x || (float)sy >= renderDim.y)
                continue;
            if (i > 0 && (uint32_t)sx == (uint32_t)x && (uint32_t)sy == (uint32_t)y)
                continue;
            const PrevTexel t = LoadPrev(f, sx, sy);
            if (t.flags.emissive)
                continue;
            float2 lensSample = f2(0, 0);
            float3 origin = prevCamPos;
            if (fc.DoF)
            {
                uint3 h = RNG::PCG3d(uint3{ (uint32_t)sx, (uint32_t)sy, (uint32_t)sx });
                RNG rngDoF = RNG::Init(h.z, h.y, fc.FrameNum - 1);
                lensSample = Sampling::UniformSampleDiskConcentric(rngDoF.Uniform2D());
                lensSample = lensSample * fc.LensRadius;
            }
            const float3 prevPos = Math::WorldPosFromScreenSpace2(f2((float)sx, (float)sy), renderDim, t.depth, fc.TanHalfFOV, fc.AspectRatio,
                f2(fc.PrevCameraJitter[0], fc.PrevCameraJitter[1]), row3(fc.PrevView, 0), row3(fc.PrevView, 1), row3(fc.PrevView, 2),
                fc.DoF != 0, lensSample, fc.FocusDepth, origin);
            const float tolerance = 0.005f * (fc.DoF ? 10.0f : 1.0f);
            if (!PlaneHeuristic(prevPos, normal, posW, viewZ, tolerance))
                continue;
            const float3 prevNormal = Math::DecodeUnitVector(t.normalEnc);
            bool ok = dot(prevNormal, normal) > 0.1f;
            if (roughness < 0.5f)
                ok = ok && (fabsf(t.roughness - roughness) < 0.15f);
            float prevEta_mat = BSDF::DEFAULT_ETA_MAT;
            if (t.flags.transmissive)
                prevEta_mat = DecodeIOR(t.iorEnc);
            ok = ok && (t.flags.transmissive == transmissive);
            ok = fc.DoF ? true : ok;
            valid[curr] = ok;
            if (ok)
            {
                TemporalSampleData& d = data[curr];
                d.sx = (int)(int16_t)sx; d.sy = (int)(int16_t)sy;
                d.posW = prevPos; d.normal = prevNormal; d.metallic = t.flags.metallic; d.roughness = t.roughness;
                d.transmissive = t.flags.transmissive; d.eta_next = prevEta_mat;
                curr++;
                if (curr == 2)
                    break;
            }
        }
        return curr;
    }

    float TargetLumAtTemporalPixel(const Frame& f, const GIReservoir& r_curr, const TemporalSampleData& c, bool testVisibility)
    {
        const zr_frame_constants& fc = *f.fc;
        float3 wi = r_curr.pos - c.posW;
        if (dot(wi, wi) == 0)
            return 0;
        const float t = length(wi);
        wi = wi / fmaxf(t, 1e-6f);
        const float3 baseColor_prev = LoadPrev(f, c.sx, c.sy).baseColor;
        float3 camPos_prev = PrevCamPos(fc);
        if (fc.DoF)
        {
            uint3 h = RNG::PCG3d(uint3{ (uint32_t)c.sx, (uint32_t)c.sy, (uint32_t)c.sx });
            RNG rngDoF = RNG::Init(h.z, h.y, fc.FrameNum - 1);
            float2 lensSample = Sampling::UniformSampleDiskConcentric(rngDoF.Uniform2D());
            lensSample = lensSample * fc.LensRadius;
            camPos_prev += mad(lensSample.x, row3(fc.PrevView, 0), lensSample.y * row3(fc.PrevView, 1));
        }
        const float3 wo_prev = normalize(camPos_prev - c.posW);
        BSDF::ShadingData surface_prev = BSDF::ShadingData::Init(c.normal, wo_prev, c.metallic, c.roughness, baseColor_prev, BSDF::ETA_AIR,
            c.eta_next, c.transmissive);
        surface_prev.SetWi(wi, c.normal);
        const float3 target_prev = r_curr.Lo * BSDF::Unified(surface_prev).f;
        const float targetLum_prev = Math::Luminance(target_prev);
        if (testVisibility && targetLum_prev > 1e-5f)
        {
            if (!Visibility_Segment(*f.sc, c.posW, wi, t, c.normal, r_curr.ID, surface_prev.Transmissive()))
                return 0;
        }
        return targetLum_prev;
    }

    float JacobianReconnectionShift(float3 x2_normal, float3 x1_r, float3 x1_q, float3 x2_q)
    {
        float3 v_r = x1_r - x2_q;
        const float t_r2 = dot(v_r, v_r);
        v_r = dot(v_r, v_r) == 0 ? v_r : v_r / fmaxf(sqrtf(t_r2), 1e-6f);
        float3 v_q = x1_q - x2_q;
        const float t_q2 = dot(v_q, v_q);
        v_q = dot(v_q, v_q) == 0 ? v_q : v_q / fmaxf(sqrtf(t_q2), 1e-6f);
        const float cosPhi_r = dot(v_r, x2_normal);
        const float cosPhi_q = dot(v_q, x2_normal);
        return (fabsf(cosPhi_r) * t_q2) / fmaxf(fabsf(cosPhi_q) * t_r2, 1e-6f);
    }

    void TemporalResample1(const Frame& f, const zr_rgi_reservoir* prevRes, float3 posW, float3 normal, BSDF::ShadingData surface,
        const TemporalSampleData& c, GIReservoir& r, RNG& rng)
    {
        GIReservoir r_prev = PartialReadReservoir_Reuse(prevRes, f.W, f.H, c.sx, c.sy);
        const float M_new = (float)(uint16_t)(r.M + r_prev.M);
        if (r.w_sum != 0)
        {
            float targetLum_prev = 0.0f;
            if (r_prev.M > 0 && Math::Luminance(r.Lo) > 1e-6f)
                targetLum_prev = TargetLumAtTemporalPixel(f, r, c, true);
            const float p_curr = Math::Luminance(r.target_z);
            const float J_curr_to_temporal = JacobianReconnectionShift(r.normal, c.posW, posW, r.pos);
            const float m_curr = p_curr / fmaxf(p_curr + r_prev.M * targetLum_prev * J_curr_to_temporal, 1e-6f);
            r.w_sum *= m_curr;
        }
        if (r_prev.ID == UINT32_MAX_ || (r_prev.Lo.x + r_prev.Lo.y + r_prev.Lo.z) == 0)
        {
            const float targetLum = Math::Luminance(r.target_z);
            r.W = targetLum > 0.0f ? r.w_sum / targetLum : 0.0f;
            r.M = M_new;
            return;
        }
        float3 wi = r_prev.pos - posW;
        const float t = length(wi);
        wi = wi / t;
        surface.SetWi(wi, normal);
        const float3 target_curr = r_prev.Lo * BSDF::Unified(surface).f;
        const float targetLum_curr = Math::Luminance(target_curr);
        if (targetLum_curr > 1e-6f)
        {
            if (Visibility_Segment(*f.sc, posW, wi, t, normal, r_prev.ID, surface.Transmissive()))
            {
                PartialReadReservoir_ReuseRest(prevRes, f.W, f.H, c.sx, c.sy, r_prev);
                const float targetLum_prev = r_prev.W > 0 ? r_prev.w_sum / r_prev.W : 0;
                const float J_temporal_to_curr = JacobianReconnectionShift(r_prev.normal, posW, c.posW, r_prev.pos);
                const float numerator = r_prev.M * targetLum_prev;
                const float denom = numerator / fmaxf(J_temporal_to_curr, 1e-6f) + targetLum_curr;
                const float m_prev = numerator / fmaxf(denom, 1e-6f);
                const float w_prev = m_prev * targetLum_curr * r_prev.W;
                r.Update(w_prev, r_prev.pos, r_prev.normal, r_prev.ID, r_prev.Lo, target_curr, rng);
            }
        }
        const float targetLum = Math::Luminance(r.target_z);
        r.W = targetLum > 0.0f ? r.w_sum / targetLum : 0.0f;
        r.M = M_new;
    }

    void TemporalResample2(const Frame& f, const zr_rgi_reservoir* prevRes, float3 posW, float3 normal, BSDF::ShadingData surface,
        const TemporalSampleData c[2], GIReservoir& r, RNG& rng)
    {
        uint16_t M_new = (uint16_t)r.M;
        GIReservoir r_prev[2];
        for (int k = 0; k < 2; k++)
        {
            r_prev[k] = PartialReadReservoir_Reuse(prevRes, f.W, f.H, c[k].sx, c[k].sy);
            M_new = (uint16_t)(M_new + (uint16_t)r_prev[k].M);
        }
        {
            const float p_curr = Math::Luminance(r.target_z);
            float denom = p_curr;
            if (Math::Luminance(r.Lo) > 1e-5f)
            {
                for (int p = 0; p < 2; p++)
                {
                    if (r_prev[p].M == 0)
                        continue;
                    const float targetLum_prev = TargetLumAtTemporalPixel(f, r, c[p], p != 0);
                    const float J_curr_to_temporal = JacobianReconnectionShift(r.normal, c[p].posW, posW, r.pos);
                    denom += r_prev[p].M * J_curr_to_temporal * targetLum_prev;
                }
            }
            const float m_curr = denom == 0 ? 0 : p_curr / denom;
            r.w_sum *= m_curr;
        }
        for (int i = 0; i < 2; i++)
        {
            float3 wi = r_prev[i].pos - posW;
            const float t = (wi.x == 0 && wi.y == 0 && wi.z == 0) ? 0 : length(wi);
            wi = wi / fmaxf(t, 1e-6f);
            surface.SetWi(wi, normal);
            const float3 target_curr = r_prev[i].Lo * BSDF::Unified(surface).f;
            const float targetLum_curr = Math::Luminance(target_curr);
            if (targetLum_curr < 1e-5f)
                continue;
            if (Visibility_Segment(*f.sc, posW, wi, t, normal, r_prev[i].ID, surface.Transmissive()))
            {
                PartialReadReservoir_ReuseRest(prevRes, f.W, f.H, c[i].sx, c[i].sy, r_prev[i]);
                const float targetLum_prev = r_prev[i].W > 0 ? r_prev[i].w_sum / r_prev[i].W : 0;
                const float J_temporal_to_curr = JacobianReconnectionShift(r_prev[i].normal, posW, c[i].posW, r_prev[i].pos);
                const float numerator = r_prev[i].M * targetLum_prev;
                float denom = (numerator / J_temporal_to_curr) + targetLum_curr;
                if (r_prev[1 - i].M > 0 && targetLum_prev > 0)
                {
                    const float J_temporal_to_temporal = JacobianReconnectionShift(r_prev[i].normal, c[1 - i].posW, c[i].posW, r_prev[i].pos);
                    const float targetLum_other = TargetLumAtTemporalPixel(f, r_prev[i], c[1 - i], true);
                    denom += r_prev[1 - i].M * targetLum_other / fmaxf(J_temporal_to_temporal, 1e-6f);
                }
                denom = J_temporal_to_curr == 0 ? 0 : denom;
                const float m_prev = denom == 0 ? 0 : numerator / denom;
                const float w_prev = m_prev * targetLum_curr * r_prev[i].W;
                r.Update(w_prev, r_prev[i].pos, r_prev[i].normal, r_prev[i].ID, r_prev[i].Lo, target_curr, rng);
            }
        }
        const float targetLum = Math::Luminance(r.target_z);
        r.W = targetLum > 0.0f ? r.w_sum / targetLum : 0.0f;
        r.M = (float)M_new;
    }

    float WaveSum32(const float v[32])
    {
        float a[32];
        for (int i = 0; i < 32; i++) a[i] = v[i];
        for (int off = 16; off >= 1; off >>= 1)
        {
            float b[32];
            for (int i = 0; i < 32; i++) b[i] = a[i] + a[i ^ off];
            for (int i = 0; i < 32; i++) a[i] = b[i];
        }
        return a[0];
    }

    // plainPT: IndirectLighting/PathTracer/PathTracer.hlsl (INTEGRATOR::PATH_TRACING): same dispatch shape, RNG seeds and
    // PathTrace loop, no reservoirs / reuse; main :98-212, EstimateIndirectLighting :58-104
    void RenderPass(const Frame& f, const GIParams& prm, bool doTemporal, bool resetTemporal, zr_rgi_reservoir* resCurr,
        const zr_rgi_reservoir* resPrev, float4* finalImg, int nthreads, bool plainPT = false)
    {
        const zr_frame_constants& fc = *f.fc;
        const Scene& sc = *f.sc;
        const uint32_t dispX = (f.W + 7) / 8, dispY = (f.H + 7) / 8;
        const uint32_t numGroupsInTile = 16 * dispY;
        const uint32_t numWaves = dispX * dispY * 2;
        parallel_for(numWaves, nthreads, [&](uint32_t w0, uint32_t w1)
        {
            std::vector<GILane> lanes(32);
            for (uint32_t wv = w0; wv < w1; wv++)
            {
                const uint32_t group = wv / 2, wave = wv % 2;
                const uint32_t Gx = group % dispX, Gy = group / dispX;
                for (int l = 0; l < 32; l++)
                {
                    GILane& s = lanes[l];
                    s = GILane();
                    uint32_t sx, sy, sgx, sgy;
                    SwizzleThreadGroup(Gx, Gy, l % 8, wave * 4 + l / 8, 8, 8, dispX, 16, 4, numGroupsInTile, sx, sy, sgx, sgy);
                    if (sx >= f.W || sy >= f.H)
                        continue;
                    s.px = (int)sx; s.py = (int)sy;
                    const size_t idx = (size_t)sy * f.W + sx;
                    const GFlags flags = FlagsAt(f.core, f.W, sx, sy);
                    if (flags.invalid || flags.emissive)
                    {
                        if (!fc.Accumulate || !fc.CameraStatic)
                            finalImg[idx] = f4(0, 0, 0, finalImg[idx].w);
                        continue;
                    }
                    s.active = true;
                    s.p = LoadPixel(f, f.core, f.coat, sx, sy, false, sx, sy);
                    const GCore g = LoadCore(f.core, idx);
                    const float3 wo = normalize(s.p.origin - s.p.pos);
                    if (plainPT)        // PathTracer.hlsl:184-185 also passes flags.trDepthGt0 as the transmission depth
                        s.surface0 = BSDF::ShadingData::Init(s.p.normal, wo, flags.metallic, g.roughness, f3(g.baseColor.x, g.baseColor.y, g.baseColor.z),
                            BSDF::ETA_AIR, s.p.eta_next, flags.transmissive, flags.trDepthGt0 ? 1.0f : 0.0f);
                    else
                    s.surface0 = BSDF::ShadingData::Init(s.p.normal, wo, flags.metallic, g.roughness, f3(g.baseColor.x, g.baseColor.y, g.baseColor.z),
                        BSDF::ETA_AIR, s.p.eta_next, flags.transmissive);
                    s.rngGroup = RNG::Init(sgx ^ 61u, sgy ^ 61u, fc.FrameNum);
                    s.rngThread = RNG::Init(sx ^ 511u, sy ^ 31u, fc.FrameNum);
                    s.maxNumBounces = (int)(flags.transmissive ? prm.maxGlossyTrBounces : prm.maxNonTrBounces);
                    // EstimateIndirectLighting
                    if (!plainPT && prm.stochasticMultiBounce && (g.roughness >= 0.1f || fc.CameraStatic))
                        s.maxNumBounces = s.rngGroup.Uniform() < 0.5f ? 1 : s.maxNumBounces;
                    s.sampleSetIdx = s.rngGroup.UniformUintBounded_Faster(sc.numSampleSets);
                    // RIS_InitialCandidates up to the path-tracing loop
                    s.r = GIReservoir::Init();
                    s.bsdfSample0 = BSDF::SampleBSDF(s.p.normal, s.surface0, s.rngThread);
                    if (s.bsdfSample0.pdf == 0)
                        continue;
                    s.hit0 = FindClosest(sc, s.p.pos, s.p.normal, s.bsdfSample0.wi, s.surface0.Transmissive());
                    if (!s.hit0.hit)
                        continue;
                    s.hitPos0 = s.p.pos + s.hit0.t * s.bsdfSample0.wi;
                    // PathTrace prologue
                    s.pos = s.p.pos; s.normal = s.p.normal;
                    s.li = f3(0); s.throughput = f3(1.0f);
                    s.eta_curr = dot(s.normal, s.bsdfSample0.wi) < 0 ? s.p.eta_next : BSDF::ETA_AIR;
                    s.eta_next = BSDF::DEFAULT_ETA_MAT;
                    s.bounce = 0;
                    s.inTranslucentMedium = dot(s.normal, s.bsdfSample0.wi) < 0;
                    s.bsdfSample = s.bsdfSample0; s.hitInfo = s.hit0;
                    s.tracing = true;
                }
                // lock-step bounce loop
                for (;;)
                {
                    bool any = false, atRR[32];
                    for (int l = 0; l < 32; l++)
                    {
                        atRR[l] = false;
                        GILane& s = lanes[l];
                        if (!s.tracing) continue;
                        if (!PT_PhaseA(sc, fc, s, plainPT)) { s.tracing = false; continue; }
                        atRR[l] = true; any = true;
                    }
                    if (!any) break;
                    float waveMax = -FLT_MAX_;
                    bool doRR = false;
                    for (int l = 0; l < 32; l++)
                        if (atRR[l])
                        {
                            doRR = prm.russianRoulette && (lanes[l].bounce >= 3);
                            waveMax = fmaxf(waveMax, Math::Luminance(lanes[l].throughput));
                        }
                    for (int l = 0; l < 32; l++)
                        if (atRR[l] && !PT_PhaseB(sc, lanes[l], doRR, waveMax))
                            lanes[l].tracing = false;
                }
                if (plainPT)
                {
                    // EstimateIndirectLighting :97-103, main :199-211
                    for (int l = 0; l < 32; l++)
                    {
                        GILane& s = lanes[l];
                        if (!s.active) continue;
                        float3 li = f3(0);
                        if (s.bsdfSample0.pdf != 0 && s.hit0.hit)
                        {
                            li = s.li;
                            if (dot(li, li) > 0)
                                li *= s.bsdfSample0.bsdfOverPdf;
                        }
                        li = isnan3(li) ? f3(0) : li;       // any(isnan(li)) ? 0 : li
                        const size_t idx = (size_t)s.py * f.W + s.px;
                        if (fc.Accumulate && fc.CameraStatic)
                        {
                            const float4 prev = finalImg[idx];
                            finalImg[idx] = f4(prev.x + li.x, prev.y + li.y, prev.z + li.z, prev.w);
                        }
                        else
                            finalImg[idx] = f4(li.x, li.y, li.z, finalImg[idx].w);
                    }
                    continue;
                }
                // rest of RIS_InitialCandidates, temporal reuse
                float wsum[32];
                for (int l = 0; l < 32; l++)
                {
                    GILane& s = lanes[l];
                    wsum[l] = 0;
                    if (!s.active) continue;
                    if (s.bsdfSample0.pdf != 0 && s.hit0.hit)
                    {
                        const float3 lo = s.li;
                        float3 target = lo;
                        if (dot(lo, lo) > 0)
                        {
                            s.surface0.SetWi(s.bsdfSample0.wi, s.p.normal);
                            target *= BSDF::Unified(s.surface0).f;
                        }
                        const float targetLum = Math::Luminance(target);
                        const float w = targetLum / fmaxf(s.bsdfSample0.pdf, 1e-6f);
                        s.r.Update(w, s.hitPos0, s.hit0.normal, s.hit0.ID, lo, target, s.rngThread);
                        s.r.W = targetLum > 0 ? 1.0f / s.bsdfSample0.pdf : 0.0f;
                    }
                    if (doTemporal)
                    {
                        const float2 renderDim = f2((float)f.W, (float)f.H);
                        const float2 motionVec = unpack_snorm16x2(f.me[(size_t)s.py * f.W + s.px].x);
                        const float2 currUV = f2((float)s.px + 0.5f, (float)s.py + 0.5f) / renderDim;
                        const float2 prevUV = currUV - motionVec;
                        TemporalSampleData data[2]; bool valid[2];
                        const GCore g = LoadCore(f.core, (size_t)s.py * f.W + s.px);
                        FindTemporalCandidate(f, s.px, s.py, s.p.pos, s.p.normal, s.p.z, g.roughness, s.surface0.specTr, prevUV, s.rngThread, data, valid);
                        if (valid[1] && g.roughness > 0.05f)
                            TemporalResample2(f, resPrev, s.p.pos, s.p.normal, s.surface0, data, s.r, s.rngThread);
                        else if (valid[0])
                            TemporalResample1(f, resPrev, s.p.pos, s.p.normal, s.surface0, data[0], s.r, s.rngThread);
                    }
                    wsum[l] = s.r.w_sum;
                }
                if (doTemporal && prm.boilingSuppression)
                {
                    const float waveSum = WaveSum32(wsum);
                    for (int l = 0; l < 32; l++)
                    {
                        GILane& s = lanes[l];
                        if (!s.active) continue;
                        const float waveAvg = (waveSum - s.r.w_sum) / 31.0f;
                        if (s.r.w_sum > 25 * waveAvg)
                            s.r.M = 1;
                    }
                }
                for (int l = 0; l < 32; l++)
                {
                    GILane& s = lanes[l];
                    if (!s.active) continue;
                    const size_t idx = (size_t)s.py * f.W + s.px;
                    if (doTemporal || resetTemporal)
                        WriteReservoir(resCurr[idx], s.r, (float)prm.M_max);
                    float3 li = s.r.target_z * s.r.W;
                    li = isnan3(li) ? f3(0) : li;
                    if (fc.Accumulate && fc.CameraStatic)
                    {
                        const float4 prev = finalImg[idx];
                        finalImg[idx] = f4(prev.x + li.x, prev.y + li.y, prev.z + li.z, prev.w);
                    }
                    else
                        finalImg[idx] = f4(li.x, li.y, li.z, finalImg[idx].w);
                }
            }
        });
    }
}
}

extern "C"
{
    // Probe for the CPU-tier device-source parity test (tests/test_device_source_vs_oracle.py): ReSTIR GI's temporal reuse at one pixel,
    // starting from a given initial reservoir record. Mirrors EstimateIndirectLighting :564-596 (candidate search, one- or
    // two-candidate resampling). out: the resulting 48-byte record, then target_z (3 words), rng state, #valid candidates.
    void orc_probe_rgi_temporal(void* scene, const zr_frame_constants* fc, const uint32_t* core_, const uint32_t* me_, const uint32_t* coat_,
        const uint32_t* pcore_, const uint32_t* pcoat_, const zr_rgi_reservoir* prevRes, const zr_rgi_reservoir* initial, int x, int y,
        uint32_t seed, uint32_t M_max, uint32_t* out)
    {
        using namespace orc;
        const uint4* core = (const uint4*)core_;
        const uint2* me = (const uint2*)me_;
        const uint2* coat = (const uint2*)coat_;
        const uint4* pcore = (const uint4*)pcore_;
        const uint2* pcoat = (const uint2*)pcoat_;
        Frame f;
        f.sc = (const Scene*)scene; f.fc = fc; f.core = core; f.me = me; f.coat = coat; f.pcore = pcore; f.pcoat = pcoat;
        f.W = fc->RenderWidth; f.H = fc->RenderHeight;
        memset(out, 0, 17 * 4);
        const size_t idx = (size_t)y * f.W + x;
        const GFlags flags = FlagsAt(core, f.W, x, y);
        if (flags.invalid || flags.emissive) return;
        Pixel p = LoadPixel(f, core, coat, x, y, false, x, y);
        const GCore g = LoadCore(core, idx);
        const float3 wo = normalize(p.origin - p.pos);
        BSDF::ShadingData surface0 = BSDF::ShadingData::Init(p.normal, wo, flags.metallic, g.roughness, f3(g.baseColor.x, g.baseColor.y, g.baseColor.z),
            BSDF::ETA_AIR, p.eta_next, flags.transmissive);
        GIReservoir r = GIReservoir::Init();
        r.pos = f3(initial->pos[0], initial->pos[1], initial->pos[2]); r.ID = initial->ID;
        r.Lo = f3(zr_f16_to_f32((uint16_t)(initial->Lo_rg & 0xffff)), zr_f16_to_f32((uint16_t)(initial->Lo_rg >> 16)), zr_f16_to_f32((uint16_t)(initial->Lo_b_M & 0xffff)));
        r.M = (float)(uint16_t)zr_f16_to_f32((uint16_t)(initial->Lo_b_M >> 16));
        r.w_sum = initial->w_sum; r.W = initial->W; r.normal = Math::DecodeOct32(initial->normal);
        if (r.ID != UINT32_MAX_)
        {
            float3 wi = r.pos - p.pos;
            const float t = length(wi);
            wi = wi / fmaxf(t, 1e-6f);
            surface0.SetWi(wi, p.normal);
            r.target_z = r.Lo * BSDF::Unified(surface0).f;
        }
        RNG rng = RNG::InitSeed(seed);
        const float2 renderDim = f2((float)f.W, (float)f.H);
        const float2 motionVec = unpack_snorm16x2(me[idx].x);
        const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / renderDim;
        const float2 prevUV = currUV - motionVec;
        TemporalSampleData data[2]; bool valid[2];
        FindTemporalCandidate(f, x, y, p.pos, p.normal, p.z, g.roughness, surface0.specTr, prevUV, rng, data, valid);
        if (valid[1] && g.roughness > 0.05f)
            TemporalResample2(f, prevRes, p.pos, p.normal, surface0, data, r, rng);
        else if (valid[0])
            TemporalResample1(f, prevRes, p.pos, p.normal, surface0, data[0], r, rng);
        zr_rgi_reservoir rec;
        WriteReservoir(rec, r, (float)M_max);
        memcpy(out, &rec, 48);
        out[12] = asuint(r.target_z.x); out[13] = asuint(r.target_z.y); out[14] = asuint(r.target_z.z);
        out[15] = rng.State; out[16] = (valid[0] ? 1u : 0u) + (valid[1] ? 1u : 0u);
    }

    // IndirectLighting with INTEGRATOR::PATH_TRACING (IndirectLighting.cpp: RenderPathTracer; PathTracer/PathTracer.hlsl), emissive NEE.
    // Of the parameters only the bounce budgets and the Russian-roulette flag are read.
    void orc_pt_render(void* scene, const zr_frame_constants* fc, const uint32_t* core_, const uint32_t* me_, const uint32_t* coat_,
        const zr_gi_params* p, float* finalImg_, int nthreads)
    {
        using namespace orc;
        const uint4* core = (const uint4*)core_;
        const uint2* me = (const uint2*)me_;
        const uint2* coat = (const uint2*)coat_;
        float4* finalImg = (float4*)finalImg_;
        Frame f;
        f.sc = (const Scene*)scene; f.fc = fc; f.core = core; f.me = me; f.coat = coat; f.pcore = core; f.pcoat = coat;
        f.W = fc->RenderWidth; f.H = fc->RenderHeight;
        const GIParams prm{ p->max_non_tr_bounces, p->max_glossy_tr_bounces, p->russian_roulette, p->stochastic_multi_bounce,
            p->boiling_suppression, p->M_max, p->temporal_resample };
        RenderPass(f, prm, false, false, nullptr, nullptr, finalImg, nthreads, true);
    }

    // state[0] = currTemporalIdx, state[1] = isTemporalReservoirValid, state[2] = reset flag (IndirectLighting.cpp:277-368, :1021-1024)
    void orc_rgi_render(void* scene, const zr_frame_constants* fc, const uint32_t* core_, const uint32_t* me_, const uint32_t* coat_,
        const uint32_t* pcore_, const uint32_t* pcoat_, const zr_gi_params* p, zr_rgi_reservoir* res0, zr_rgi_reservoir* res1,
        float* finalImg_, uint32_t* state, int nthreads)
    {
        using namespace orc;
        const uint4* core = (const uint4*)core_;
        const uint2* me = (const uint2*)me_;
        const uint2* coat = (const uint2*)coat_;
        const uint4* pcore = (const uint4*)pcore_;
        const uint2* pcoat = (const uint2*)pcoat_;
        float4* finalImg = (float4*)finalImg_;
        Frame f;
        f.sc = (const Scene*)scene; f.fc = fc; f.core = core; f.me = me; f.coat = coat; f.pcore = pcore; f.pcoat = pcoat;
        f.W = fc->RenderWidth; f.H = fc->RenderHeight;
        const GIParams prm{ p->max_non_tr_bounces, p->max_glossy_tr_bounces, p->russian_roulette, p->stochastic_multi_bounce,
            p->boiling_suppression, p->M_max, p->temporal_resample };
        zr_rgi_reservoir* res[2] = { res0, res1 };
        const int cur = (int)state[0];
        const bool doTemporal = prm.temporalResample && state[1];
        RenderPass(f, prm, doTemporal, state[2] != 0, res[cur], res[1 - cur], finalImg, nthreads);
        state[1] = 1;
        state[0] = 1 - cur;
        state[2] = 0;
    }
}
