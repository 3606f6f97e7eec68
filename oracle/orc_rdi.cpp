// ORACLE -- test infrastructure, not product code (see orc_math.h header).
//
// CPU restatement of ReSTIR DI for emissive triangles (SURVEY 8a-12):
//   DirectLighting/Emissive/ReSTIR_DI_Temporal.hlsl  RIS_InitialCandidates :29-188, EstimateDirectLighting :190-244, main :250-390
//   DirectLighting/Emissive/ReSTIR_DI_Spatial.hlsl   main :27-192
//   DirectLighting/Emissive/Resampling.hlsli         FindTemporalCandidate :36-130, OffsetPathTarget_CtT/TtC :132-274,
//                                                    TemporalResample1 :276-339, SpatialResample :341-519
//   DirectLighting/Emissive/PairwiseMIS.hlsli        :10-232
//   DirectLighting/Emissive/Reservoir.hlsli          :10-213 (A RGBA32UI + B RG32F -> one 32-byte record)
//   DirectLighting/Emissive/Util.hlsli               EmissiveData :9-57, FindClosestHit :68-120
//   DirectLighting/Emissive/DirectLighting.cpp:166-284 host sequencing
// Compiled configuration: USE_HALF_VECTOR_COPY_SHIFT 0, no presampled sets (Params.hlsli:4-17).
// Parity unpinned: the reference has no tests for this code.
#include "orc_api.h"
#include "orc_pixel.h"

using namespace orc;

namespace
{
    struct DIParams { uint32_t temporal, spatial, stochasticSpatial, extraDisocclusion, M_max; float alpha_min; uint32_t reset; };

    struct Reservoir
    {
        float w_sum, W; float3 le; uint32_t lightIdx; float2 bary; uint32_t M;
        float3 target; uint32_t lightID; float3 lightPos, lightNormal; bool doubleSided;

        static Reservoir Init()
        {
            Reservoir r;
            r.le = f3(0); r.M = 0; r.w_sum = 0; r.W = 0; r.lightIdx = UINT32_MAX_; r.bary = f2(0, 0);
            r.target = f3(0); r.lightID = UINT32_MAX_; r.lightPos = f3(0); r.lightNormal = f3(0); r.doubleSided = false;
            return r;
        }
        bool Update(float weight, float3 le_, uint32_t lightIdx_, float2 bary_, RNG& rng)
        {
            if (weight != weight) return false;
            M += 1;
            if (weight == 0) return false;
            w_sum += weight;
            if (rng.Uniform() < (weight / w_sum))
            {
                le = le_; lightIdx = lightIdx_; bary = bary_;
                return true;
            }
            return false;
        }
        static Reservoir Load(const zr_rdi_reservoir& s)
        {
            Reservoir r = Init();
            r.le = f3(half_lo(s.le_rg), half_hi(s.le_rg), half_lo(s.le_b_meta));
            r.M = (s.le_b_meta >> 16) & 0x1f;
            r.w_sum = s.w_sum; r.W = s.W;
            r.lightIdx = s.lightIdx;
            r.bary = Math::DecodeUNorm2(s.bary);
            return r;
        }
        void Write(zr_rdi_reservoir& s, uint32_t M_max) const
        {
            uint32_t M_capped = M < M_max ? M : M_max;
            s.bary = Math::EncodeUNorm2(bary);
            s.le_rg = pack_half2(le.x, le.y);
            s.le_b_meta = (uint32_t)zr_f32_to_f16(le.z) | (M_capped << 16);
            s.lightIdx = lightIdx;
            s.w_sum = w_sum; s.W = W;
            s.pad[0] = 0; s.pad[1] = 0;
        }
    };

    // RGBA16F target plane
    void WriteTarget(uint2* target, size_t idx, float3 t)
    {
        t = Math::Sanitize(t);
        target[idx] = uint2{ pack_half2(t.x, t.y), pack_half2(t.z, 0.0f) };
    }
    float3 LoadTarget(const uint2* target, size_t idx)
    {
        uint2 p = target[idx];
        return f3(half_lo(p.x), half_hi(p.x), half_lo(p.y));
    }

    struct BSDFHitInfo { uint32_t emissiveTriIdx; float2 bary; float3 lightPos; float t; bool hit; };

    // Util.hlsli:68-120
    BSDFHitInfo FindClosestHitDI(const Scene& sc, float3 pos, float3 normal, float3 wi, bool transmissive)
    {
        BSDFHitInfo ret;
        ret.hit = false; ret.emissiveTriIdx = UINT32_MAX_; ret.bary = f2(0, 0); ret.lightPos = f3(0); ret.t = 0;
        float ndotwi = dot(normal, wi);
        if (ndotwi == 0) return ret;
        bool wiBackface = ndotwi < 0;
        if (wiBackface)
        {
            if (transmissive) normal = -normal;
            else return ret;
        }
        const float3 adjustedOrigin = RTU::OffsetRayRTG(pos, normal);
        RayHit h = sc.Closest(adjustedOrigin, wi, wiBackface ? 3e-4f : 0.0f, FLT_MAX_);
        if (h.hit)
        {
            const uint32_t meshIdx = sc.triMesh[h.tri];
            const zr_mesh_instance& meshData = sc.instances[meshIdx];
            if (meshData.BaseEmissiveTriOffset == UINT32_MAX_)
                return ret;
            ret.emissiveTriIdx = meshData.BaseEmissiveTriOffset + sc.triPrim[h.tri];
            ret.bary = h.bary;
            ret.lightPos = mad(h.t, wi, adjustedOrigin);
            ret.t = h.t;
            ret.hit = true;
        }
        return ret;
    }

    // Util.hlsli:9-57
    struct EmissiveData
    {
        float3 wi; float t; uint32_t ID; float3 lightPos, lightNormal; bool doubleSided;
        static EmissiveData Init(const Scene& sc, uint32_t lightIdx, float2 bary)
        {
            EmissiveData ret;
            const zr_emissive_tri& tri = sc.emissives[lightIdx];
            ret.ID = tri.ID;
            const float3 vtx0 = Light::Vtx0(tri);
            const float3 vtx1 = Light::DecodeEmissiveTriV1(tri);
            const float3 vtx2 = Light::DecodeEmissiveTriV2(tri);
            ret.lightPos = (1.0f - bary.x - bary.y) * vtx0 + bary.x * vtx1 + bary.y * vtx2;
            ret.lightNormal = cross(vtx1 - vtx0, vtx2 - vtx0);
            ret.lightNormal = dot(ret.lightNormal, ret.lightNormal) == 0 ? ret.lightNormal : normalize(ret.lightNormal);
            ret.doubleSided = Light::IsDoubleSided(tri);
            ret.wi = f3(0); ret.t = 0;
            return ret;
        }
        void SetSurfacePos(float3 pos)
        {
            wi = lightPos - pos;
            t = dot(wi, wi) == 0 ? 0 : length(wi);
            wi = t == 0 ? f3(0) : wi / t;
            lightNormal = doubleSided && dot(-wi, lightNormal) < 0 ? -lightNormal : lightNormal;
        }
        float dWdA() const
        {
            float cosThetaPrime = saturate(dot(lightNormal, -wi));
            return t == 0 ? 0 : cosThetaPrime / (t * t);
        }
    };

    // inverse of the thread-group swizzle: which dispatched group (SV_GroupID) renders the pixels of swizzled group (sgx, sgy)
    void UnswizzleGroup(uint32_t sgx, uint32_t sgy, uint32_t dispX, uint32_t dispY, uint32_t& Gx, uint32_t& Gy)
    {
        const uint32_t tileWidth = 16, numGroupsInTile = 16 * dispY;
        const uint32_t tileID = sgx / tileWidth, gx = sgx % tileWidth, gy = sgy;
        const uint32_t numFullTiles = dispX / tileWidth;
        const uint32_t w = tileID < numFullTiles ? tileWidth : dispX - tileWidth * numFullTiles;
        const uint32_t flat = tileID * numGroupsInTile + gy * w + gx;
        Gx = flat % dispX; Gy = flat / dispX;
    }

    Reservoir RIS_InitialCandidates(const Scene& sc, float3 pos, float3 normal, float roughness, BSDF::ShadingData surface, uint32_t sampleSetIdx,
        int numBsdfSamples, RNG& rng)
    {
        Reservoir r = Reservoir::Init();
        const bool specular = surface.GlossSpecular() && (surface.metallic || surface.specTr) && (!surface.Coated() || surface.CoatSpecular());
        const int numLightSamples = !specular ? 3 : 0;
        for (int s_b = 0; s_b < numBsdfSamples; s_b++)
        {
            BSDF::BSDFSample bsdfSample = BSDF::SampleBSDF_NoDiffuse(normal, surface, rng);
            float3 wi = bsdfSample.wi;
            float pdf_w = bsdfSample.pdf;
            BSDFHitInfo hitInfo = FindClosestHitDI(sc, pos, normal, wi, surface.Transmissive());
            float w_b = 0;
            float3 le = f3(0), lightNormal = f3(0), target = f3(0);
            uint32_t emissiveID = UINT32_MAX_;
            bool doubleSided = false;
            if (hitInfo.hit)
            {
                const zr_emissive_tri& emissive = sc.emissives[hitInfo.emissiveTriIdx];
                le = Light::Le_EmissiveTriangle(emissive);
                const float3 vtx0 = Light::Vtx0(emissive);
                const float3 vtx1 = Light::DecodeEmissiveTriV1(emissive);
                const float3 vtx2 = Light::DecodeEmissiveTriV2(emissive);
                lightNormal = cross(vtx1 - vtx0, vtx2 - vtx0);
                float twoArea = length(lightNormal);
                lightNormal = dot(lightNormal, lightNormal) == 0 ? f3(0) : lightNormal / twoArea;
                lightNormal = Light::IsDoubleSided(emissive) && dot(-wi, lightNormal) < 0 ? -lightNormal : lightNormal;
                doubleSided = Light::IsDoubleSided(emissive);
                emissiveID = emissive.ID;
                if (dot(-wi, lightNormal) > 0)
                {
                    const float lightSourcePdf = sc.aliasTable[hitInfo.emissiveTriIdx].CachedP_Orig;
                    const float pdf_light = lightSourcePdf * (1.0f / (0.5f * twoArea));
                    const float dwdA = saturate(dot(lightNormal, -wi)) / (hitInfo.t * hitInfo.t);
                    pdf_w *= dwdA;
                    const bool sampleIsSpecular = (surface.GlossSpecular() && bsdfSample.lobe == BSDF::GLOSSY_R) ||
                        (surface.CoatSpecular() && bsdfSample.lobe == BSDF::COAT);
                    float denom = (float)numBsdfSamples * pdf_w + (!sampleIsSpecular ? 1.0f : 0.0f) * (float)numLightSamples * pdf_light;
                    const float m_i = 1.0f / denom;
                    target = le * bsdfSample.f * dwdA;
                    w_b = m_i * Math::Luminance(target);
                }
            }
            if (r.Update(w_b, le, hitInfo.emissiveTriIdx, hitInfo.bary, rng))
            {
                r.target = target; r.lightID = emissiveID; r.lightPos = hitInfo.lightPos; r.lightNormal = lightNormal; r.doubleSided = doubleSided;
            }
        }
        for (int s_l = 0; s_l < numLightSamples; s_l++)
        {
            const Light::LightSample lightSample = Light::SampleLight(sc, pos, sampleSetIdx, rng, false);
            float3 le = lightSample.le;
            const float pdf_light = lightSample.pdf;
            const uint32_t emissiveIdx = lightSample.idx;
            const uint32_t lightID = lightSample.ID;
            const bool doubleSided = lightSample.twoSided;
            float3 target = f3(0);
            float3 wi = lightSample.pos - pos;
            const bool isZero = dot(wi, wi) == 0;
            const float t = isZero ? 0 : length(wi);
            wi = isZero ? wi : wi / t;
            const float dwdA = isZero ? 0 : saturate(dot(lightSample.normal, -wi)) / (t * t);
            surface.SetWi(wi, normal);
            if (dot(lightSample.normal, -wi) > 0)
            {
                target = le * BSDF::Unified(surface).f * dwdA;
                if (dot(target, target) > 0)
                    target *= Visibility_Segment(sc, pos, wi, t, normal, lightID, surface.Transmissive()) ? 1.0f : 0.0f;
            }
            const float denom = (float)numLightSamples * pdf_light + (float)numBsdfSamples * BSDF::BSDFSamplerPdf_NoDiffuse(normal, surface, wi) * dwdA;
            const float m_l = denom > 0 ? 1.0f / denom : 0;
            const float w_l = m_l * Math::Luminance(target);
            if (r.Update(w_l, le, emissiveIdx, lightSample.bary, rng))
            {
                r.target = target; r.lightID = lightID; r.lightNormal = lightSample.normal; r.lightPos = lightSample.pos; r.doubleSided = doubleSided;
            }
        }
        float targetLum = Math::Luminance(r.target);
        r.W = targetLum > 0.0f ? r.w_sum / targetLum : 0.0f;
        return r;
    }

    bool PlaneHeuristicDI(float3 samplePos, float3 currNormal, float3 currPos, float linearDepth, float tolerance = 1e-1f)
    {
        float planeDist = dot(currNormal, samplePos - currPos);
        return fabsf(planeDist) <= tolerance * linearDepth;
    }

    struct TemporalCandidate { BSDF::ShadingData surface; float3 pos, normal; int px, py; bool valid; };

    TemporalCandidate FindTemporalCandidate(const Frame& f, float3 pos, float3 normal, float roughness, const BSDF::ShadingData& surface, float2 prevUV)
    {
        TemporalCandidate c; c.valid = false; c.px = c.py = 0; c.pos = c.normal = f3(0);
        if (prevUV.x < 0.0f || prevUV.y < 0.0f || prevUV.x > 1.0f || prevUV.y > 1.0f) return c;
        const float2 renderDim = f2((float)f.W, (float)f.H);
        float2 pp = prevUV * renderDim;
        int ppx = (int)pp.x, ppy = (int)pp.y;
        float prevRoughness;
        GFlags prevFlags = FlagsAt(f.pcore, f.W, ppx, ppy, &prevRoughness);
        if (prevFlags.invalid || prevFlags.emissive || (fabsf(prevRoughness - roughness) > 0.15f) ||
            (prevFlags.metallic != surface.metallic) || (prevFlags.transmissive != surface.specTr))
            return c;
        Pixel p = LoadPixel(f, f.pcore, f.pcoat, ppx, ppy, true, ppx, ppy);
        // note: the depth passed to the plane test is the PREVIOUS pixel's (Resampling.hlsli:77)
        if (!PlaneHeuristicDI(p.pos, normal, pos, p.z))
            return c;
        c.surface = p.surface; c.px = ppx; c.py = ppy; c.pos = p.pos; c.normal = p.normal; c.valid = true;
        return c;
    }

    float OffsetPathTarget_CtT(const Scene& sc, const Reservoir& r_curr, TemporalCandidate candidate)
    {
        float3 wi_offset = r_curr.lightPos - candidate.pos;
        const bool isZero = dot(wi_offset, wi_offset) == 0;
        float t_offset = isZero ? 0 : length(wi_offset);
        wi_offset = isZero ? wi_offset : wi_offset / t_offset;
        candidate.surface.SetWi(wi_offset, candidate.normal);
        float3 lightNormal = r_curr.lightNormal;
        if (r_curr.doubleSided && dot(-wi_offset, lightNormal) < 0)
            lightNormal = -lightNormal;
        float cosThetaPrime = saturate(dot(lightNormal, -wi_offset));
        const float dwdA = isZero ? 0 : cosThetaPrime / (t_offset * t_offset);
        float3 target_offset = r_curr.le * dwdA;
        target_offset *= BSDF::Unified(candidate.surface).f;
        float targetLum_offset = Math::Luminance(target_offset);
        if (targetLum_offset > 0)
            targetLum_offset *= Visibility_Segment(sc, candidate.pos, wi_offset, t_offset, candidate.normal, r_curr.lightID,
                candidate.surface.Transmissive()) ? 1.0f : 0.0f;
        return targetLum_offset;
    }

    float3 OffsetPathTarget_TtC(const Scene& sc, const Reservoir& r_prev, float3 pos, float3 normal, BSDF::ShadingData surface)
    {
        EmissiveData prevEmissive = EmissiveData::Init(sc, r_prev.lightIdx, r_prev.bary);
        prevEmissive.SetSurfacePos(pos);
        float dwdA = prevEmissive.dWdA();
        surface.SetWi(prevEmissive.wi, normal);
        float3 target_offset = r_prev.le * dwdA;
        target_offset *= BSDF::Unified(surface).f;
        if (dot(target_offset, target_offset) > 0)
            target_offset *= Visibility_Segment(sc, pos, prevEmissive.wi, prevEmissive.t, normal, prevEmissive.ID, surface.Transmissive()) ? 1.0f : 0.0f;
        return target_offset;
    }

    void TemporalResample1(const Scene& sc, float3 pos, float3 normal, const BSDF::ShadingData& surface, const TemporalCandidate& candidate,
        const zr_rdi_reservoir* prevRes, uint32_t W, Reservoir& r_curr, RNG& rng)
    {
        Reservoir r_prev = Reservoir::Load(prevRes[(size_t)candidate.py * W + candidate.px]);
        const uint32_t newM = r_curr.M + r_prev.M;
        if (r_curr.w_sum != 0)
        {
            float targetLum_prev = OffsetPathTarget_CtT(sc, r_curr, candidate);
            const float numerator = (float)r_curr.M * Math::Luminance(r_curr.target);
            const float denom = numerator + (float)r_prev.M * targetLum_prev * 1.0f;
            const float m_curr = denom > 0 ? numerator / denom : 0;
            r_curr.w_sum *= m_curr;
        }
        if (r_prev.lightIdx != UINT32_MAX_)
        {
            const float3 target_curr = OffsetPathTarget_TtC(sc, r_prev, pos, normal, surface);
            const float targetLum_curr = Math::Luminance(target_curr);
            if (targetLum_curr > 0)
            {
                const float targetLum_prev = r_prev.W > 0 ? r_prev.w_sum / r_prev.W : 0;
                const float numerator = (float)r_prev.M * targetLum_prev;
                const float denom = numerator / 1.0f + (float)r_curr.M * targetLum_curr;
                const float m_prev = denom > 0 ? numerator / denom : 0;
                const float w_prev = m_prev * targetLum_curr * r_prev.W;
                if (r_curr.Update(w_prev, r_prev.le, r_prev.lightIdx, r_prev.bary, rng))
                    r_curr.target = target_curr;
            }
        }
        float targetLum = Math::Luminance(r_curr.target);
        r_curr.W = targetLum > 0.0f ? r_curr.w_sum / targetLum : 0.0f;
        r_curr.M = newM;
    }

    void WriteFinal(const zr_frame_constants& fc, float4* finalImg, size_t idx, float3 li)
    {
        li = isnan3(li) ? f3(0) : li;
        if (fc.Accumulate && fc.CameraStatic && fc.NumFramesCameraStatic > 1)
        {
            float4 prev = finalImg[idx];
            finalImg[idx] = f4(prev.x + li.x, prev.y + li.y, prev.z + li.z, prev.w);
        }
        else
            finalImg[idx] = f4(li.x, li.y, li.z, finalImg[idx].w);
    }

    void TemporalPass(const Frame& f, const DIParams& prm, zr_rdi_reservoir* resCurr, const zr_rdi_reservoir* resPrev, uint2* target,
        float4* finalImg, int nthreads)
    {
        const zr_frame_constants& fc = *f.fc;
        parallel_for(f.H, nthreads, [&](uint32_t y0, uint32_t y1)
        {
            for (uint32_t y = y0; y < y1; y++)
                for (uint32_t x = 0; x < f.W; x++)
                {
                    const size_t idx = (size_t)y * f.W + x;
                    GFlags flags = FlagsAt(f.core, f.W, x, y);
                    if (flags.invalid)
                    {
                        // Le_SkyWithSunDisk is part of the sun/sky path (out of scope): background stays black
                        finalImg[idx] = f4(0, 0, 0, finalImg[idx].w);
                        continue;
                    }
                    if (flags.emissive && !prm.spatial)
                    {
                        float3 le = unpack_r11g11b10(f.me[idx].y);
                        if (fc.Accumulate && fc.CameraStatic)
                        {
                            float4 prev = finalImg[idx];
                            finalImg[idx] = f4(prev.x + le.x, prev.y + le.y, prev.z + le.z, prev.w);
                        }
                        else
                            finalImg[idx] = f4(le.x, le.y, le.z, finalImg[idx].w);
                        continue;
                    }
                    Pixel p = LoadPixel(f, f.core, f.coat, x, y, false, x, y);
                    RNG rng_thread = RNG::Init(x, y, fc.FrameNum);
                    const int numBsdfSamples = (!p.surface.GlossSpecular() && p.roughness < 0.3f) ? 2 : 1;
                    // group-uniform sample set (ReSTIR_DI_Temporal.hlsl:368-370): Gid of the 8x8 group that renders this pixel
                    uint32_t Gx, Gy;
                    UnswizzleGroup(x / 8, y / 8, (f.W + 7) / 8, (f.H + 7) / 8, Gx, Gy);
                    RNG rng_group = RNG::Init(Gx, Gy, fc.FrameNum);
                    const uint32_t sampleSetIdx = rng_group.UniformUintBounded_Faster(f.sc->numSampleSets);
                    Reservoir r = RIS_InitialCandidates(*f.sc, p.pos, p.normal, p.roughness, p.surface, sampleSetIdx, numBsdfSamples, rng_thread);
                    if (prm.temporal)
                    {
                        float2 motionVec = unpack_snorm16x2(f.me[idx].x);
                        const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / f2((float)f.W, (float)f.H);
                        float2 prevUV = currUV - motionVec;
                        TemporalCandidate tc = FindTemporalCandidate(f, p.pos, p.normal, p.roughness, p.surface, prevUV);
                        if (tc.valid)
                            TemporalResample1(*f.sc, p.pos, p.normal, p.surface, tc, resPrev, f.W, r, rng_thread);
                        if (prm.spatial)
                        {
                            bool disoccluded = !tc.valid && (dot(motionVec, motionVec) > 0);
                            r.target = disoccluded ? -r.target : r.target;
                            WriteTarget(target, idx, r.target);
                            r.target = Math::Sanitize(r.target);
                        }
                    }
                    if (prm.temporal || prm.reset)
                        r.Write(resCurr[idx], prm.M_max);
                    if (!prm.spatial || !prm.temporal)
                        WriteFinal(fc, finalImg, idx, r.target * r.W);
                }
        });
    }

    // ---- PairwiseMIS.hlsli ----
    struct PairwiseMIS
    {
        Reservoir r_s; float m_c; float M_s; uint32_t k;
        static PairwiseMIS Init(uint32_t numStrategies, const Reservoir& r_c)
        {
            PairwiseMIS ret;
            ret.r_s = Reservoir::Init(); ret.m_c = 1.0f; ret.M_s = to_half((float)r_c.M); ret.k = numStrategies;
            return ret;
        }
        float Compute_m_i(const Reservoir& r_c, const Reservoir& r_i, float targetLum, float jacobian) const
        {
            const float p_i_y_i = r_i.W > 0 ? r_i.w_sum / r_i.W : 0;
            const float p_c_y_i = targetLum;
            float numerator = (float)r_i.M * p_i_y_i;
            float denom = (numerator / jacobian) + ((float)r_c.M / (float)k) * p_c_y_i;
            return denom > 0 ? numerator / denom : 0;
        }
        void Update_m_c(const Reservoir& r_c, const Reservoir& r_i, float targetLum, float jacobian)
        {
            const float p_i_y_c = targetLum;
            const float p_c_y_c = Math::Luminance(r_c.target);
            const float numerator = (float)r_i.M * p_i_y_c * jacobian;
            const float denom = numerator + ((float)r_c.M / (float)k) * p_c_y_c;
            m_c += 1 - (numerator / denom);
        }
        void Stream(const Scene& sc, const Reservoir& r_c, float3 pos_c, float3 normal_c, BSDF::ShadingData surface_c, const Reservoir& r_i,
            float3 pos_i, float3 normal_i, BSDF::ShadingData surface_i, RNG& rng)
        {
            float3 target_c_y_i = f3(0), target_i_y_c = f3(0.0f);
            float m_i = 0;
            if (r_i.lightIdx != UINT32_MAX_)
            {
                float jacobian_i_to_c = 1;      // IsShiftInvertible == true, halfVectorCopyShift == false
                EmissiveData emissive_i = EmissiveData::Init(sc, r_i.lightIdx, r_i.bary);
                emissive_i.SetSurfacePos(pos_c);
                float dwdA = emissive_i.dWdA();
                surface_c.SetWi(emissive_i.wi, normal_c);
                target_c_y_i = r_i.le * dwdA;
                if (dot(target_c_y_i, target_c_y_i) > 0)
                    target_c_y_i *= Visibility_Segment(sc, pos_c, emissive_i.wi, emissive_i.t, normal_c, emissive_i.ID, surface_c.Transmissive()) ? 1.0f : 0.0f;
                target_c_y_i *= BSDF::Unified(surface_c).f;
                const float targetLum = Math::Luminance(target_c_y_i);
                m_i = Compute_m_i(r_c, r_i, targetLum, jacobian_i_to_c);
            }
            float jacobian_c_to_i = 0;
            if (r_c.lightIdx != UINT32_MAX_)
            {
                jacobian_c_to_i = 1;
                float3 wi_i = r_c.lightPos - pos_i;
                const bool isZero = dot(wi_i, wi_i) == 0;
                float t_i = isZero ? 0 : length(wi_i);
                wi_i = isZero ? f3(0) : wi_i / t_i;
                surface_i.SetWi(wi_i, normal_i);
                const float3 lightNormal = dot(r_c.lightNormal, -wi_i) < 0 && r_c.doubleSided ? -r_c.lightNormal : r_c.lightNormal;
                const float cosThetaPrime = saturate(dot(lightNormal, -wi_i));
                const float dwdA = isZero ? 0 : cosThetaPrime / (t_i * t_i);
                target_i_y_c = r_c.le * dwdA;
                if (dot(target_i_y_c, target_i_y_c) > 0)
                    target_i_y_c *= Visibility_Segment(sc, pos_i, wi_i, t_i, normal_i, r_c.lightID, surface_i.Transmissive()) ? 1.0f : 0.0f;
                target_i_y_c *= BSDF::Unified(surface_i).f;
            }
            const float targetLum = Math::Luminance(target_i_y_c);
            Update_m_c(r_c, r_i, targetLum, jacobian_c_to_i);
            if (r_i.lightIdx != UINT32_MAX_)
            {
                const float w_i = m_i * Math::Luminance(target_c_y_i) * r_i.W;
                if (r_s.Update(w_i, r_i.le, r_i.lightIdx, r_i.bary, rng))
                    r_s.target = target_c_y_i;
            }
            M_s = to_half(M_s + (float)r_i.M);
        }
        void End(const Reservoir& r_c, RNG& rng)
        {
            const float w_c = m_c * r_c.w_sum;
            if (r_s.Update(w_c, r_c.le, r_c.lightIdx, r_c.bary, rng))
                r_s.target = r_c.target;
            r_s.M = (uint32_t)M_s;
            const float targetLum = Math::Luminance(r_s.target);
            r_s.W = targetLum > 0 ? r_s.w_sum / (targetLum * (1 + (float)k)) : 0;
        }
    };

    const float* g_disk32 = nullptr;    // 32 x (x, y)

    void SpatialPass(const Frame& f, const DIParams& prm, const zr_rdi_reservoir* resCurr, const uint2* target, float4* finalImg, int nthreads)
    {
        const zr_frame_constants& fc = *f.fc;
        const uint32_t dispX = (f.W + 7) / 8, dispY = (f.H + 7) / 8;
        parallel_for(dispX * dispY * 2, nthreads, [&](uint32_t w0, uint32_t w1)
        {
            for (uint32_t wv = w0; wv < w1; wv++)
            {
                const uint32_t g = wv / 2, wave = wv % 2;
                const uint32_t Gx = g % dispX, Gy = g / dispX;
                struct L { bool active; int x, y; size_t idx; Pixel p; Reservoir r; bool disoccluded; };
                L lanes[32];
                for (int l = 0; l < 32; l++)
                {
                    L& s = lanes[l];
                    s.active = false; s.disoccluded = false;
                    uint32_t sx, sy, sgx, sgy;
                    SwizzleThreadGroup(Gx, Gy, l % 8, wave * 4 + l / 8, 8, 8, dispX, 16, 4, 16 * dispY, sx, sy, sgx, sgy);
                    if (sx >= f.W || sy >= f.H) continue;
                    const size_t idx = (size_t)sy * f.W + sx;
                    GFlags flags = FlagsAt(f.core, f.W, sx, sy);
                    if (flags.invalid) continue;
                    if (flags.emissive)
                    {
                        float3 le = unpack_r11g11b10(f.me[idx].y);
                        if (fc.Accumulate && fc.CameraStatic)
                        {
                            float4 prev = finalImg[idx];
                            finalImg[idx] = f4(prev.x + le.x, prev.y + le.y, prev.z + le.z, prev.w);
                        }
                        else
                            finalImg[idx] = f4(le.x, le.y, le.z, finalImg[idx].w);
                        continue;
                    }
                    s.active = true; s.x = (int)sx; s.y = (int)sy; s.idx = idx;
                    s.p = LoadPixel(f, f.core, f.coat, sx, sy, false, sx, sy);
                    s.r = Reservoir::Load(resCurr[idx]);
                    if (s.r.lightIdx != UINT32_MAX_)
                    {
                        const zr_emissive_tri& tri = f.sc->emissives[s.r.lightIdx];
                        s.r.lightID = tri.ID;
                        const float3 vtx0 = Light::Vtx0(tri);
                        const float3 vtx1 = Light::DecodeEmissiveTriV1(tri);
                        const float3 vtx2 = Light::DecodeEmissiveTriV2(tri);
                        s.r.lightPos = (1.0f - s.r.bary.x - s.r.bary.y) * vtx0 + s.r.bary.x * vtx1 + s.r.bary.y * vtx2;
                        s.r.lightNormal = cross(vtx1 - vtx0, vtx2 - vtx0);
                        s.r.lightNormal = dot(s.r.lightNormal, s.r.lightNormal) == 0 ? s.r.lightNormal : normalize(s.r.lightNormal);
                        s.r.doubleSided = Light::IsDoubleSided(tri);
                        s.r.target = LoadTarget(target, idx);
                        s.disoccluded = s.r.target.x < 0 || s.r.target.y < 0 || s.r.target.z < 0;
                        s.r.target = abs3(s.r.target);
                    }
                }
                uint32_t waveDisoccluded = 0;
                for (int l = 0; l < 32; l++) if (lanes[l].active && lanes[l].disoccluded) waveDisoccluded++;
                RNG rng_group = RNG::Init(Gx, Gy, fc.FrameNum);
                rng_group.UniformUintBounded_Faster(f.sc->numSampleSets);    // sample-set index: drawn, unused here (ReSTIR_DI_Spatial.hlsl:137)
                const bool extra = !prm.stochasticSpatial || (rng_group.Uniform() < 0.6f);
                for (int l = 0; l < 32; l++)
                {
                    L& s = lanes[l];
                    if (!s.active) continue;
                    bool disoccluded = s.disoccluded;
                    if (prm.extraDisocclusion)
                        disoccluded = disoccluded && (waveDisoccluded > 3);
                    int numSamples = extra ? 2 : 1;
                    numSamples = !disoccluded ? numSamples : 4;
                    RNG rng = RNG::Init((uint32_t)s.x, (uint32_t)s.y, fc.FrameNum);
                    // SpatialResample
                    const float u0 = rng.Uniform();
                    const int offset = (int)rng.UniformUintBounded_Faster(8);
                    const float theta = u0 * TWO_PI;
                    float sinTheta, cosTheta;
                    zr_sincosf(theta, &sinTheta, &cosTheta);
                    PairwiseMIS pairwiseMIS = PairwiseMIS::Init((uint32_t)numSamples, s.r);
                    float3 samplePos[4]; int spx[4], spy[4]; uint32_t k = 0;
                    for (int i = 0; i < numSamples; i++)
                    {
                        float2 sampleUV = f2(g_disk32[((offset + i) & 31) * 2], g_disk32[((offset + i) & 31) * 2 + 1]);
                        float2 rotated;
                        rotated.x = dot(sampleUV, f2(cosTheta, -sinTheta));
                        rotated.y = dot(sampleUV, f2(sinTheta, cosTheta));
                        rotated = rotated * 16.0f;
                        // (uint2)round(...): D3D's float -> uint conversion clamps negative values to 0
                        float fx = fmaxf(rintf((float)s.x + rotated.x), 0.0f), fy = fmaxf(rintf((float)s.y + rotated.y), 0.0f);
                        if (fx >= (float)f.W || fy >= (float)f.H) continue;
                        int px = (int)fx, py = (int)fy;
                        float rough_i;
                        GFlags flags_i = FlagsAt(f.core, f.W, px, py, &rough_i);
                        if (flags_i.invalid || flags_i.emissive) continue;
                        Pixel pi = LoadPixel(f, f.core, f.coat, px, py, false, px, py);
                        bool valid = PlaneHeuristicDI(pi.pos, s.p.normal, s.p.pos, s.p.z);
                        valid = valid && (fabsf(rough_i - s.p.roughness) < 0.15f);
                        if (!valid) continue;
                        samplePos[k] = pi.pos; spx[k] = px; spy[k] = py;
                        k++;
                    }
                    pairwiseMIS.k = k;
                    for (uint32_t i = 0; i < k; i++)
                    {
                        Pixel pi = LoadPixel(f, f.core, f.coat, spx[i], spy[i], false, spx[i], spy[i]);
                        // the neighbour surface is rebuilt with transmissionDepth = false (Resampling.hlsli:507-510)
                        GCore gc = LoadCore(f.core, (size_t)spy[i] * f.W + spx[i]);
                        const float4 bc = pi.flags.subsurface ? gc.baseColor : f4(gc.baseColor.x, gc.baseColor.y, gc.baseColor.z, 0);
                        float cw = 0; float3 ccol = f3(0.0f); float cr = 0; float cior = BSDF::DEFAULT_ETA_COAT;
                        if (pi.flags.coated)
                        {
                            Coat c = UnpackCoat(LoadCoat(f.coat, (size_t)spy[i] * f.W + spx[i]));
                            cw = c.weight; ccol = c.color; cr = c.roughness; cior = c.ior;
                        }
                        const float3 wo_i = normalize(pi.origin - samplePos[i]);
                        BSDF::ShadingData surface_i = BSDF::ShadingData::Init(pi.normal, wo_i, pi.flags.metallic, pi.roughness,
                            f3(bc.x, bc.y, bc.z), BSDF::ETA_AIR, pi.eta_next, pi.flags.transmissive, 0.0f, to_half(bc.w), cw, ccol, cr, cior);
                        Reservoir r_spatial = Reservoir::Load(resCurr[(size_t)spy[i] * f.W + spx[i]]);
                        pairwiseMIS.Stream(*f.sc, s.r, s.p.pos, s.p.normal, s.p.surface, r_spatial, samplePos[i], pi.normal, surface_i, rng);
                    }
                    pairwiseMIS.End(s.r, rng);
                    Reservoir r = pairwiseMIS.r_s;
                    WriteFinal(fc, finalImg, s.idx, r.target * r.W);
                }
            }
        });
    }
}

extern "C"
{
    // Probe for the CPU-tier device-source parity test: ReSTIR DI at one pixel as the temporal kernel does it (mirrored by
    // tests/hostsim/hostsim_di.cpp). out (14 words): the 32-byte reservoir record, target (3), rng state, candidate valid, #BSDF samples
    void orc_probe_rdi_pixel(void* scene, const zr_frame_constants* fc, const uint32_t* core_, const uint32_t* me_, const uint32_t* coat_,
        const uint32_t* pcore_, const uint32_t* pcoat_, const zr_rdi_reservoir* prevRes, int x, int y, uint32_t sampleSetIdx, int temporal,
        uint32_t M_max, uint32_t* out)
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
        memset(out, 0, 14 * 4);
        const size_t idx = (size_t)y * f.W + x;
        const GFlags flags = FlagsAt(core, f.W, x, y);
        if (flags.invalid || flags.emissive) { out[13] = 0xffffffffu; return; }
        Pixel p = LoadPixel(f, core, coat, x, y, false, x, y);
        RNG rng = RNG::Init((uint32_t)x, (uint32_t)y, fc->FrameNum);
        const int numBsdfSamples = (!p.surface.GlossSpecular() && p.roughness < 0.3f) ? 2 : 1;
        Reservoir r = RIS_InitialCandidates(*f.sc, p.pos, p.normal, p.roughness, p.surface, sampleSetIdx, numBsdfSamples, rng);
        bool valid = false;
        if (temporal)
        {
            const float2 motionVec = unpack_snorm16x2(me[idx].x);
            const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / f2((float)f.W, (float)f.H);
            const float2 prevUV = currUV - motionVec;
            TemporalCandidate tc = FindTemporalCandidate(f, p.pos, p.normal, p.roughness, p.surface, prevUV);
            valid = tc.valid;
            if (tc.valid)
                TemporalResample1(*f.sc, p.pos, p.normal, p.surface, tc, prevRes, f.W, r, rng);
        }
        zr_rdi_reservoir rec;
        r.Write(rec, M_max);
        memcpy(out, &rec, 32);
        out[8] = asuint(r.target.x); out[9] = asuint(r.target.y); out[10] = asuint(r.target.z);
        out[11] = rng.State; out[12] = valid; out[13] = (uint32_t)numBsdfSamples;
    }

    void orc_rdi_set_sample_pattern(const float* p) { g_disk32 = p; }

    // state[0] = currTemporalIdx, state[1] = isTemporalReservoirValid, state[2] = reset flag
    void orc_rdi_render(void* scene_, const zr_frame_constants* fc, const uint32_t* core_, const uint32_t* me_, const uint32_t* coat_,
        const uint32_t* pcore_, const uint32_t* pcoat_, const zr_direct_params* p, zr_rdi_reservoir* res0, zr_rdi_reservoir* res1,
        uint32_t* target_, float* finalImg_, uint32_t* state, int nthreads)
    {
        const uint4* core = (const uint4*)core_;
        const uint2* me = (const uint2*)me_;
        const uint2* coat = (const uint2*)coat_;
        const uint4* pcore = (const uint4*)pcore_;
        const uint2* pcoat = (const uint2*)pcoat_;
        uint2* target = (uint2*)target_;
        float4* finalImg = (float4*)finalImg_;
        Frame f;
        f.sc = (Scene*)scene_; f.fc = fc; f.core = core; f.me = me; f.coat = coat; f.pcore = pcore; f.pcoat = pcoat;
        f.W = fc->RenderWidth; f.H = fc->RenderHeight;
        const bool doTemporal = state[1] && p->temporal_resample;
        const bool doSpatial = doTemporal && p->spatial_resample;
        DIParams prm{ doTemporal, doSpatial, p->stochastic_spatial, p->extra_disocclusion_sampling, p->M_max, p->alpha_min, state[2] };
        zr_rdi_reservoir* res[2] = { res0, res1 };
        const uint32_t cur = state[0];
        TemporalPass(f, prm, res[cur], res[1 - cur], target, finalImg, nthreads);
        if (doSpatial)
            SpatialPass(f, prm, res[cur], target, finalImg, nthreads);
        state[1] = 1;
        state[0] = 1 - cur;
        state[2] = 0;
    }
}

extern "C"
{
    // Pairwise-MIS spatial reuse (PairwiseMIS.hlsli) of the centre pixel (x, y) with neighbours (nx[i], ny[i]): the centre reservoir is
    // completed from the emissive buffer + target plane as k_di_spatial does it; neighbours enter with their own LoadPixel surface.
    // out (14 words): the resulting 32-byte record (Write with M_max 0 = no clamp), target (3), W, m_c, rng state
    void orc_probe_rdi_pairwise(void* scene, const zr_frame_constants* fc, const uint32_t* core_, const uint32_t* coat_,
        const zr_rdi_reservoir* res, const void* target, int x, int y, const int* nx, const int* ny, int numNeighbors, uint32_t seed, uint32_t* out)
    {
        using namespace orc;
        const uint4* core = (const uint4*)core_;
        const uint2* coat = (const uint2*)coat_;
        Frame f;
        f.sc = (const Scene*)scene; f.fc = fc; f.core = core; f.me = nullptr; f.coat = coat; f.pcore = core; f.pcoat = coat;
        f.W = fc->RenderWidth; f.H = fc->RenderHeight;
        const Scene& sc = *f.sc;
        memset(out, 0, 14 * 4);
        const size_t idx = (size_t)y * f.W + x;
        const GFlags flags = FlagsAt(f.core, f.W, x, y);
        if (flags.invalid || flags.emissive) { out[13] = 0xffffffffu; return; }
        Pixel p = LoadPixel(f, f.core, f.coat, x, y, false, x, y);
        Reservoir r = Reservoir::Load(res[idx]);
        if (r.lightIdx != UINT32_MAX_)
        {
            const zr_emissive_tri& tri = sc.emissives[r.lightIdx];
            r.lightID = tri.ID;
            const float3 vtx0 = Light::Vtx0(tri);
            const float3 vtx1 = Light::DecodeEmissiveTriV1(tri);
            const float3 vtx2 = Light::DecodeEmissiveTriV2(tri);
            r.lightPos = (1.0f - r.bary.x - r.bary.y) * vtx0 + r.bary.x * vtx1 + r.bary.y * vtx2;
            r.lightNormal = cross(vtx1 - vtx0, vtx2 - vtx0);
            r.lightNormal = dot(r.lightNormal, r.lightNormal) == 0 ? r.lightNormal : normalize(r.lightNormal);
            r.doubleSided = Light::IsDoubleSided(tri);
            r.target = abs3(LoadTarget((const uint2*)target, idx));
        }
        RNG rng = RNG::InitSeed(seed);
        PairwiseMIS mis = PairwiseMIS::Init((uint32_t)numNeighbors, r);
        for (int i = 0; i < numNeighbors; i++)
        {
            const GFlags fi = FlagsAt(f.core, f.W, nx[i], ny[i]);
            if (fi.invalid || fi.emissive) continue;
            Pixel pi = LoadPixel(f, f.core, f.coat, nx[i], ny[i], false, nx[i], ny[i]);
            const Reservoir r_i = Reservoir::Load(res[(size_t)ny[i] * f.W + nx[i]]);
            mis.Stream(sc, r, p.pos, p.normal, p.surface, r_i, pi.pos, pi.normal, pi.surface, rng);
        }
        mis.End(r, rng);
        zr_rdi_reservoir rec;
        mis.r_s.Write(rec, 0xffffffffu);
        memcpy(out, &rec, 32);
        out[8] = asuint(mis.r_s.target.x); out[9] = asuint(mis.r_s.target.y); out[10] = asuint(mis.r_s.target.z);
        out[11] = asuint(mis.r_s.W); out[12] = asuint(mis.m_c); out[13] = rng.State;
    }
}
