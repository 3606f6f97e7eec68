// zr_rdi.cuh -- the device functions of ReSTIR DI (reservoir record, emissive-light data, RIS over BSDF and light candidates, temporal
// candidate + resampling, pairwise MIS for the spatial pass), kept in a header so that the host build of the device source
// (tests/hostsim) can hold them to the oracle without a GPU; rdi.cu adds the two kernels and the pass object.
//   DirectLighting/Emissive/ReSTIR_DI_Temporal.hlsl  RIS_InitialCandidates :29-188, EstimateDirectLighting :190-244
//   DirectLighting/Emissive/Resampling.hlsli         FindTemporalCandidate :42-79, TemporalResample1 :276-339
//   DirectLighting/Emissive/PairwiseMIS.hlsli        :23-226
//   DirectLighting/Emissive/Reservoir.hlsli          :134-199;  Util.hlsli :9-120
#pragma once
#include "zr_pixel.cuh"

namespace zr
{
namespace
{
    struct DIParams
    {
        uint32_t temporal, spatial, stochasticSpatial, extraDisocclusion, M_max; float alpha_min; uint32_t reset;
        uint32_t rowBegin, rowEnd;              // rows this device owns (strip-sharded frames)
        unsigned long long* costMap;            // optional: SM cycles spent per 32x32-pixel tile
    };

    __constant__ float c_disk32[64];

struct Reservoir
{
    float w_sum, W; float3 le; uint32_t lightIdx; float2 bary; uint32_t M;
    float3 target; uint32_t lightID; float3 lightPos, lightNormal; bool doubleSided;

    static ZR_D Reservoir Init()
    {
        Reservoir r;
        r.le = f3(0); r.M = 0; r.w_sum = 0; r.W = 0; r.lightIdx = UINT32_MAX_; r.bary = f2(0, 0);
        r.target = f3(0); r.lightID = UINT32_MAX_; r.lightPos = f3(0); r.lightNormal = f3(0); r.doubleSided = false;
        return r;
    }
    ZR_D bool Update(float weight, float3 le_, uint32_t lightIdx_, float2 bary_, RNG& rng)
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
    static ZR_D Reservoir Load(const zr_rdi_reservoir& s)
    {
        Reservoir r = Init();
        r.le = f3(half_lo(s.le_rg), half_hi(s.le_rg), half_lo(s.le_b_meta));
        r.M = (s.le_b_meta >> 16) & 0x1f;
        r.w_sum = s.w_sum; r.W = s.W;
        r.lightIdx = s.lightIdx;
        r.bary = Math::DecodeUNorm2(s.bary);
        return r;
    }
    ZR_D void Write(zr_rdi_reservoir& s, uint32_t M_max) const
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
ZR_D void WriteTarget(uint2* target, size_t idx, float3 t)
{
    t = Math::Sanitize(t);
    target[idx] = make_uint2(pack_half2(t.x, t.y), pack_half2(t.z, 0.0f));
}
ZR_D float3 LoadTarget(const uint2* target, size_t idx)
{
    uint2 p = target[idx];
    return f3(half_lo(p.x), half_hi(p.x), half_lo(p.y));
}

struct BSDFHitInfo { uint32_t emissiveTriIdx; float2 bary; float3 lightPos; float t; bool hit; };

// Util.hlsli:68-120
ZR_D BSDFHitInfo FindClosestHitDI(const SceneDev& sc, float3 pos, float3 normal, float3 wi, bool transmissive)
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
    RayHit h = TraceClosest(sc, adjustedOrigin, wi, wiBackface ? 3e-4f : 0.0f, FLT_MAX_);
    if (h.hit)
    {
        const uint32_t meshIdx = __ldg(&sc.triMesh[h.tri]);
        const uint32_t baseEmissive = __ldg(&sc.instances[meshIdx].BaseEmissiveTriOffset);
        if (baseEmissive == UINT32_MAX_)
            return ret;
        ret.emissiveTriIdx = baseEmissive + (h.tri - __ldg(&sc.meshFirstTri[meshIdx]));
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
    static ZR_D EmissiveData Init(const SceneDev& sc, uint32_t lightIdx, float2 bary)
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
    ZR_D void SetSurfacePos(float3 pos)
    {
        wi = lightPos - pos;
        t = dot(wi, wi) == 0 ? 0 : length(wi);
        wi = t == 0 ? f3(0) : wi / t;
        lightNormal = doubleSided && dot(-wi, lightNormal) < 0 ? -lightNormal : lightNormal;
    }
    ZR_D float dWdA() const
    {
        float cosThetaPrime = saturate(dot(lightNormal, -wi));
        return t == 0 ? 0 : cosThetaPrime / (t * t);
    }
};

// RIS over BSDF and light samples (Resampling.hlsli:116-331) as block-synchronous phases (zr_rpt.cuh): every
// thread of the block walks the same 2 + 3 sample slots, `act` / the per-pixel sample counts predicate the work.
#define ZR_PHASE() __syncthreads()
// The result is built in `r`, which may live in shared memory (k_di_temporal parks it there).
template<class SD>
ZR_D void RIS_InitialCandidates_Sync(Reservoir& r, bool act, const SceneDev& sc, float3 pos, float3 normal, float roughness, SD surface,
    uint32_t sampleSetIdx, int numBsdfSamples, RNG& rng)
{
    r = Reservoir::Init();
    const bool specular = surface.GlossSpecular() && (surface.metallic || surface.specTr) && (!surface.Coated() || surface.CoatSpecular());
    const int numLightSamples = !specular ? 3 : 0;
    for (int s_b = 0; s_b < 2; s_b++)
    {
        const bool go = act && (s_b < numBsdfSamples);
        BSDF::BSDFSample bsdfSample = BSDF::BSDFSample::Init();
        ZR_PHASE();
        if (go)
            bsdfSample = BSDF::SampleBSDF_NoDiffuse(normal, surface, rng);
        ZR_PHASE();
        BSDFHitInfo hitInfo;
        hitInfo.hit = false;
        if (go)
            hitInfo = FindClosestHitDI(sc, pos, normal, bsdfSample.wi, surface.Transmissive());
        ZR_PHASE();
        if (go)
        {
            float3 wi = bsdfSample.wi;
            float pdf_w = bsdfSample.pdf;
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
    }
    for (int s_l = 0; s_l < 3; s_l++)
    {
        const bool go = act && (s_l < numLightSamples);
        Light::LightSample lightSample;
        float3 le = f3(0), target = f3(0), wi = f3(0);
        float pdf_light = 0, t = 0, dwdA = 0;
        uint32_t emissiveIdx = 0, lightID = UINT32_MAX_;
        bool doubleSided = false, facing = false;
        ZR_PHASE();
        if (go)
        {
            lightSample = Light::SampleLight(sc, pos, sampleSetIdx, rng, false);
            le = lightSample.le;
            pdf_light = lightSample.pdf;
            emissiveIdx = lightSample.idx;
            lightID = lightSample.ID;
            doubleSided = lightSample.twoSided;
            wi = lightSample.pos - pos;
            const bool isZero = dot(wi, wi) == 0;
            t = isZero ? 0 : length(wi);
            wi = isZero ? wi : wi / t;
            dwdA = isZero ? 0 : saturate(dot(lightSample.normal, -wi)) / (t * t);
            surface.SetWi(wi, normal);
            facing = dot(lightSample.normal, -wi) > 0;
            if (facing)
                target = le * BSDF::Unified(surface).f * dwdA;
        }
        ZR_PHASE();
        if (go && facing && (dot(target, target) > 0))
            target *= Visibility_Segment(sc, pos, wi, t, normal, lightID, surface.Transmissive()) ? 1.0f : 0.0f;
        ZR_PHASE();
        if (go)
        {
            const float denom = (float)numLightSamples * pdf_light + (float)numBsdfSamples * BSDF::BSDFSamplerPdf_NoDiffuse(normal, surface, wi) * dwdA;
            const float m_l = denom > 0 ? 1.0f / denom : 0;
            const float w_l = m_l * Math::Luminance(target);
            if (r.Update(w_l, le, emissiveIdx, lightSample.bary, rng))
            {
                r.target = target; r.lightID = lightID; r.lightNormal = lightSample.normal; r.lightPos = lightSample.pos; r.doubleSided = doubleSided;
            }
        }
    }
    float targetLum = Math::Luminance(r.target);
    r.W = targetLum > 0.0f ? r.w_sum / targetLum : 0.0f;
}
// The same, returning the reservoir (the host build of the device source in tests/hostsim calls this form).
template<class SD>
ZR_D Reservoir RIS_InitialCandidates_Sync(bool act, const SceneDev& sc, float3 pos, float3 normal, float roughness, SD surface,
    uint32_t sampleSetIdx, int numBsdfSamples, RNG& rng)
{
    Reservoir r;
    RIS_InitialCandidates_Sync(r, act, sc, pos, normal, roughness, surface, sampleSetIdx, numBsdfSamples, rng);
    return r;
}

ZR_D bool PlaneHeuristicDI(float3 samplePos, float3 currNormal, float3 currPos, float linearDepth, float tolerance = 1e-1f)
{
    float planeDist = dot(currNormal, samplePos - currPos);
    return fabsf(planeDist) <= tolerance * linearDepth;
}

template<class SD>
struct TemporalCandidateT { SD surface; float3 pos, normal; int px, py; bool valid; };
using TemporalCandidate = TemporalCandidateT<BSDF::ShadingData>;

template<class SD>
ZR_D TemporalCandidateT<SD> FindTemporalCandidate(const FrameView& f, const SceneDev& sc, float3 pos, float3 normal, float roughness, const SD& surface, float2 prevUV)
{
    TemporalCandidateT<SD> c; c.valid = false; c.px = c.py = 0; c.pos = c.normal = f3(0);
    if (prevUV.x < 0.0f || prevUV.y < 0.0f || prevUV.x > 1.0f || prevUV.y > 1.0f) return c;
    const float2 renderDim = f2((float)f.W, (float)f.H);
    float2 pp = prevUV * renderDim;
    int ppx = (int)pp.x, ppy = (int)pp.y;
    float prevRoughness;
    GFlags prevFlags = FlagsAt(f.pcore, f.W, ppx, ppy, &prevRoughness);
    if (prevFlags.invalid || prevFlags.emissive || (fabsf(prevRoughness - roughness) > 0.15f) ||
        (prevFlags.metallic != surface.metallic) || (prevFlags.transmissive != surface.specTr))
        return c;
    const PixelT<SD> p = LoadPixel<SD>(f, sc, f.pcore, f.pcoat, ppx, ppy, true, ppx, ppy);
    // note: the depth passed to the plane test is the PREVIOUS pixel's (Resampling.hlsli:77)
    if (!PlaneHeuristicDI(p.pos, normal, pos, p.z))
        return c;
    c.surface = p.surface; c.px = ppx; c.py = ppy; c.pos = p.pos; c.normal = p.normal; c.valid = true;
    return c;
}

// Resampling.hlsli temporal resample (OffsetPathTarget_CtT / _TtC + TemporalResample1) as phases:
// BSDF value at the temporal pixel | its shadow segment | BSDF value at the current pixel | its shadow segment
template<class SD>
ZR_D void TemporalResample1_Sync(bool act, const SceneDev& sc, float3 pos, float3 normal, const SD& surface, TemporalCandidateT<SD> candidate,
    const zr_rdi_reservoir* prevRes, uint32_t W, Reservoir& r_curr, RNG& rng)
{
    Reservoir r_prev = Reservoir::Init();
    if (act)
        r_prev = Reservoir::Load(prevRes[(size_t)candidate.py * W + candidate.px]);
    const uint32_t newM = r_curr.M + r_prev.M;
    // ---- current sample in the temporal domain ----
    const bool doCtT = act && (r_curr.w_sum != 0);
    float3 wi_offset = f3(0);
    float t_offset = 0, targetLum_offset = 0;
    float3 target_offset = f3(0);
    if (doCtT)
    {
        wi_offset = r_curr.lightPos - candidate.pos;
        const bool isZero = dot(wi_offset, wi_offset) == 0;
        t_offset = isZero ? 0 : length(wi_offset);
        wi_offset = isZero ? wi_offset : wi_offset / t_offset;
        candidate.surface.SetWi(wi_offset, candidate.normal);
        float3 lightNormal = r_curr.lightNormal;
        if (r_curr.doubleSided && dot(-wi_offset, lightNormal) < 0)
            lightNormal = -lightNormal;
        float cosThetaPrime = saturate(dot(lightNormal, -wi_offset));
        const float dwdA = isZero ? 0 : cosThetaPrime / (t_offset * t_offset);
        target_offset = r_curr.le * dwdA;
    }
    ZR_PHASE();
    if (doCtT)
    {
        target_offset *= BSDF::Unified(candidate.surface).f;
        targetLum_offset = Math::Luminance(target_offset);
    }
    ZR_PHASE();
    if (doCtT)
    {
        if (targetLum_offset > 0)
            targetLum_offset *= Visibility_Segment(sc, candidate.pos, wi_offset, t_offset, candidate.normal, r_curr.lightID,
                candidate.surface.Transmissive()) ? 1.0f : 0.0f;
        const float numerator = (float)r_curr.M * Math::Luminance(r_curr.target);
        const float denom = numerator + (float)r_prev.M * targetLum_offset * 1.0f;
        const float m_curr = denom > 0 ? numerator / denom : 0;
        r_curr.w_sum *= m_curr;
    }
    // ---- temporal sample in the current domain ----
    const bool doTtC = act && (r_prev.lightIdx != UINT32_MAX_);
    EmissiveData prevEmissive;
    SD surfaceWi = surface;
    float3 target_curr = f3(0);
    if (doTtC)
    {
        prevEmissive = EmissiveData::Init(sc, r_prev.lightIdx, r_prev.bary);
        prevEmissive.SetSurfacePos(pos);
        const float dwdA = prevEmissive.dWdA();
        surfaceWi.SetWi(prevEmissive.wi, normal);
        target_curr = r_prev.le * dwdA;
    }
    ZR_PHASE();
    if (doTtC)
        target_curr *= BSDF::Unified(surfaceWi).f;
    ZR_PHASE();
    if (doTtC)
    {
        if (dot(target_curr, target_curr) > 0)
            target_curr *= Visibility_Segment(sc, pos, prevEmissive.wi, prevEmissive.t, normal, prevEmissive.ID, surfaceWi.Transmissive()) ? 1.0f : 0.0f;
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
    if (act)
    {
        float targetLum = Math::Luminance(r_curr.target);
        r_curr.W = targetLum > 0.0f ? r_curr.w_sum / targetLum : 0.0f;
        r_curr.M = newM;
    }
}

// ---- PairwiseMIS.hlsli ----
struct PairwiseMIS
{
    Reservoir r_s; float m_c; float M_s; uint32_t k;
    static ZR_D PairwiseMIS Init(uint32_t numStrategies, const Reservoir& r_c)
    {
        PairwiseMIS ret;
        ret.r_s = Reservoir::Init(); ret.m_c = 1.0f; ret.M_s = to_half((float)r_c.M); ret.k = numStrategies;
        return ret;
    }
    ZR_D float Compute_m_i(const Reservoir& r_c, const Reservoir& r_i, float targetLum, float jacobian) const
    {
        const float p_i_y_i = r_i.W > 0 ? r_i.w_sum / r_i.W : 0;
        const float p_c_y_i = targetLum;
        float numerator = (float)r_i.M * p_i_y_i;
        float denom = (numerator / jacobian) + ((float)r_c.M / (float)k) * p_c_y_i;
        return denom > 0 ? numerator / denom : 0;
    }
    ZR_D void Update_m_c(const Reservoir& r_c, const Reservoir& r_i, float targetLum, float jacobian)
    {
        const float p_i_y_c = targetLum;
        const float p_c_y_c = Math::Luminance(r_c.target);
        const float numerator = (float)r_i.M * p_i_y_c * jacobian;
        const float denom = numerator + ((float)r_c.M / (float)k) * p_c_y_c;
        m_c += 1 - (numerator / denom);
    }
    // phases: shadow segment c<-i | BSDF value c<-i | shadow segment i<-c | BSDF value i<-c
    template<class SD>
    ZR_D void Stream_Sync(bool act, const SceneDev& sc, const Reservoir& r_c, float3 pos_c, float3 normal_c, SD surface_c, const Reservoir& r_i,
        float3 pos_i, float3 normal_i, SD surface_i, RNG& rng)
    {
        float3 target_c_y_i = f3(0), target_i_y_c = f3(0.0f);
        float m_i = 0;
        const bool has_i = act && (r_i.lightIdx != UINT32_MAX_);
        const float jacobian_i_to_c = 1;      // IsShiftInvertible == true, halfVectorCopyShift == false
        EmissiveData emissive_i;
        if (has_i)
        {
            emissive_i = EmissiveData::Init(sc, r_i.lightIdx, r_i.bary);
            emissive_i.SetSurfacePos(pos_c);
            float dwdA = emissive_i.dWdA();
            surface_c.SetWi(emissive_i.wi, normal_c);
            target_c_y_i = r_i.le * dwdA;
        }
        ZR_PHASE();
        if (has_i && (dot(target_c_y_i, target_c_y_i) > 0))
            target_c_y_i *= Visibility_Segment(sc, pos_c, emissive_i.wi, emissive_i.t, normal_c, emissive_i.ID, surface_c.Transmissive()) ? 1.0f : 0.0f;
        ZR_PHASE();
        if (has_i)
        {
            target_c_y_i *= BSDF::Unified(surface_c).f;
            const float targetLum = Math::Luminance(target_c_y_i);
            m_i = Compute_m_i(r_c, r_i, targetLum, jacobian_i_to_c);
        }
        float jacobian_c_to_i = 0;
        const bool has_c = act && (r_c.lightIdx != UINT32_MAX_);
        float3 wi_i = f3(0);
        float t_i = 0;
        if (has_c)
        {
            jacobian_c_to_i = 1;
            wi_i = r_c.lightPos - pos_i;
            const bool isZero = dot(wi_i, wi_i) == 0;
            t_i = isZero ? 0 : length(wi_i);
            wi_i = isZero ? f3(0) : wi_i / t_i;
            surface_i.SetWi(wi_i, normal_i);
            const float3 lightNormal = dot(r_c.lightNormal, -wi_i) < 0 && r_c.doubleSided ? -r_c.lightNormal : r_c.lightNormal;
            const float cosThetaPrime = saturate(dot(lightNormal, -wi_i));
            const float dwdA = isZero ? 0 : cosThetaPrime / (t_i * t_i);
            target_i_y_c = r_c.le * dwdA;
        }
        ZR_PHASE();
        if (has_c && (dot(target_i_y_c, target_i_y_c) > 0))
            target_i_y_c *= Visibility_Segment(sc, pos_i, wi_i, t_i, normal_i, r_c.lightID, surface_i.Transmissive()) ? 1.0f : 0.0f;
        ZR_PHASE();
        if (has_c)
            target_i_y_c *= BSDF::Unified(surface_i).f;
        if (act)
        {
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
    }
    ZR_D void End(const Reservoir& r_c, RNG& rng)
    {
        const float w_c = m_c * r_c.w_sum;
        if (r_s.Update(w_c, r_c.le, r_c.lightIdx, r_c.bary, rng))
            r_s.target = r_c.target;
        r_s.M = (uint32_t)M_s;
        const float targetLum = Math::Luminance(r_s.target);
        r_s.W = targetLum > 0 ? r_s.w_sum / (targetLum * (1 + (float)k)) : 0;
    }
};


    ZR_D void LoadRdi(const zr_rdi_reservoir* __restrict__ p, zr_rdi_reservoir& r)
    {
        const uint4* q = reinterpret_cast<const uint4*>(p);
        uint4 v[2] = { q[0], q[1] };
        memcpy(&r, v, 32);
    }
    ZR_D void StoreRdi(zr_rdi_reservoir* __restrict__ p, const zr_rdi_reservoir& r)
    {
        uint4 v[2];
        memcpy(v, &r, 32);
        uint4* q = reinterpret_cast<uint4*>(p);
        q[0] = v[0]; q[1] = v[1];
    }

    ZR_D void WriteFinal(const zr_frame_constants& fc, float4* __restrict__ finalImg, size_t idx, float3 li)
    {
        li = isnan3(li) ? f3(0) : li;
        if (fc.Accumulate && fc.CameraStatic && fc.NumFramesCameraStatic > 1)
        {
            const float4 prev = finalImg[idx];
            finalImg[idx] = f4(prev.x + li.x, prev.y + li.y, prev.z + li.z, prev.w);
        }
        else
            finalImg[idx] = f4(li.x, li.y, li.z, 0.0f);
    }

    ZR_D void WriteEmissive(const zr_frame_constants& fc, const FrameView& f, float4* __restrict__ finalImg, size_t idx)
    {
        const float3 le = unpack_r11g11b10(__ldg(&f.me[idx].y));
        if (fc.Accumulate && fc.CameraStatic)
        {
            const float4 prev = finalImg[idx];
            finalImg[idx] = f4(prev.x + le.x, prev.y + le.y, prev.z + le.z, prev.w);
        }
        else
            finalImg[idx] = f4(le.x, le.y, le.z, 0.0f);
    }
}
} // namespace zr
