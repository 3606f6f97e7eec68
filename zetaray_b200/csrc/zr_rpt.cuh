// zr_rpt.cuh -- ReSTIR PT state containers and the hybrid (random replay + reconnection) shift on the device.
//   IndirectLighting/ReSTIR_PT/Shift.hlsli        Reconnection :16-172, OffsetPathContext :191-358, CanReconnect :360-375,
//                                                 Replay :377-474, StepPath :476-546, Shift2 :662-816, Replay_kGt2 :818-859
//   IndirectLighting/ReSTIR_PT/Reservoir.hlsli    Reservoir :9-463 -- the 7 planes A..G live in ONE 64-byte record
//                                                 (zr_rpt_reservoir, 4 x 128-bit accesses)
//   IndirectLighting/ReSTIR_PT/ReSTIR_PT_NEE.hlsli NEE_Bsdf :145-222, NEE_Emissive :224-302, EvalDirect_Emissive_Case2/3 :306-391
// The replay context stays in registers between replay and reconnection (the reference round-trips it
// through 42 B/px r-buffers); OffsetPathContext::Quantize applies the r-buffer storage precision so the
// numbers are unchanged.
#pragma once
#include "zr_rt.cuh"

namespace zr
{
namespace RPT
{
    using BSDF::LOBE;
    using BSDF::ShadingData;
    using Light::TYPE;

    struct Reconnection
    {
        static constexpr uint32_t EMPTY = 0xf;
        float3 x_k;
        uint32_t ID;
        uint32_t meshIdx;
        float partialJacobian;
        float3 w_k_lightNormal_w_sky;
        float lightPdf;
        uint32_t seed_replay;
        uint32_t seed_nee;
        float dwdA;
        float3 L;           // half3: values are rounded to binary16 on assignment
        uint32_t k;
        LOBE lobe_k_min_1;
        LOBE lobe_k;
        TYPE lt_k;
        TYPE lt_k_plus_1;
        bool x_k_in_motion;

        static ZR_D Reconnection Init()
        {
            Reconnection ret;
            ret.k = EMPTY;
            ret.lt_k = Light::NONE;
            ret.lt_k_plus_1 = Light::NONE;
            ret.partialJacobian = 0;
            ret.x_k = f3(FLT_MAX_);
            ret.seed_replay = 0;
            ret.w_k_lightNormal_w_sky = f3(0);
            ret.L = f3(0);
            ret.lightPdf = 0;
            ret.seed_nee = 0;
            ret.dwdA = 0;
            ret.ID = 0; ret.meshIdx = 0; ret.lobe_k_min_1 = BSDF::DIFFUSE_R; ret.lobe_k = BSDF::DIFFUSE_R; ret.x_k_in_motion = false;
            return ret;
        }
        ZR_D bool Empty() const { return k == EMPTY; }
        ZR_D bool IsCase2() const { return lt_k_plus_1 != Light::NONE; }
        ZR_D bool IsCase3() const { return lt_k != Light::NONE; }
        ZR_D bool IsCase1() const { return !IsCase2() && !IsCase3(); }
        ZR_D void Clear() { k = EMPTY; lt_k = Light::NONE; lt_k_plus_1 = Light::NONE; }
        static ZR_D float3 half3(float3 v) { return f3(to_half(v.x), to_half(v.y), to_half(v.z)); }

        ZR_D void SetCase1(int k_, float3 x_k_, float t, float3 normal_k, uint32_t hitID, uint32_t meshIdx_, float3 w_k_min_1,
            LOBE l_k_min_1, float pdf_w_k_min_1, float3 w_k, LOBE l_k, float pdf_w_k)
        {
            lobe_k_min_1 = l_k_min_1;
            k = (uint32_t)k_; x_k = x_k_; ID = hitID; meshIdx = meshIdx_;
            lt_k = Light::NONE; lobe_k = l_k; w_k_lightNormal_w_sky = w_k;
            lt_k_plus_1 = Light::NONE;
            partialJacobian = pdf_w_k_min_1;
            float cos_theta_k = fabsf(dot(-w_k_min_1, normal_k));
            partialJacobian *= cos_theta_k / (t * t);
            partialJacobian *= pdf_w_k;
        }
        ZR_D void SetCase2(int k_, float3 x_k_, float t, float3 normal_k, uint32_t hitID, uint32_t meshIdx_, float3 w_k_min_1,
            LOBE l_k_min_1, float pdf_w_k_min_1, float3 w_k, LOBE l_k, float pdf_w_k, TYPE t_k_plus_1, float pdf_light,
            float3 le, uint32_t seed, float dwdA_)
        {
            lobe_k_min_1 = l_k_min_1;
            k = (uint32_t)k_; x_k = x_k_; ID = hitID; meshIdx = meshIdx_;
            lt_k = Light::NONE; lobe_k = l_k; w_k_lightNormal_w_sky = w_k;
            lt_k_plus_1 = t_k_plus_1;
            lightPdf = pdf_light; dwdA = dwdA_; seed_nee = seed; L = half3(le);
            partialJacobian = pdf_w_k_min_1;
            float cos_theta_k = fabsf(dot(-w_k_min_1, normal_k));
            partialJacobian *= cos_theta_k / (t * t);
            if (lobe_k != BSDF::ALL)
                partialJacobian *= pdf_w_k;
        }
        ZR_D void SetCase3(int k_, float3 x_k_, TYPE t, LOBE l_k_min_1, uint32_t lightID, float3 le, float3 lightNormal,
            float pdf_solidAngle, float pdf_light, float dwdA_, float3 w_sky, bool twoSided, uint32_t seed)
        {
            lobe_k_min_1 = l_k_min_1;
            k = (uint32_t)k_; x_k = x_k_; ID = lightID; lt_k = t; seed_nee = seed;
            partialJacobian = l_k_min_1 == BSDF::ALL ? 1.0f : pdf_solidAngle * dwdA_;
            lightPdf = twoSided ? pdf_light : -pdf_light;
            L = half3(le);
            lt_k_plus_1 = Light::NONE;
            if (t == Light::EMISSIVE) w_k_lightNormal_w_sky = lightNormal;
            else if (t == Light::SKY) w_k_lightNormal_w_sky = w_sky;
        }
    };

    struct Reservoir
    {
        float w_sum, W;
        float3 target;
        Reconnection rc;
        uint32_t M;

        static ZR_D Reservoir Init()
        {
            Reservoir r;
            r.rc = Reconnection::Init();
            r.w_sum = 0; r.W = 0; r.M = 0; r.target = f3(0);
            return r;
        }
        ZR_D bool Update(float weight, float3 target_, const Reconnection& rc_, RNG& rng)
        {
            if ((weight != weight) || isinf1(weight))
                return false;
            M += 1;
            if (weight == 0)
                return false;
            w_sum += weight;
            if (rng.Uniform() < (weight / w_sum))
            {
                rc = rc_;
                target = target_;
                return true;
            }
            return false;
        }

        // ---- 64-byte record <-> reservoir (Reservoir.hlsli:52-463, Emissive == true) ----
        ZR_D void UnpackMetadata(uint32_t meta)
        {
            const uint32_t x = meta & 0xff, y = (meta >> 8) & 0xff, z = (meta >> 16) & 0xff;
            uint32_t k = x & 0xf;
            rc.k = k == Reconnection::EMPTY ? k : k + 2;
            rc.lobe_k_min_1 = BSDF::LobeFromValue(y & 0x7);
            rc.lobe_k = BSDF::LobeFromValue((y >> 3) & 0x7);
            rc.lt_k = Light::TypeFromValue((y >> 6) & 0x3);
            rc.lt_k_plus_1 = Light::TypeFromValue(z & 0x3);
            rc.x_k_in_motion = (z >> 2) != 0;
            M = x >> 4;
        }
        static ZR_D Reservoir Load_NonReconnection(const zr_rpt_reservoir& s)
        {
            Reservoir r = Init();
            r.UnpackMetadata(s.meta);
            r.w_sum = s.w_sum; r.W = s.W;
            return r;
        }
        ZR_D void Load_Reconnection(const zr_rpt_reservoir& s)
        {
            const float3 L_ = f3(half_lo(s.L_rg), half_hi(s.L_rg), half_lo(s.L_b));
            if (rc.IsCase1())
            {
                rc.partialJacobian = asfloat(s.jacobian_or_seed_nee);
                rc.seed_replay = s.seed_replay; rc.ID = s.ID;
                rc.w_k_lightNormal_w_sky = Math::DecodeOct32(s.w_k);
                rc.x_k = f3(asfloat(s.x_k_x), asfloat(s.x_k_y), asfloat(s.x_k_z));
                rc.meshIdx = s.meshIdx;
                rc.L = L_;
            }
            else if (rc.IsCase2())
            {
                rc.partialJacobian = asfloat(s.jacobian_or_seed_nee);
                rc.seed_replay = s.seed_replay; rc.ID = s.ID;
                rc.x_k = f3(asfloat(s.x_k_x), asfloat(s.x_k_y), asfloat(s.x_k_z));
                rc.L = L_;
                rc.w_k_lightNormal_w_sky = Math::DecodeOct32(s.w_k);
                rc.lightPdf = s.lightPdf; rc.dwdA = s.dwdA; rc.seed_nee = s.seed_nee; rc.meshIdx = s.meshIdx;
            }
            else
            {
                rc.seed_replay = s.seed_replay; rc.ID = s.ID;
                rc.partialJacobian = rc.lobe_k_min_1 == BSDF::ALL ? 1.0f : asfloat(s.jacobian_or_seed_nee);
                rc.x_k = f3(asfloat(s.x_k_x), asfloat(s.x_k_y), asfloat(s.x_k_z));
                rc.L = L_;
                rc.lightPdf = s.lightPdf;
                rc.seed_nee = s.jacobian_or_seed_nee;
                rc.w_k_lightNormal_w_sky = Math::DecodeOct32(s.w_k);
            }
        }
        static ZR_D Reservoir Load(const zr_rpt_reservoir& s)
        {
            Reservoir r = Load_NonReconnection(s);
            if (r.rc.Empty())
                return r;
            r.Load_Reconnection(s);
            return r;
        }
        ZR_D uint32_t PackMeta(uint32_t M_max) const
        {
            uint32_t m = M_max == 0 ? M : (M < M_max ? M : M_max);
            if (m > 15) m = 15;
            uint32_t k = rc.Empty() ? rc.k : (rc.k > 2 ? rc.k : 2) - 2;
            uint32_t x = (k | (m << 4)) & 0xff;
            uint32_t y = (uint32_t)rc.lobe_k_min_1 | ((uint32_t)rc.lobe_k << 3) | ((uint32_t)rc.lt_k << 6);
            uint32_t z = (uint32_t)rc.lt_k_plus_1 | ((rc.x_k_in_motion ? 1u : 0u) << 2);
            return x | ((y & 0xff) << 8) | ((z & 0xff) << 16);
        }
        // Reservoir::Write<true>: the whole record; fields a case does not store are zero
        ZR_D void Write(zr_rpt_reservoir& s, uint32_t M_max = 0)
        {
            memset(&s, 0, sizeof(s));
            s.meta = PackMeta(M_max);
            w_sum = Math::Sanitize(w_sum);
            W = Math::Sanitize(W);
            s.w_sum = w_sum; s.W = W;
            if (rc.Empty())
                return;
            const uint32_t w_k_encoded = Math::EncodeOct32u(rc.w_k_lightNormal_w_sky);
            s.seed_replay = rc.seed_replay; s.ID = rc.ID;
            s.x_k_x = asuint(rc.x_k.x); s.x_k_y = asuint(rc.x_k.y); s.x_k_z = asuint(rc.x_k.z);
            s.w_k = w_k_encoded;
            s.L_rg = pack_half2(rc.L.x, rc.L.y);
            s.L_b = zr_f32_to_f16(rc.L.z);
            if (rc.IsCase1())
            {
                s.jacobian_or_seed_nee = asuint(rc.partialJacobian);
                s.meshIdx = rc.meshIdx;
            }
            else if (rc.IsCase2())
            {
                s.jacobian_or_seed_nee = asuint(rc.partialJacobian);
                s.lightPdf = rc.lightPdf; s.dwdA = rc.dwdA; s.seed_nee = rc.seed_nee; s.meshIdx = rc.meshIdx;
            }
            else
            {
                s.jacobian_or_seed_nee = rc.lobe_k_min_1 == BSDF::ALL ? rc.seed_nee : asuint(rc.partialJacobian);
                s.lightPdf = rc.lightPdf;
            }
        }
        // WriteReservoirData: A.x and B only
        ZR_D void WriteReservoirData(zr_rpt_reservoir& s, uint32_t M_max) const
        {
            uint32_t k = rc.Empty() ? rc.k : (rc.k > 2 ? rc.k : 2) - 2;
            uint32_t m = M < M_max ? M : M_max;
            s.meta = (s.meta & 0xffffff00u) | ((k | (m << 4)) & 0xff);
            s.w_sum = w_sum; s.W = W;
        }
    };

    // Shift.hlsli:360-375
    ZR_D bool CanReconnect(float alpha_lobe_k_min_1, float alpha_lobe_k, LOBE lobe_k_min_1, LOBE lobe_k, float alpha_min)
    {
        if ((alpha_lobe_k_min_1 < alpha_min) || (alpha_lobe_k < alpha_min)) return false;
        if ((lobe_k_min_1 == BSDF::GLOSSY_T) && (lobe_k == BSDF::GLOSSY_T)) return false;
        return true;
    }

    struct DirectLightingEstimate
    {
        float3 ld, le, wi, pos, normal;
        float pdf_solidAngle, dwdA;
        TYPE lt; LOBE lobe; uint32_t ID; float pdf_light; bool twoSided;
        static ZR_D DirectLightingEstimate Init()
        {
            DirectLightingEstimate r;
            r.ld = f3(0); r.le = f3(0); r.wi = f3(0); r.pdf_solidAngle = 0; r.dwdA = 1; r.lt = Light::NONE;
            r.ID = UINT32_MAX_; r.pos = f3(0); r.pdf_light = 0; r.twoSided = true; r.normal = f3(0); r.lobe = BSDF::DIFFUSE_R;
            return r;
        }
    };

    template<class SD>
    ZR_D bool IsSpecularSurface(const SD& surface)
    {
        return surface.GlossSpecular() && (surface.metallic || surface.specTr) && (!surface.Coated() || surface.CoatSpecular());
    }

    // -----------------------------------------------------------------------------------------------------------
    // Block-synchronous phases.
    //
    // The lighting kernels execute far more code than the 32 KB instruction cache of an SM holds, and a warp
    // walks through it almost linearly, so a free-running warp pays an L2 round trip per 128-byte instruction
    // line (ncu: ~80% of stall cycles were "no instruction"). Every function below whose name ends in _Sync is
    // therefore written as a sequence of predicated phases separated by ZR_PHASE() block barriers: all warps of a
    // block enter a phase together, so a line fetched for the first warp is a cache hit for the others.
    // Rules: a _Sync function is called from block-uniform control flow by every thread of the block, `act` says
    // whether this thread has work; what used to be an early return clears a predicate instead. Per-thread results
    // are unchanged -- the phases run the same statements in the same order for each thread.
    // -----------------------------------------------------------------------------------------------------------
#define ZR_PHASE() __syncthreads()

    // ray set-up halves of Hit_Emissive::FindClosest / Hit::FindClosest / Visibility_Segment (zr_rt.cuh)
    struct RaySetup { float3 o; float tmin, tmax; bool go; };

    ZR_D RaySetup SetupClosestEmissive(float3 pos, float3 normal, float3 wi, bool transmissive)
    {
        RaySetup rs; rs.o = f3(0); rs.tmin = 0; rs.tmax = FLT_MAX_; rs.go = true;
        const bool wiBackface = dot(normal, wi) <= 0;
        if (wiBackface)
        {
            if (transmissive) normal = -normal;
            else { rs.go = false; return rs; }
        }
        rs.o = RTU::OffsetRayRTG(pos, normal);
        rs.tmin = wiBackface ? T_MIN_TR_RAY : T_MIN_REFL_RAY;
        return rs;
    }
    ZR_D HitEmissive FinishClosestEmissive(const SceneDev& sc, const RaySetup& rs, const RayHit& h, float3 wi)
    {
        HitEmissive ret;
        ret.hit = false;
        ret.emissiveTriIdx = UINT32_MAX_;
        ret.t = 0; ret.geoIdx = 0; ret.primIdx = 0; ret.bary = f2(0, 0); ret.lightPos = f3(0);
        if (rs.go && h.hit)
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
            ret.lightPos = mad(h.t, wi, rs.o);
        }
        return ret;
    }
    ZR_D RaySetup SetupClosest(float3 pos, float3 normal, float3 wi, bool transmissive)
    {
        RaySetup rs; rs.o = f3(0); rs.tmin = 0; rs.tmax = FLT_MAX_; rs.go = true;
        const float ndotwi = dot(normal, wi);
        if (ndotwi == 0) { rs.go = false; return rs; }
        const bool wiBackface = ndotwi < 0;
        if (wiBackface)
        {
            if (!transmissive) { rs.go = false; return rs; }
            normal = -normal;
        }
        rs.o = RTU::OffsetRayRTG(pos, normal);
        rs.tmin = wiBackface ? T_MIN_TR_RAY : T_MIN_REFL_RAY;
        return rs;
    }
    ZR_D Hit MissHit()
    {
        Hit ret;
        ret.hit = false;
        ret.ID = UINT32_MAX_;
        ret.t = 0; ret.uv = f2(0, 0); ret.normal = f3(0); ret.meshIdx = 0; ret.matIdx = 0;
        return ret;
    }
    ZR_D Hit FinishClosest(const SceneDev& sc, const RaySetup& rs, const RayHit& h)
    {
        if (!(rs.go && h.hit))
            return MissHit();
        const uint32_t mesh = __ldg(&sc.triMesh[h.tri]);
        return HitAttributes(sc, mesh, h.tri - __ldg(&sc.meshFirstTri[mesh]), h.bary, h.t);
    }
    // go == false: the segment counts as occluded without tracing
    ZR_D RaySetup SetupSegment(float3 origin, float3 wi, float rayT, float3 normal, uint32_t triID, bool transmissive)
    {
        RaySetup rs; rs.o = f3(0); rs.tmin = 0; rs.tmax = 0; rs.go = false;
        if (triID == UINT32_MAX_) return rs;
        if (rayT < 1e-6f) return rs;
        const float ndotwi = dot(normal, wi);
        if (ndotwi == 0) return rs;
        const bool wiBackface = ndotwi < 0;
        if (wiBackface)
        {
            if (transmissive) normal = -normal;
            else return rs;
        }
        rs.o = RTU::OffsetRayRTG(origin, normal);
        rs.tmin = 3e-6f;
        rs.tmax = Math::PrevFloat32(rayT * 0.999f - Math::NextFloat32(rs.tmin));
        rs.go = true;
        return rs;
    }

    // ReSTIR_PT_NEE.hlsli:145-222 -- everything after the closest-hit query of the BSDF-sampled direction
    template<class SD>
    ZR_D DirectLightingEstimate NEE_Bsdf_Finish(const SceneDev& sc, float3 pos, const SD& surface, int nextBounce,
        int maxNumBounces, BSDF::BSDFSample& bsdfSample, const HitEmissive& hitInfo)
    {
        DirectLightingEstimate ret = DirectLightingEstimate::Init();
        const bool specular = IsSpecularSurface(surface);
        const int numLightSamples = specular ? 0 : 1;
        const float wiPdf = bsdfSample.pdf;
        const float3 wi = bsdfSample.wi;
        const float3 f = bsdfSample.f;
        if (hitInfo.HitWasEmissive())
        {
            const zr_emissive_tri& emissive = sc.emissives[hitInfo.emissiveTriIdx];
            const float3 le = Light::Le_EmissiveTriangle(emissive);
            const float3 vtx0 = Light::Vtx0(emissive);
            const float3 vtx1 = Light::DecodeEmissiveTriV1(emissive);
            const float3 vtx2 = Light::DecodeEmissiveTriV2(emissive);
            float3 lightNormal = cross(vtx1 - vtx0, vtx2 - vtx0);
            float twoArea = length(lightNormal);
            lightNormal = dot(lightNormal, lightNormal) == 0 ? f3(0.0f) : lightNormal / twoArea;
            lightNormal = Light::IsDoubleSided(emissive) && (dot(-wi, lightNormal) < 0) ? -lightNormal : lightNormal;
            float lightPdf = 0;
            if (!specular)
            {
                const float lightSourcePdf = numLightSamples > 0 ? sc.aliasTable[hitInfo.emissiveTriIdx].CachedP_Orig : 0;
                lightPdf = twoArea > 0 ? lightSourcePdf * (2.0f / twoArea) : 0;
            }
            float dwdA = saturate(dot(lightNormal, -wi)) / (hitInfo.t * hitInfo.t);
            float wiPdf_area = wiPdf * dwdA;
            float3 ld = le * f * dwdA;
            ret.ld = specular ? (wiPdf_area > 0 ? ld / wiPdf_area : f3(0)) : RT::PowerHeuristic(wiPdf_area, lightPdf, ld);
            ret.le = le; ret.wi = wi; ret.pdf_solidAngle = wiPdf; ret.dwdA = dwdA; ret.ID = emissive.ID;
            ret.pos = mad(hitInfo.t, wi, pos);
            ret.normal = lightNormal; ret.pdf_light = lightPdf; ret.lobe = bsdfSample.lobe; ret.lt = Light::EMISSIVE;
            ret.twoSided = Light::IsDoubleSided(emissive);
        }
        if (nextBounce >= maxNumBounces)
            bsdfSample.bsdfOverPdf = f3(0);
        return ret;
    }

    // ReSTIR_PT_NEE.hlsli:224-302 (alias-table path) in three steps: light sample + BSDF value, shadow segment,
    // sampler pdf + MIS. `surface` is the caller's copy with wi set (the reference passes it by value).
    struct NeeLightState { DirectLightingEstimate ret; float3 ld; float t, lightPdf, dwdA; bool facing; };

    template<class SD>
    ZR_D NeeLightState NEE_Emissive_Begin(const SceneDev& sc, float3 pos, float3 normal, SD& surface, uint32_t sampleSetIdx, RNG& rng)
    {
        NeeLightState st;
        st.ret = DirectLightingEstimate::Init();
        st.ret.lt = Light::EMISSIVE;
        st.ret.lobe = BSDF::ALL;
        const Light::LightSample lightSample = Light::SampleLight(sc, pos, sampleSetIdx, rng, true);
        const float3 le = lightSample.le;
        st.lightPdf = lightSample.pdf;
        st.t = length(lightSample.pos - pos);
        const float3 wi = (lightSample.pos - pos) / st.t;
        st.facing = (dot(lightSample.normal, -wi) > 0) && (st.t > 0);
        st.ld = f3(0); st.dwdA = 0;
        if (st.facing)
        {
            st.dwdA = saturate(dot(lightSample.normal, -wi)) / (st.t * st.t);
            surface.SetWi(wi, normal);
            st.ld = le * BSDF::Unified(surface).f * st.dwdA;
            st.ret.le = le; st.ret.wi = wi; st.ret.ID = lightSample.ID;
            st.ret.pos = lightSample.pos; st.ret.normal = lightSample.normal; st.ret.twoSided = lightSample.twoSided;
        }
        return st;
    }
    ZR_D DirectLightingEstimate NEE_Emissive_Finish(const NeeLightState& st, float bsdfPdf)
    {
        DirectLightingEstimate ret = st.ret;
        if (st.facing)
        {
            ret.ld = RT::PowerHeuristic(st.lightPdf, bsdfPdf, st.ld);
            ret.pdf_solidAngle = st.lightPdf / st.dwdA; ret.dwdA = st.dwdA; ret.pdf_light = st.lightPdf;
        }
        return ret;
    }

    struct OffsetPath { float3 target; float partialJacobian; bool surfKMin1Tramsmissive; };

    // Path context carried from replay to the reconnection step. The reference round-trips it
    // through the r-buffers (RGBA16F + 2 x RGBA32UI + R16UI, Shift.hlsli:191-358); Quantize() applies
    // that storage precision so keeping the context on chip gives the same numbers.
    template<class SD>
    struct OffsetPathContextT
    {
        float3 throughput, pos, normal;
        SD surface;
        float eta_curr, eta_next;
        RNG rngReplay;

        static ZR_D OffsetPathContextT Init()
        {
            OffsetPathContextT c;
            c.throughput = f3(0); c.pos = f3(0); c.normal = f3(0);
            c.surface = SD::InitEmpty();
            c.eta_curr = BSDF::ETA_AIR; c.eta_next = BSDF::DEFAULT_ETA_MAT; c.rngReplay.State = 0;
            return c;
        }
        ZR_D OffsetPathContextT Quantize() const
        {
            OffsetPathContextT ctx = Init();
            ctx.throughput = f3(to_half(throughput.x), to_half(throughput.y), to_half(throughput.z));
            if (dot(ctx.throughput, ctx.throughput) == 0)
                return ctx;
            ctx.pos = pos;
            ctx.normal = Math::DecodeOct32(Math::EncodeOct32u(normal));
            ctx.eta_curr = mad(Math::UNorm8ToFloat(Math::FloatToUNorm8((eta_curr - 1.0f) / 1.5f)), 1.5f, 1.0f);
            ctx.eta_next = mad(Math::UNorm8ToFloat(Math::FloatToUNorm8((eta_next - 1.0f) / 1.5f)), 1.5f, 1.0f);
            float3 wo = Math::DecodeOct32(Math::EncodeOct32u(surface.wo));
            float roughness = Math::UNorm8ToFloat(Math::FloatToUNorm8(!surface.GlossSpecular() ? sqrtf(surface.alpha) : 0));
            float3 baseColor = Math::UnpackRGB8(Math::Float3ToRGB8(surface.baseColor_Fr0_TrCol));
            bool metallic = surface.metallic;
            bool specTr = surface.specTr;
            float trDepth = surface.trDepth > 0 ? 1.0f : 0.0f;
            bool coated = surface.Coated();
            float subsurface = Math::UNorm8ToFloat(Math::FloatToUNorm8(surface.subsurface));
            float eta_next_ = ctx.eta_curr == BSDF::ETA_AIR ? ctx.eta_next : BSDF::ETA_AIR;
            float coat_weight = 0; float3 coat_color = f3(0.0f); float coat_roughness = 0; float coat_ior = BSDF::DEFAULT_ETA_COAT;
            if (coated)
            {
                coat_weight = Math::UNorm8ToFloat(Math::FloatToUNorm8(surface.coat_weight));
                coat_color = Math::UnpackRGB8(Math::Float3ToRGB8(surface.coat_color));
                coat_roughness = Math::UNorm8ToFloat(Math::FloatToUNorm8(!surface.CoatSpecular() ? sqrtf(surface.coat_alpha) : 0));
                float coat_eta = surface.coat_eta >= 1.0f ? surface.coat_eta : 1.0f / surface.coat_eta;
                coat_ior = mad(Math::UNorm8ToFloat(Math::FloatToUNorm8((coat_eta - 1.0f) / 1.5f)), 1.5f, 1.0f);
            }
            ctx.surface = SD::Init(ctx.normal, wo, metallic, roughness, baseColor, ctx.eta_curr, eta_next_, specTr,
                trDepth, to_half(subsurface), coat_weight, coat_color, coat_roughness, coat_ior, surface.rho);
            return ctx;
        }
    };
    using OffsetPathContext = OffsetPathContextT<ShadingData>;

    // Shift.hlsli:377-474 (Replay) + :818-859 (Replay_kGt2) as one phase loop: random replay of the first k-2
    // bounces from a new primary vertex. Returns the unquantised context; throughput == 0 means the replay failed.
    template<class SD>
    ZR_D OffsetPathContextT<SD> Replay_kGt2_Sync(bool act, const SceneDev& sc, float3 pos, float3 normal, float ior, const SD& surface,
        const Reconnection& rc, float alpha_min)
    {
        OffsetPathContextT<SD> ctx = OffsetPathContextT<SD>::Init();
        BSDF::BSDFSample bsdfSample = BSDF::BSDFSample::Init();
        const int numBounces = (int)rc.k - 2;
        int bounce = 0;
        bool go = act, inTranslucentMedium = false;
        float alpha_lobe_prev = 0;
        LOBE lobe_prev = BSDF::DIFFUSE_R;
        if (go)
        {
            ctx.pos = pos; ctx.normal = normal; ctx.surface = surface;
            ctx.rngReplay = RNG::InitSeed(rc.seed_replay);
            ctx.eta_curr = BSDF::ETA_AIR; ctx.eta_next = ior;
            ctx.throughput = f3(1);
            bsdfSample = BSDF::SampleBSDF(ctx.normal, ctx.surface, ctx.rngReplay);
            if (dot(bsdfSample.bsdfOverPdf, bsdfSample.bsdfOverPdf) == 0) { ctx.throughput = f3(0); go = false; }
            else
            {
                ctx.throughput = bsdfSample.bsdfOverPdf;
                ctx.eta_curr = dot(ctx.normal, bsdfSample.wi) < 0 ? ctx.eta_next : BSDF::ETA_AIR;
                inTranslucentMedium = ctx.eta_curr != BSDF::ETA_AIR;
                alpha_lobe_prev = BSDF::LobeAlpha(ctx.surface, bsdfSample.lobe);
                lobe_prev = bsdfSample.lobe;
            }
        }
        while (__syncthreads_or(go))
        {
            RaySetup rs; rs.go = false;
            RayHit h; h.hit = false;
            if (go)
            {
                rs = SetupClosest(ctx.pos, ctx.normal, bsdfSample.wi, ctx.surface.Transmissive());
                if (rs.go)
                    h = TraceClosest(sc, rs.o, bsdfSample.wi, rs.tmin, FLT_MAX_);
            }
            ZR_PHASE();
            if (go)
            {
                Hit hitInfo = FinishClosest(sc, rs, h);
                if (!hitInfo.hit) { ctx.throughput = f3(0); go = false; }
                else if (!GetMaterialData(sc, -bsdfSample.wi, ctx.eta_curr, hitInfo, ctx.surface, ctx.eta_next)) { ctx.throughput = f3(0); go = false; }
                else
                {
                    ctx.pos = mad(hitInfo.t, bsdfSample.wi, ctx.pos);
                    ctx.normal = hitInfo.normal;
                    bounce++;
                    if (inTranslucentMedium && ctx.surface.TrDepthGt0())
                    {
                        float3 c = ctx.surface.baseColor_Fr0_TrCol;
                        float3 extCoeff = f3(-zr_logf(c.x), -zr_logf(c.y), -zr_logf(c.z)) / ctx.surface.trDepth;
                        ctx.throughput *= f3(zr_expf(-hitInfo.t * extCoeff.x), zr_expf(-hitInfo.t * extCoeff.y), zr_expf(-hitInfo.t * extCoeff.z));
                    }
                    if (bounce >= numBounces)
                        go = false;         // replay complete
                }
            }
            ZR_PHASE();
            if (go)
            {
                bsdfSample = BSDF::SampleBSDF(ctx.normal, ctx.surface, ctx.rngReplay);
                if (dot(bsdfSample.bsdfOverPdf, bsdfSample.bsdfOverPdf) == 0) { ctx.throughput = f3(0); go = false; }
                else
                {
                    const float alpha_lobe = BSDF::LobeAlpha(ctx.surface, bsdfSample.lobe);
                    if (CanReconnect(alpha_lobe_prev, alpha_lobe, lobe_prev, bsdfSample.lobe, alpha_min)) { ctx.throughput = f3(0); go = false; }
                    else
                    {
                        const bool transmitted = dot(ctx.normal, bsdfSample.wi) < 0;
                        ctx.eta_curr = transmitted ? (ctx.eta_curr == BSDF::ETA_AIR ? ctx.eta_next : BSDF::ETA_AIR) : ctx.eta_curr;
                        ctx.throughput *= bsdfSample.bsdfOverPdf;
                        inTranslucentMedium = ctx.eta_curr != BSDF::ETA_AIR;
                        alpha_lobe_prev = alpha_lobe;
                        lobe_prev = bsdfSample.lobe;
                    }
                }
            }
        }
        return ctx;
    }

    // Shift.hlsli:662-816 (Emissive == true) with StepPath (:476-546) and EvalDirect_Emissive_Case2/3
    // (ReSTIR_PT_NEE.hlsli:306-391) unrolled into seven phases:
    //   sampler eval at x_{k-1} | closest hit towards x_k | attributes + material at y_k | BSDF value at the
    //   reconnection vertex | shadow segment (case 3) | sampler eval (case 1, or lobe-sampled NEE) | sampler pdf (light-sampled NEE)
    // `replayed` = context from Replay_kGt2_Sync (already quantised) when k > 2.
    // CASE: 0 = the reconnection case is read from `rc` (fused kernels); 1 / 2 / 3 = every thread of the block holds that case
    // (the queued kernels draw their work from per-case queues), so the phases of the other cases compile away.
    template<int CASE = 0, class SD>
    ZR_D OffsetPath Shift2_Sync(bool act, const SceneDev& sc, float3 pos, float3 normal, float ior, const SD& surface,
        const Reconnection& rc, const OffsetPathContextT<SD>* replayed, float alpha_min)
    {
        OffsetPath ret; ret.target = f3(0); ret.partialJacobian = 0; ret.surfKMin1Tramsmissive = false;
        OffsetPathContextT<SD> ctx = OffsetPathContextT<SD>::Init();
        const bool case1 = CASE == 0 ? rc.IsCase1() : CASE == 1, case2 = CASE == 0 ? rc.IsCase2() : CASE == 2,
            case3 = CASE == 0 ? rc.IsCase3() : CASE == 3;
        bool go = act;
        if (go)
        {
            ctx.pos = pos; ctx.normal = normal; ctx.surface = surface;
            ctx.rngReplay = RNG::InitSeed(rc.seed_replay);
            ctx.eta_curr = BSDF::ETA_AIR; ctx.eta_next = ior;
            ctx.throughput = f3(1);
            const int numBounces = (int)rc.k - 2;
            if (numBounces != 0)
            {
                ctx = *replayed;
                if (dot(ctx.throughput, ctx.throughput) == 0)
                    go = false;
                else
                {
                    // OffsetPathContext::Load leaves rngReplay at 0; the reference then advances it (Shift.hlsli:705-713)
                    ctx.rngReplay.State = 0;
                    for (int bounce = 0; bounce < numBounces; bounce++)
                    {
                        ctx.rngReplay.Uniform4D();
                        ctx.rngReplay.Uniform4D();
                        ctx.rngReplay.Uniform();
                    }
                }
            }
            if (go)
                ret.surfKMin1Tramsmissive = ctx.surface.specTr;
        }
        // ---- StepPath (cases 1, 2): x_{k-1} -> x_k ----
        bool step = go && !case3;
        float3 w_k_min_1 = f3(0);
        if (step)
        {
            if (!BSDF::IsLobeValid(ctx.surface, rc.lobe_k_min_1))
                step = false;
            else
            {
                const float alpha_lobe_k_min_1 = BSDF::LobeAlpha(ctx.surface, rc.lobe_k_min_1);
                if (!CanReconnect(alpha_lobe_k_min_1, 1, rc.lobe_k_min_1, rc.lobe_k, alpha_min))
                    step = false;
            }
            if (step) w_k_min_1 = normalize(rc.x_k - ctx.pos);
            else go = false;
        }
        if (go && case3)
        {
            if (!BSDF::IsLobeValid(ctx.surface, rc.lobe_k_min_1))
                go = false;
            else if (BSDF::LobeAlpha(ctx.surface, rc.lobe_k_min_1) < alpha_min)
                go = false;
        }
        ZR_PHASE();
        BSDF::BSDFSamplerEval eval; eval.pdf = 0; eval.bsdfOverPdf = f3(0); eval.f = f3(0);
        if (step)
        {
            eval = BSDF::EvalBSDFSampler(ctx.normal, ctx.surface, w_k_min_1, rc.lobe_k_min_1, ctx.rngReplay);
            if (dot(eval.bsdfOverPdf, eval.bsdfOverPdf) == 0) { step = false; go = false; }
        }
        ZR_PHASE();
        RaySetup rs; rs.go = false;
        RayHit h; h.hit = false;
        if (step)
        {
            rs = SetupClosest(ctx.pos, ctx.normal, w_k_min_1, ctx.surface.Transmissive());
            if (rs.go)
                h = TraceClosest(sc, rs.o, w_k_min_1, rs.tmin, FLT_MAX_);
        }
        ZR_PHASE();
        if (step)
        {
            Hit hitInfo = FinishClosest(sc, rs, h);
            if (!hitInfo.hit || (hitInfo.ID != rc.ID)) { step = false; go = false; }
            else
            {
                const float3 y_k = mad(hitInfo.t, w_k_min_1, ctx.pos);
                const bool transmitted = dot(ctx.normal, w_k_min_1) < 0;
                ctx.eta_curr = transmitted ? (ctx.eta_curr == BSDF::ETA_AIR ? ctx.eta_next : BSDF::ETA_AIR) : ctx.eta_curr;
                const bool inTranslucentMedium = ctx.eta_curr != BSDF::ETA_AIR;
                if (!GetMaterialData(sc, -w_k_min_1, ctx.eta_curr, hitInfo, ctx.surface, ctx.eta_next)) { step = false; go = false; }
                else
                {
                    if (inTranslucentMedium && ctx.surface.TrDepthGt0())
                    {
                        float3 c = ctx.surface.baseColor_Fr0_TrCol;
                        float3 extCoeff = f3(-zr_logf(c.x), -zr_logf(c.y), -zr_logf(c.z)) / ctx.surface.trDepth;
                        ctx.throughput *= f3(zr_expf(-hitInfo.t * extCoeff.x), zr_expf(-hitInfo.t * extCoeff.y), zr_expf(-hitInfo.t * extCoeff.z));
                    }
                    float partialJacobian = eval.pdf;
                    partialJacobian *= fabsf(dot(-w_k_min_1, hitInfo.normal));
                    partialJacobian /= (hitInfo.t * hitInfo.t);
                    ctx.pos = y_k;
                    ctx.normal = hitInfo.normal;
                    ctx.throughput *= eval.bsdfOverPdf;
                    ret.partialJacobian = partialJacobian;
                    if (partialJacobian == 0) go = false;
                }
            }
        }
        // ---- the reconnection vertex: case 1 re-evaluates the sampler towards x_{k+1}; cases 2/3 re-evaluate NEE ----
        const bool nee = go && !case1;
        SD surfWi = ctx.surface;          // EvalDirect_* take the surface by value and set wi on the copy
        float3 wiE = rc.w_k_lightNormal_w_sky;      // case 1 / 2: w_k
        float3 nrmE = ctx.normal;
        LOBE lobeE = rc.lobe_k;
        float dwdA = rc.dwdA, tE = 0, lightPdfE = rc.lightPdf;
        float3 ld = f3(0);
        RNG rngNEE = RNG::InitSeed(rc.seed_nee);
        bool needBsdf = nee;
        if (nee && case3)
        {
            wiE = rc.x_k - ctx.pos;
            tE = length(wiE);
            wiE /= tE;
            const float3 lightNormal = rc.w_k_lightNormal_w_sky;
            const bool twoSided = rc.lightPdf > 0;
            lightPdfE = fabsf(rc.lightPdf);
            // note: the reference passes ctx.pos for the normal argument (Shift.hlsli:765-767)
            nrmE = ctx.pos;
            lobeE = rc.lobe_k_min_1;
            const float wiDotLightNormal = dot(lightNormal, -wiE);
            dwdA = fabsf(wiDotLightNormal) / (tE * tE);
            needBsdf = (wiDotLightNormal > 0) || twoSided;
        }
        if (nee)
            surfWi.SetWi(wiE, nrmE);
        ZR_PHASE();
        if (nee && needBsdf)
            ld = rc.L * BSDF::Unified(surfWi).f * dwdA;
        ZR_PHASE();
        if (nee && case3 && (dot(ld, ld) > 0))
        {
            const RaySetup seg = SetupSegment(ctx.pos, wiE, tE, nrmE, rc.ID, surfWi.Transmissive());
            const bool visible = seg.go ? !TraceAnyExcept(sc, seg.o, wiE, seg.tmin, seg.tmax, rc.ID) : false;
            ld *= visible ? 1.0f : 0.0f;
        }
        ZR_PHASE();
        const bool lit = nee && !(dot(ld, ld) == 0);
        const bool lightSampled = lit && (lobeE == BSDF::ALL);
        const bool useEval = (go && case1) || (lit && !lightSampled);
        BSDF::BSDFSamplerEval ev; ev.pdf = 0; ev.bsdfOverPdf = f3(0); ev.f = f3(0);
        if (useEval)
            ev = BSDF::EvalBSDFSampler(nrmE, surfWi, wiE, lobeE, ctx.rngReplay);
        ZR_PHASE();
        float bsdfPdf = 0;
        if (lightSampled)
        {
            rngNEE.Uniform4D();
            bsdfPdf = BSDF::BSDFSamplerPdf(nrmE, surfWi, wiE, rngNEE);
        }
        if (go && case1)
        {
            ctx.throughput *= ev.bsdfOverPdf;
            ret.target = ctx.throughput * rc.L;
            ret.partialJacobian *= ev.pdf;
        }
        else if (nee)
        {
            float3 ls_ld = f3(0);
            float ls_pdf_solidAngle = 0;
            if (lightSampled)
            {
                const float bsdfPdf_area = bsdfPdf * dwdA;
                ls_ld = RT::PowerHeuristic(lightPdfE, bsdfPdf_area, ld);
                ls_pdf_solidAngle = 1.0f;
            }
            else if (lit)
            {
                const bool specular = IsSpecularSurface(surfWi);
                const float bsdfPdf_area = ev.pdf * dwdA;
                ls_ld = specular ? (bsdfPdf_area > 0 ? ld / bsdfPdf_area : f3(0)) : RT::PowerHeuristic(bsdfPdf_area, lightPdfE, ld);
                ls_pdf_solidAngle = case2 ? ev.pdf : bsdfPdf_area;
            }
            ret.target = ctx.throughput * ls_ld;
            if (case2) ret.partialJacobian *= ls_pdf_solidAngle;
            else ret.partialJacobian = ls_pdf_solidAngle;
        }
        return ret;
    }
}
} // namespace zr
