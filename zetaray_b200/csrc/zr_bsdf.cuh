// zr_bsdf.cuh -- the surface shader on the device: OpenPBR-style layered BSDF evaluation, sampling and
// pdfs (ZetaRenderPass/Common/BSDF.hlsli:106-1266, BSDFSampling.hlsli:59-765, RT.hlsli:264-288).
// Same numeric contract as the rest of the library (zr_common.cuh). Func == NoOp everywhere: the
// emissive-light variants never pass a target function.
#pragma once
#include "zr_common.cuh"

namespace zr
{
namespace RT
{
    ZR_D float BalanceHeuristic(float p_1, float p_2, float f, float n_1 = 1, float n_2 = 1)
    {
        float denom = n_1 * p_1 + n_2 * p_2;
        if (denom == 0) return 0;
        return (n_1 * f) / denom;
    }
    ZR_D float BalanceHeuristic3(float p_1, float p_2, float p_3, float f, float n_1 = 1, float n_2 = 1, float n_3 = 1)
    {
        float denom = n_1 * p_1 + n_2 * p_2 + n_3 * p_3;
        if (denom == 0) return 0;
        return (n_1 * f) / denom;
    }
    ZR_D float3 PowerHeuristic(float p_1, float p_2, float3 f, float n_1 = 1, float n_2 = 1)
    {
        float a = n_1 * p_1;
        float b = n_2 * p_2;
        float denom = a * a + b * b;
        if (denom == 0) return f3(0);
        return ((n_1 * n_1 * p_1 * f) / denom);
    }
}

// 64 x 32 x 16 R16_UNORM table, trilinear + clamp (g_samLinearClamp); manual filtering keeps the
// weights in full float precision (hardware filtering would quantise them to 8 bits)
ZR_D float RhoFetch(const uint16_t* __restrict__ data, int x, int y, int z)
{
    x = x < 0 ? 0 : (x > 63 ? 63 : x);
    y = y < 0 ? 0 : (y > 31 ? 31 : y);
    z = z < 0 ? 0 : (z > 15 ? 15 : z);
    return (float)__ldg(&data[(z * 32 + y) * 64 + x]) / 65535.0f;
}
ZR_D float RhoSample(const uint16_t* __restrict__ data, float3 uvw)
{
    float px = uvw.x * 64.0f - 0.5f, py = uvw.y * 32.0f - 0.5f, pz = uvw.z * 16.0f - 0.5f;
    float x0 = floorf(px), y0 = floorf(py), z0 = floorf(pz);
    float fx = px - x0, fy = py - y0, fz = pz - z0;
    int ix = (int)x0, iy = (int)y0, iz = (int)z0;
    float c00 = RhoFetch(data, ix, iy, iz) * (1.0f - fx) + RhoFetch(data, ix + 1, iy, iz) * fx;
    float c10 = RhoFetch(data, ix, iy + 1, iz) * (1.0f - fx) + RhoFetch(data, ix + 1, iy + 1, iz) * fx;
    float c01 = RhoFetch(data, ix, iy, iz + 1) * (1.0f - fx) + RhoFetch(data, ix + 1, iy, iz + 1) * fx;
    float c11 = RhoFetch(data, ix, iy + 1, iz + 1) * (1.0f - fx) + RhoFetch(data, ix + 1, iy + 1, iz + 1) * fx;
    float c0 = c00 * (1.0f - fy) + c10 * fy;
    float c1 = c01 * (1.0f - fy) + c11 * fy;
    return c0 * (1.0f - fz) + c1 * fz;
}

namespace BSDF
{
    constexpr float MIN_N_DOT_H_SPECULAR = 0.99998f;
    constexpr float MAX_ALPHA_SPECULAR = 0.0016f;
    constexpr float DEFAULT_ETA_MAT = 1.5f;
    constexpr float DEFAULT_ETA_COAT = 1.6f;
    constexpr float ETA_AIR = 1.0f;

    enum LOBE : uint32_t { DIFFUSE_R = 0, DIFFUSE_T = 1, GLOSSY_R = 2, GLOSSY_T = 3, COAT = 4, ALL = 5 };
    ZR_D LOBE LobeFromValue(uint32_t x) { return x <= 4 ? (LOBE)x : ALL; }

    ZR_D float DielectricF0(float eta) { float f0 = (eta - 1) / (eta + 1); return f0 * f0; }
    ZR_D float3 FresnelSchlick(float3 F0, float whdotwx)
    {
        float tmp = 1.0f - whdotwx;
        float tmpSq = tmp * tmp;
        return mad(f3(tmpSq * tmpSq * tmp), 1.0f - F0, F0);
    }
    ZR_D float FresnelSchlick_Dielectric(float F0, float whdotwx)
    {
        float tmp = 1.0f - whdotwx;
        float tmpSq = tmp * tmp;
        return mad(tmpSq * tmpSq * tmp, 1 - F0, F0);
    }
    ZR_D float Fresnel_Dielectric(float ndotwi, float eta, float cosTheta_t)
    {
        float r_parallel = mad(-eta, cosTheta_t, ndotwi) / mad(eta, cosTheta_t, ndotwi);
        float r_perp = mad(eta, ndotwi, -cosTheta_t) / mad(eta, ndotwi, cosTheta_t);
        return 0.5f * dot(f2(r_parallel, r_perp), f2(r_parallel, r_perp));
    }
    ZR_D float GGX(float ndotwh, float alphaSq)
    {
        float denom = mad(ndotwh * ndotwh, alphaSq - 1.0f, 1.0f);
        return alphaSq / (PI * denom * denom);
    }
    ZR_D float SmithG1(float alphaSq, float ndotx)
    {
        float ndotxSq = ndotx * ndotx;
        float tanThetaSq = (1.0f - ndotxSq) / ndotxSq;
        return 2.0f / (sqrtf(mad(alphaSq, tanThetaSq, 1.0f)) + 1.0f);
    }
    ZR_D float SmithHeightCorrelatedG2_Opt(int n, float alphaSq, float ndotwi, float ndotwo)
    {
        float denomWo = ndotwi * sqrtf(mad(mad(-ndotwo, alphaSq, ndotwo), ndotwo, alphaSq));
        float denomWi = ndotwo * sqrtf(mad(mad(-ndotwi, alphaSq, ndotwi), ndotwi, alphaSq));
        return (0.5f * (float)n) / (denomWo + denomWi);
    }
    ZR_D float SmithHeightCorrelatedG2OverG1(float alphaSq, float ndotwi, float ndotwo)
    {
        float G1wi = SmithG1(alphaSq, ndotwi);
        float G1wo = SmithG1(alphaSq, ndotwo);
        return G1wi / (G1wi + G1wo - G1wi * G1wo);
    }
    ZR_D float GGXReflectance_Dielectric(const uint16_t* rho, float alpha, float ndotwo, float eta)
    {
        float3 uvw;
        uvw.x = ndotwo;
        uvw.y = ((alpha - 0.002025f) / (1.0f - 0.002025f));
        uvw.z = ((eta - 0.5f) / (1.99f - 0.5f));
        return saturate(RhoSample(rho, uvw));
    }
    ZR_D float E_FON_approx(float cosTheta, float roughness)
    {
        float mucomp = 1.0f - cosTheta;
        float mucomp2 = mucomp * mucomp;
        // mul(float2x2(0.0571085289, 0.491881867, -0.332181442, 0.0714429953), float2(mucomp, mucomp2))
        float2 q = f2(dot(f2(0.0571085289f, 0.491881867f), f2(mucomp, mucomp2)),
                      dot(f2(-0.332181442f, 0.0714429953f), f2(mucomp, mucomp2)));
        float GoverPi = dot(q, f2(1.0f, mucomp2));
        return mad(roughness, GoverPi, 1.0f) / mad(0.287793398f, roughness, 1.0f);
    }
    ZR_D float3 OrenNayar(bool AccountForMultiScattering, float3 rho, float sigma, float ndotwo, float ndotwi,
        float wodotwi, float g_wo)
    {
        if (sigma == 0)
            return ONE_OVER_PI * ndotwi * rho;
        float A = 1.0f / mad(0.287793398f, sigma, 1.0f);
        float B = sigma * A;
        float s_over_t = mad(-ndotwi, ndotwo, wodotwi);
        s_over_t = s_over_t > 0 ? s_over_t / fmaxf(ndotwi, ndotwo) : s_over_t;
        float3 f = f3(ONE_OVER_PI * mad(B, s_over_t, A));
        float3 f_comp = f3(0);
        if (AccountForMultiScattering)
        {
            float avgReflectance = mad(0.0724882111f, B, A);
            float one_min_avgReflectance = 1 - avgReflectance;
            float tmp = ONE_OVER_PI * (avgReflectance / one_min_avgReflectance);
            float3 rho_ms_over_piSq = tmp / mad(-rho, one_min_avgReflectance, 1.0f);
            rho_ms_over_piSq *= rho;
            float E_wo = g_wo;
            float E_wi = E_FON_approx(ndotwi, sigma);
            f_comp = (1 - E_wo) * (1 - E_wi) * rho_ms_over_piSq;
        }
        return ndotwi * (f + f_comp) * rho;
    }
    ZR_D float3 GGXMicrofacetBRDF(float alpha, float ndotwh, float ndotwo, float ndotwi, float3 fr, bool specular)
    {
        if (specular)
            return (ndotwh >= MIN_N_DOT_H_SPECULAR ? 1.0f : 0.0f) * fr;
        float alphaSq = alpha * alpha;
        float NDF = GGX(ndotwh, alphaSq);
        float G2DivDenom = SmithHeightCorrelatedG2_Opt(1, alphaSq, ndotwi, ndotwo);
        float f = NDF * G2DivDenom * ndotwi;
        return f * fr;
    }
    ZR_D float JacobianHalfVecToIncident_Tr(float eta, float whdotwo, float whdotwi)
    {
        float denom = mad(whdotwo, 1 / eta, whdotwi);
        denom *= denom;
        return denom > 0 ? whdotwi / denom : 0;
    }
    ZR_D float GGXMicrofacetBTDF(float alpha, float ndotwh, float ndotwo, float ndotwi, float whdotwo,
        float whdotwi, float eta, float fr, bool specular)
    {
        if (specular)
        {
            float f = ndotwh >= MIN_N_DOT_H_SPECULAR ? 1.0f : 0.0f;
            return f * (1 - fr);
        }
        float alphaSq = alpha * alpha;
        float NDF = GGX(ndotwh, alphaSq);
        float G2opt = SmithHeightCorrelatedG2_Opt(4, alphaSq, ndotwi, ndotwo);
        float f = NDF * G2opt * whdotwo;
        float dwh_dwi = JacobianHalfVecToIncident_Tr(eta, whdotwo, whdotwi);
        f *= dwh_dwi;
        f *= ndotwi;
        return f * (1 - fr);
    }
    ZR_D float3 SampleGGXVNDF(float3 wo, float alpha_x, float alpha_y, float2 u)
    {
        float3 Vh = normalize(f3(alpha_x * wo.x, alpha_y * wo.y, wo.z));
        float phi = TWO_PI * u.x;
        float z = mad((1.0f - u.y), (1.0f + Vh.z), -Vh.z);
        float sinTheta = sqrtf(saturate(1.0f - z * z));
        float s, c;
        zr_sincosf(phi, &s, &c);
        float x = sinTheta * c;
        float y = sinTheta * s;
        float3 cc = f3(x, y, z);
        float3 Nh = cc + Vh;
        return normalize(f3(alpha_x * Nh.x, alpha_y * Nh.y, fmaxf(0.0f, Nh.z)));
    }
    ZR_D float3 SampleGGXMicrofacet(float3 wo, float alpha, float3 shadingNormal, float2 u)
    {
        Math::CoordinateSystem onb = Math::CoordinateSystem::Build(shadingNormal);
        float3 woLocal = f3(dot(onb.b1, wo), dot(onb.b2, wo), dot(shadingNormal, wo));
        float3 whLocal = SampleGGXVNDF(woLocal, alpha, alpha, u);
        return mad(whLocal.x, onb.b1, mad(whLocal.y, onb.b2, whLocal.z * shadingNormal));
    }
    ZR_D float GGXMicrofacetPdf(float alpha, float ndotwh, float ndotwo)
    {
        float alphaSq = alpha * alpha;
        float NDF = GGX(ndotwh, alphaSq);
        float G1 = SmithG1(alphaSq, ndotwo);
        return (NDF * G1) / ndotwo;
    }

    // Material features (ZR_MATERIAL_* bits): the optional lobes a ShadingDataT<MF> compiles in. For a feature outside MF the
    // predicates that guard its code -- Coated(), ThinWalled(), Transmissive(), specTr -- are compile-time false, so a kernel
    // instantiated for MF_NONE carries no clear-coat, specular-transmission, thin-walled or medium code. Such a surface type may
    // only shade materials without those features (zr_scene::materialFeatures); for them every value it computes is the one
    // MF_ALL computes, because the predicates it drops are false at run time too.
    constexpr uint32_t MF_NONE = 0;
    constexpr uint32_t MF_ALL = ZR_MATERIAL_COAT | ZR_MATERIAL_TRANSMISSION | ZR_MATERIAL_THIN_WALLED;

    template<bool Stored> struct SpecTrField { bool specTr; };
    template<> struct SpecTrField<false> { static constexpr bool specTr = false; };

    template<uint32_t MF>
    struct ShadingDataT : SpecTrField<(MF & ZR_MATERIAL_TRANSMISSION) != 0>
    {
        static constexpr bool HasCoat = (MF & ZR_MATERIAL_COAT) != 0;
        static constexpr bool HasTransmission = (MF & ZR_MATERIAL_TRANSMISSION) != 0;
        static constexpr bool HasThinWalled = (MF & ZR_MATERIAL_THIN_WALLED) != 0;
        using ShadingData = ShadingDataT;
        using SpecTrField<HasTransmission>::specTr;

        float alpha;
        float3 wo;
        float ndotwi, ndotwo, ndotwh, whdotwi, whdotwo, wodotwi, g_wo;
        float3 baseColor_Fr0_TrCol;
        float eta;
        bool metallic, backfacing_wo, invalid, reflection;
        float trDepth;      // half
        float subsurface;   // half
        float coat_weight;
        float3 coat_color;
        float coat_alpha;
        float coat_eta;
        const uint16_t* rho;   // directional-albedo table (scene-owned)

        static ZR_D ShadingData InitEmpty()
        {
            ShadingData ret;
            memset(&ret, 0, sizeof(ret));
            ret.eta = DEFAULT_ETA_MAT / ETA_AIR;
            ret.coat_eta = DEFAULT_ETA_COAT;
            return ret;
        }
        static ZR_D ShadingData Init(float3 shadingNormal, float3 wo, bool metallic, float roughness, float3 baseColor,
            float eta_curr = ETA_AIR, float eta_next = DEFAULT_ETA_MAT, bool specTr = false,
            float transmissionDepth = 0, float subsurface = 0, float coat_weight = 0, float3 coat_color = f3(0.0f),
            float coat_roughness = 0, float eta_coat = DEFAULT_ETA_COAT, const uint16_t* rhoTable = nullptr)
        {
            float2 roughness4 = f2(roughness, coat_roughness);
            if (HasCoat && coat_weight > 0 && coat_roughness > 0)
            {
                roughness4 = roughness4 * roughness4;
                roughness4 = roughness4 * roughness4;
                float roughness_coated = fminf(roughness4.x + 2 * roughness4.y, 1);
                roughness_coated = rsqrt_(rsqrt_(roughness_coated));
                roughness = Math::Lerp(roughness, roughness_coated, coat_weight);
            }
            ShadingData si;
            memset(&si, 0, sizeof(si));
            si.wo = wo;
            float ndotwo = dot(shadingNormal, wo);
            si.backfacing_wo = ndotwo <= 0;
            si.ndotwo = fmaxf(ndotwo, 1e-5f);
            si.metallic = metallic;
            si.alpha = roughness * roughness;
            si.baseColor_Fr0_TrCol = baseColor;
            if constexpr (HasTransmission)
                si.specTr = specTr;
            si.trDepth = to_half(transmissionDepth);
            si.subsurface = to_half(subsurface);
            float eta_base = eta_curr == ETA_AIR ? eta_next : eta_curr;
            float eta_no_coat = eta_next / eta_curr;
            float eta_coated = eta_base >= eta_coat ? eta_base / eta_coat : eta_coat / eta_base;
            si.eta = Math::Lerp(eta_no_coat, eta_coated, coat_weight);
            si.g_wo = !metallic && !specTr ? E_FON_approx(fmaxf(ndotwo, 1e-4f), roughness) : 0;
            si.coat_weight = coat_weight;
            si.coat_color = coat_color;
            si.coat_alpha = coat_roughness * coat_roughness;
            si.coat_eta = eta_curr == ETA_AIR ? eta_coat / ETA_AIR : ETA_AIR / eta_coat;
            si.rho = rhoTable;
            return si;
        }

        ZR_D bool ThinWalled() const { return HasThinWalled && subsurface > 0; }
        ZR_D bool Transmissive() const { return specTr || ThinWalled(); }
        ZR_D bool Coated() const { return HasCoat && coat_weight != 0; }
        // the transmission depth of a medium the path travels through (only transmissive materials have one)
        ZR_D bool TrDepthGt0() const { return HasTransmission && trDepth > 0; }
        ZR_D bool GlossSpecular() const { return alpha <= MAX_ALPHA_SPECULAR; }
        ZR_D bool CoatSpecular() const { return coat_alpha <= MAX_ALPHA_SPECULAR; }
        ZR_D float3 TransmissionTint() const { return trDepth > 0 ? f3(1) : baseColor_Fr0_TrCol; }

        ZR_D void SetWi_Refl(float3 wi, float3 shadingNormal, float3 wh)
        {
            reflection = true;
            float ndotwi_n = dot(shadingNormal, wi);
            ndotwh = saturate(dot(shadingNormal, wh));
            whdotwo = saturate(dot(wh, wo));
            whdotwi = whdotwo;
            bool isInvalid = backfacing_wo || ndotwh == 0 || whdotwo == 0;
            invalid = isInvalid || ndotwi_n <= 0;
            ndotwi = fmaxf(ndotwi_n, 1e-5f);
            wodotwi = dot(wo, wi);
        }
        ZR_D void SetWi_Refl(float3 wi, float3 shadingNormal)
        {
            float3 wh = normalize(wi + wo);
            SetWi_Refl(wi, shadingNormal, wh);
        }
        ZR_D void SetWi_Tr(float3 wi, float3 shadingNormal, float3 wh)
        {
            reflection = false;
            float ndotwi_n = dot(shadingNormal, wi);
            ndotwh = saturate(dot(shadingNormal, wh));
            whdotwo = saturate(dot(wh, wo));
            whdotwi = fabsf(dot(wh, wi));
            bool isInvalid = backfacing_wo || (specTr && (ndotwh == 0 || whdotwo == 0));
            invalid = isInvalid || ndotwi_n >= 0 || !Transmissive() || metallic;
            ndotwi = fmaxf(fabsf(ndotwi_n), 1e-5f);
            wodotwi = dot(wo, wi);
        }
        ZR_D void SetWi(float3 wi, float3 shadingNormal, float3 wh)
        {
            float ndotwi_n = dot(shadingNormal, wi);
            reflection = ndotwi_n >= 0;
            ndotwh = saturate(dot(shadingNormal, wh));
            whdotwo = saturate(dot(wh, wo));
            bool backfacing_r = ndotwi_n <= 0;
            bool backfacing_t = ndotwi_n >= 0 || !Transmissive() || metallic;
            bool isInvalid = backfacing_wo || (specTr && (ndotwh == 0 || whdotwo == 0));
            invalid = isInvalid || (reflection && backfacing_r) || (!reflection && backfacing_t);
            ndotwi = fmaxf(fabsf(ndotwi_n), 1e-5f);
            whdotwi = fabsf(dot(wh, wi));
            wodotwi = dot(wo, wi);
        }
        ZR_D float3 SetWi(float3 wi, float3 shadingNormal)
        {
            float ndotwi_n = dot(shadingNormal, wi);
            reflection = ndotwi_n >= 0;
            float s = reflection ? 1 : eta;
            float3 wh = normalize(mad(wi, s, wo));
            wh = !reflection && eta > 1 ? -wh : wh;
            SetWi(wi, shadingNormal, wh);
            return wh;
        }
        ZR_D float3 Fresnel(float3 fr0, bool& tir) const
        {
            float cosTheta_i = whdotwo;
            tir = false;
            if (metallic)
                return FresnelSchlick(fr0, cosTheta_i);
            float eta_relative = 1.0f / eta;
            float sinTheta_iSq = saturate(mad(-cosTheta_i, cosTheta_i, 1.0f));
            float cosTheta_tSq = mad(-eta_relative * eta_relative, sinTheta_iSq, 1.0f);
            tir = cosTheta_tSq <= 0;
            if (tir)
                return f3(1);
            float cosTheta_t = sqrtf(cosTheta_tSq);
            return f3(Fresnel_Dielectric(cosTheta_i, eta_relative, cosTheta_t));
        }
        ZR_D float3 Fresnel() const
        {
            float3 fr0 = metallic ? baseColor_Fr0_TrCol : f3(DielectricF0(eta));
            bool unused;
            return Fresnel(fr0, unused);
        }
        ZR_D float Fresnel_Coat(float& cosTheta_t) const
        {
            cosTheta_t = 0;
            float cosTheta_i = whdotwo;
            float eta_relative = 1.0f / coat_eta;
            float sinTheta_iSq = saturate(mad(-cosTheta_i, cosTheta_i, 1.0f));
            float cosTheta_tSq = mad(-eta_relative * eta_relative, sinTheta_iSq, 1.0f);
            if (cosTheta_tSq <= 0)
                return 1;
            cosTheta_t = sqrtf(cosTheta_tSq);
            float Fr0 = DielectricF0(coat_eta);
            float cosTheta = coat_eta > 1 ? cosTheta_i : cosTheta_t;
            return FresnelSchlick_Dielectric(Fr0, cosTheta);
        }
    };
    using ShadingData = ShadingDataT<MF_ALL>;

    template<class SD>
    ZR_D bool IsLobeValid(const SD& surface, LOBE lt)
    {
        if (lt == ALL) return true;
        if (surface.metallic && (lt != GLOSSY_R) && (lt != COAT)) return false;
        if (!surface.specTr && (lt == GLOSSY_T)) return false;
        if (surface.specTr && (lt == DIFFUSE_R)) return false;
        if (!surface.ThinWalled() && (lt == DIFFUSE_T)) return false;
        if (!surface.Coated() && (lt == COAT)) return false;
        return true;
    }
    template<class SD>
    ZR_D float LobeAlpha(const SD& surface, LOBE lt)
    {
        if (lt == GLOSSY_R || lt == GLOSSY_T) return surface.alpha;
        if (lt == COAT) return surface.coat_alpha;
        return 1.0f;
    }

    template<class SD>
    ZR_D float3 EvalDiffuse(bool EON, const SD& surface)
    {
        float s = surface.subsurface == 0 ? 1 : surface.subsurface * 0.5f;
        float diffuseRoughness = sqrtf(surface.alpha);
        float3 diffuse = OrenNayar(EON, surface.baseColor_Fr0_TrCol, diffuseRoughness, surface.ndotwo, surface.ndotwi,
            surface.wodotwi, surface.g_wo);
        return s * diffuse;
    }
    ZR_D float3 SampleDiffuse(float3 normal, float2 u, float& pdf)
    {
        float3 wiLocal = Sampling::SampleCosineWeightedHemisphere(u, pdf);
        Math::CoordinateSystem onb = Math::CoordinateSystem::Build(normal);
        return mad(wiLocal.x, onb.b1, mad(wiLocal.y, onb.b2, wiLocal.z * normal));
    }
    template<class SD>
    ZR_D float DiffusePdf(const SD& surface) { return surface.ndotwi * ONE_OVER_PI; }
    template<class SD>
    ZR_D float3 EvalGloss(const SD& surface, float3 fr)
    {
        return GGXMicrofacetBRDF(surface.alpha, surface.ndotwh, surface.ndotwo, surface.ndotwi, fr, surface.GlossSpecular());
    }
    template<class SD>
    ZR_D float3 SampleGloss(const SD& surface, float3 shadingNormal, float2 u)
    {
        if (surface.GlossSpecular())
            return reflect(-surface.wo, shadingNormal);
        float3 wh = SampleGGXMicrofacet(surface.wo, surface.alpha, shadingNormal, u);
        return reflect(-surface.wo, wh);
    }
    template<class SD>
    ZR_D float GlossPdf(const SD& surface)
    {
        if (surface.GlossSpecular())
            return surface.ndotwh >= MIN_N_DOT_H_SPECULAR ? 1.0f : 0.0f;
        float pdf = GGXMicrofacetPdf(surface.alpha, surface.ndotwh, surface.ndotwo);
        return pdf / 4.0f;
    }
    template<class SD>
    ZR_D float EvalTranslucentTr(const SD& surface, float fr)
    {
        return GGXMicrofacetBTDF(surface.alpha, surface.ndotwh, surface.ndotwo, surface.ndotwi, surface.whdotwo,
            surface.whdotwi, surface.eta, fr, surface.GlossSpecular());
    }
    template<class SD>
    ZR_D float EvalCoat(const SD& surface, float Fr)
    {
        return surface.coat_weight * GGXMicrofacetBRDF(surface.coat_alpha, surface.ndotwh, surface.ndotwo, surface.ndotwi,
            f3(Fr), surface.CoatSpecular()).x;
    }
    template<class SD>
    ZR_D float3 SampleCoat(const SD& surface, float3 shadingNormal, float2 u)
    {
        float3 wh = surface.CoatSpecular() ? shadingNormal :
            SampleGGXMicrofacet(surface.wo, surface.coat_alpha, shadingNormal, u);
        return reflect(-surface.wo, wh);
    }
    template<class SD>
    ZR_D float CoatPdf(const SD& surface)
    {
        if (surface.CoatSpecular())
            return surface.ndotwh >= MIN_N_DOT_H_SPECULAR ? 1.0f : 0.0f;
        float pdf = GGXMicrofacetPdf(surface.coat_alpha, surface.ndotwh, surface.ndotwo);
        return pdf / 4.0f;
    }
    template<class SD>
    ZR_D float3 TranslucentTrOverPdf(const SD& surface, float fr)
    {
        if (surface.GlossSpecular())
            return (1 - fr) * surface.TransmissionTint();
        float alphaSq = surface.alpha * surface.alpha;
        return SmithHeightCorrelatedG2OverG1(alphaSq, surface.ndotwi, surface.ndotwo) * (1 - fr) * surface.TransmissionTint();
    }
    ZR_D float3 coat_tr_pow(float3 coat_color, float c)
    {
        // exp(c * log(coat_color))
        return f3(zr_expf(c * zr_logf(coat_color.x)), zr_expf(c * zr_logf(coat_color.y)), zr_expf(c * zr_logf(coat_color.z)));
    }
    template<class SD>
    ZR_D float3 BaseWeight(const SD& surface)
    {
        float3 base_weight = f3(1);
        if (surface.Coated())
        {
            float cosTheta_t;
            float Fr_coat = surface.Fresnel_Coat(cosTheta_t);
            bool tir_c = cosTheta_t <= 0;
            if (tir_c)
                return f3(0);
            float reflectance_c = surface.CoatSpecular() ? Fr_coat :
                GGXReflectance_Dielectric(surface.rho, surface.coat_alpha, surface.ndotwo, surface.coat_eta);
            float c = 0.5f / cosTheta_t + 0.5f / surface.whdotwo;
            float3 coat_tr = coat_tr_pow(surface.coat_color, c);
            base_weight = Math::Lerp(f3(1.0f), (1 - reflectance_c) * coat_tr, surface.coat_weight);
        }
        return base_weight;
    }
    template<class SD>
    ZR_D float3 TransmittanceToDielectricBaseTr(const SD& surface)
    {
        float3 base_weight = BaseWeight(surface);
        float reflectance_g = surface.GlossSpecular() ? 0 :
            GGXReflectance_Dielectric(surface.rho, surface.alpha, surface.ndotwo, surface.eta);
        return (1 - reflectance_g) * base_weight;
    }
    template<class SD>
    ZR_D float3 DielectricBaseSpecularTr(const SD& surface, float Fr_g)
    {
        if (surface.invalid || !surface.specTr)
            return f3(0);
        float3 transmittance = TransmittanceToDielectricBaseTr(surface);
        float glossyTr = EvalTranslucentTr(surface, Fr_g);
        return glossyTr * surface.TransmissionTint() * transmittance;
    }
    template<class SD>
    ZR_D float3 DielectricBaseDiffuseTr(const SD& surface, float Fr_g)
    {
        if (surface.invalid)
            return f3(0);
        float3 base_weight = BaseWeight(surface);
        float reflectance_g = surface.GlossSpecular() ? Fr_g :
            GGXReflectance_Dielectric(surface.rho, surface.alpha, surface.ndotwo, surface.eta);
        return (1 - reflectance_g) * EvalDiffuse(false, surface) * base_weight;
    }

    struct BSDFEval { float3 f; float3 Fr_g; bool tir; };

    template<class SD>
    ZR_D BSDFEval Unified(const SD& surface)
    {
        BSDFEval ret;
        ret.f = f3(0); ret.Fr_g = f3(0); ret.tir = false;
        if (surface.invalid)
            return ret;
        float3 base_weight = f3(1);
        if (surface.Coated())
        {
            float cosThetaT_o;
            float Fr_coat = surface.Fresnel_Coat(cosThetaT_o);
            bool tir_c = cosThetaT_o <= 0;
            if (!surface.reflection && tir_c)
                return ret;
            if (surface.reflection)
            {
                ret.f = f3(EvalCoat(surface, Fr_coat));
                if (tir_c)
                    return ret;
            }
            float reflectance_c = surface.CoatSpecular() ? Fr_coat :
                GGXReflectance_Dielectric(surface.rho, surface.coat_alpha, surface.ndotwo, surface.coat_eta);
            float c = 1.0f / cosThetaT_o;
            float3 coat_tr = coat_tr_pow(surface.coat_color, c);
            base_weight = Math::Lerp(f3(1.0f), (1 - reflectance_c) * coat_tr, surface.coat_weight);
        }
        float3 fr0 = surface.metallic ? surface.baseColor_Fr0_TrCol : f3(DielectricF0(surface.eta));
        ret.Fr_g = surface.Fresnel(fr0, ret.tir);
        float3 glossyRefl = EvalGloss(surface, ret.Fr_g);
        if (surface.metallic || ret.tir)
        {
            ret.f += base_weight * glossyRefl;
            return ret;
        }
        float reflectance_g = surface.GlossSpecular() ? ret.Fr_g.x :
            GGXReflectance_Dielectric(surface.rho, surface.alpha, surface.ndotwo, surface.eta);
        if (!surface.specTr)
        {
            float3 diffuse = EvalDiffuse(true, surface);
            ret.f += base_weight * ((1 - reflectance_g) * diffuse + glossyRefl * (surface.reflection ? 1.0f : 0.0f));
            return ret;
        }
        if (surface.reflection)
        {
            ret.f += glossyRefl * base_weight;
            return ret;
        }
        reflectance_g = surface.GlossSpecular() ? 0 : reflectance_g;
        float glossyTr = EvalTranslucentTr(surface, ret.Fr_g.x);
        ret.f = ((1 - reflectance_g) * glossyTr * surface.TransmissionTint()) * base_weight;
        return ret;
    }

    // ---------------------------------------------------------------------------------------
    // BSDFSampling.hlsli (Func == NoOp: the emissive variants never pass a target function)
    // ---------------------------------------------------------------------------------------
    struct BSDFSample
    {
        float3 wi; LOBE lobe; float pdf; float3 bsdfOverPdf; float3 f;
        static ZR_D BSDFSample Init() { BSDFSample r; r.wi = f3(0); r.lobe = DIFFUSE_R; r.pdf = 0; r.bsdfOverPdf = f3(0); r.f = f3(0); return r; }
    };
    struct BSDFSamplerEval { float pdf; float3 bsdfOverPdf; float3 f; };

    template<class SD>
    ZR_D BSDFSample SampleBSDF_NoDiffuse(float3 normal, SD surface, float2 u_c, float2 u_g,
        float u_wrs_0, float u_wrs_1)
    {
        BSDFSample ret = BSDFSample::Init();
        float pdf_base = 1;
        if (surface.Coated())
        {
            float reflectance_c = GGXReflectance_Dielectric(surface.rho, surface.coat_alpha, surface.ndotwo, surface.coat_eta);
            float pdf_coat = reflectance_c * surface.coat_weight;
            pdf_base = 1 - pdf_coat;
            if (u_wrs_0 < pdf_coat)
            {
                float3 wi_c = SampleCoat(surface, normal, u_c);
                surface.SetWi_Refl(wi_c, normal);
                BSDFEval eval = Unified(surface);
                ret.wi = wi_c;
                ret.lobe = COAT;
                ret.f = eval.f;
                ret.pdf = CoatPdf(surface) * pdf_coat;
                ret.bsdfOverPdf = ret.f / ret.pdf;
                return ret;
            }
        }
        float3 wh = surface.GlossSpecular() ? normal : SampleGGXMicrofacet(surface.wo, surface.alpha, normal, u_g);
        float3 wi_r = reflect(-surface.wo, wh);
        surface.SetWi_Refl(wi_r, normal, wh);
        float wh_pdf = GGXMicrofacetPdf(surface.alpha, surface.ndotwh, surface.ndotwo);
        ret.wi = wi_r;
        ret.lobe = GLOSSY_R;
        ret.pdf = surface.GlossSpecular() ? 1 : wh_pdf / 4.0f;
        ret.pdf *= pdf_base;
        BSDFEval eval = Unified(surface);
        ret.f = eval.f;
        ret.bsdfOverPdf = ret.f / ret.pdf;
        if (surface.metallic || !surface.specTr || eval.tir)
            return ret;
        float3 wi_t = refract(-surface.wo, wh, 1 / surface.eta);
        float p_r = eval.Fr_g.x * Math::Luminance(f3(1.0f));
        p_r = p_r / (p_r + (1 - eval.Fr_g.x) * Math::Luminance(f3(1.0f)));
        if (u_wrs_1 < p_r)
        {
            ret.bsdfOverPdf /= p_r;
            ret.pdf *= p_r;
        }
        else
        {
            surface.SetWi_Tr(wi_t, normal, wh);
            ret.pdf = (1 - p_r) * pdf_base;
            if (!surface.GlossSpecular())
            {
                ret.pdf *= wh_pdf * surface.whdotwo;
                float dwh_dwi = JacobianHalfVecToIncident_Tr(surface.eta, surface.whdotwo, surface.whdotwi);
                ret.pdf *= dwh_dwi;
            }
            ret.f = DielectricBaseSpecularTr(surface, eval.Fr_g.x);
            ret.bsdfOverPdf = ret.pdf > 0 ? ret.f / ret.pdf : f3(0);
            ret.wi = wi_t;
            ret.lobe = GLOSSY_T;
        }
        return ret;
    }

    template<class SD>
    ZR_D BSDFSample SampleBSDF_NoDiffuse(float3 normal, const SD& surface, RNG& rng)
    {
        float2 u_c = rng.Uniform2D();
        float2 u_g = rng.Uniform2D();
        float u_wrs_0 = rng.Uniform();
        float u_wrs_1 = rng.Uniform();
        return SampleBSDF_NoDiffuse(normal, surface, u_c, u_g, u_wrs_0, u_wrs_1);
    }

    template<class SD>
    ZR_D BSDFSample SampleBSDF_NoSpecTr(float3 normal, SD surface, float2 u_coat, float2 u_g, float2 u_d,
        float u_wrs_g, float u_wrs_dr, float u_wrs_dt)
    {
        BSDFSample ret = BSDFSample::Init();
        float w_sum = 0;
        float3 target = f3(0);
        if (surface.Coated())
        {
            float3 wi_c = SampleCoat(surface, normal, u_coat);
            surface.SetWi_Refl(wi_c, normal);
            BSDFEval eval = Unified(surface);
            target = eval.f;
            ret.wi = wi_c;
            ret.lobe = COAT;
            ret.f = target;
            float pdf_c = CoatPdf(surface);
            float pdf_g = GlossPdf(surface);
            float pdf_d = !surface.metallic ? DiffusePdf(surface) : 0;
            float targetLum_c = Math::Luminance(target);
            w_sum = RT::BalanceHeuristic3(pdf_c, pdf_g, pdf_d, targetLum_c);
        }
        {
            float3 wi_g = SampleGloss(surface, normal, u_g);
            surface.SetWi_Refl(wi_g, normal);
            BSDFEval eval = Unified(surface);
            float3 target_g = eval.f;
            float pdf_g = GlossPdf(surface);
            float pdf_d = !surface.metallic && !eval.tir ? DiffusePdf(surface) : 0;
            float pdf_c = surface.Coated() ? CoatPdf(surface) : 0;
            float w_g = RT::BalanceHeuristic3(pdf_g, pdf_d, pdf_c, Math::Luminance(target_g));
            w_sum += w_g;
            if ((w_sum > 0) && (u_wrs_g < (w_g / w_sum)))
            {
                target = target_g;
                ret.wi = wi_g;
                ret.lobe = GLOSSY_R;
                ret.f = target_g;
            }
        }
        if (!surface.metallic)
        {
            float pdf_d;
            float3 wi_d = SampleDiffuse(normal, u_d, pdf_d);
            float Fr_g;
            {
                surface.SetWi_Refl(wi_d, normal);
                BSDFEval eval = Unified(surface);
                float3 target_dr = eval.f;
                Fr_g = eval.Fr_g.x;
                float pdf_g = GlossPdf(surface);
                float pdf_c = surface.Coated() ? CoatPdf(surface) : 0;
                float w_dr = RT::BalanceHeuristic3(pdf_d, pdf_g, pdf_c, Math::Luminance(target_dr));
                w_sum += w_dr;
                if ((w_sum > 0) && (u_wrs_dr < (w_dr / w_sum)))
                {
                    target = target_dr;
                    ret.wi = wi_d;
                    ret.lobe = DIFFUSE_R;
                    ret.f = target_dr;
                }
            }
            if (surface.ThinWalled())
            {
                float3 wi_dt = -wi_d;
                float3 target_dt = DielectricBaseDiffuseTr(surface, Fr_g);
                float w_dt = Math::Luminance(target_dt) / pdf_d;
                w_sum += w_dt;
                if ((w_sum > 0) && (u_wrs_dt < (w_dt / w_sum)))
                {
                    target = target_dt;
                    ret.wi = wi_dt;
                    ret.lobe = DIFFUSE_T;
                    ret.f = target_dt;
                }
            }
        }
        float targetLum = Math::Luminance(target);
        ret.bsdfOverPdf = targetLum > 0 ? target * w_sum / targetLum : f3(0);
        ret.pdf = w_sum > 0 ? targetLum / w_sum : 0;
        return ret;
    }

    // Always consumes exactly 9 uniforms (BSDFSampling.hlsli:318-327)
    template<class SD>
    ZR_D BSDFSample SampleBSDF(float3 normal, const SD& surface, RNG& rng)
    {
        float2 u_c = rng.Uniform2D();
        float2 u_g = rng.Uniform2D();
        float2 u_d = rng.Uniform2D();
        float u_wrs_0 = rng.Uniform();
        float u_wrs_1 = rng.Uniform();
        float u_wrs_2 = rng.Uniform();
        if (!surface.specTr)
            return SampleBSDF_NoSpecTr(normal, surface, u_c, u_g, u_d, u_wrs_0, u_wrs_1, u_wrs_2);
        return SampleBSDF_NoDiffuse(normal, surface, u_c, u_g, u_wrs_0, u_wrs_1);
    }

    template<class SD>
    ZR_D BSDFSamplerEval EvalBSDFSampler_NoSpecTr(float3 normal, SD surface, float3 wi, LOBE lobe,
        float2 u_c, float2 u_g, float2 u_d)
    {
        BSDFSamplerEval ret;
        float w_sum = 0;
        float3 target = f3(0);
        if (surface.Coated())
        {
            const bool isZ_c = lobe == COAT;
            const float3 wi_c = isZ_c ? wi : SampleCoat(surface, normal, u_c);
            surface.SetWi_Refl(wi_c, normal);
            target = Unified(surface).f;
            const float targetLum_c = Math::Luminance(target);
            const float pdf_c = CoatPdf(surface);
            const float pdf_g = GlossPdf(surface);
            const float pdf_d = !surface.metallic ? DiffusePdf(surface) : 0;
            w_sum = RT::BalanceHeuristic3(pdf_c, pdf_g, pdf_d, targetLum_c);
        }
        {
            const bool isZ_g = lobe == GLOSSY_R;
            const float3 wi_g = isZ_g ? wi : SampleGloss(surface, normal, u_g);
            surface.SetWi_Refl(wi_g, normal);
            const float3 target_g = Unified(surface).f;
            const float targetLum_g = Math::Luminance(target_g);
            const float pdf_g = GlossPdf(surface);
            const float pdf_d = !surface.metallic ? DiffusePdf(surface) : 0;
            const float pdf_c = surface.Coated() ? CoatPdf(surface) : 0;
            w_sum += RT::BalanceHeuristic3(pdf_g, pdf_d, pdf_c, targetLum_g);
            target = isZ_g ? target_g : target;
        }
        if (!surface.metallic)
        {
            float pdfUnused;
            float3 w_d = SampleDiffuse(normal, u_d, pdfUnused);
            float Fr_g;
            {
                const bool isZ_dr = lobe == DIFFUSE_R;
                const float3 wi_d = isZ_dr ? wi : w_d;
                surface.SetWi_Refl(wi_d, normal);
                BSDFEval eval = Unified(surface);
                const float3 target_dr = eval.f;
                Fr_g = eval.Fr_g.x;
                const float targetLum_dr = Math::Luminance(target_dr);
                const float pdf_d = DiffusePdf(surface);
                const float pdf_g = GlossPdf(surface);
                const float pdf_c = surface.Coated() ? CoatPdf(surface) : 0;
                w_sum += RT::BalanceHeuristic3(pdf_d, pdf_g, pdf_c, targetLum_dr);
                target = isZ_dr ? target_dr : target;
            }
            if (surface.ThinWalled())
            {
                const bool isZ_dt = lobe == DIFFUSE_T;
                const float3 target_dt = DielectricBaseDiffuseTr(surface, Fr_g);
                const float targetLum_dt = Math::Luminance(target_dt);
                const float pdf_d = DiffusePdf(surface);
                w_sum += targetLum_dt / pdf_d;
                target = isZ_dt ? target_dt : target;
            }
        }
        float targetLum = Math::Luminance(target);
        ret.bsdfOverPdf = targetLum > 0 ? target * w_sum / targetLum : f3(0);
        ret.pdf = w_sum > 0 ? targetLum / w_sum : 0;
        ret.f = target;
        return ret;
    }

    template<class SD>
    ZR_D BSDFSamplerEval EvalBSDFSampler_NoDiffuse(float3 normal, SD surface, float3 wi, LOBE lobe)
    {
        float3 wh = surface.SetWi(wi, normal);
        BSDFEval eval = Unified(surface);
        float pdf_base = 1;
        BSDFSamplerEval ret;
        ret.f = eval.f;
        if (surface.Coated())
        {
            float reflectance_c = GGXReflectance_Dielectric(surface.rho, surface.coat_alpha, surface.ndotwo, surface.coat_eta);
            float pdf_coat = reflectance_c * surface.coat_weight;
            pdf_base = 1 - pdf_coat;
            if (lobe == COAT)
            {
                ret.pdf = CoatPdf(surface) * pdf_coat;
                ret.bsdfOverPdf = ret.f / ret.pdf;
                return ret;
            }
        }
        const float wh_pdf = GGXMicrofacetPdf(surface.alpha, surface.ndotwh, surface.ndotwo);
        ret.pdf = !surface.GlossSpecular() ? wh_pdf / 4.0f : (surface.ndotwh >= MIN_N_DOT_H_SPECULAR ? 1.0f : 0.0f);
        ret.pdf *= pdf_base;
        ret.bsdfOverPdf = ret.f / ret.pdf;
        if (surface.metallic || !surface.specTr || eval.tir)
            return ret;
        float targetScaleLum = Math::Luminance(f3(1.0f));
        float targetScaleOtherLum = Math::Luminance(f3(1.0f));
        float p_r = eval.Fr_g.x * (lobe == GLOSSY_R ? targetScaleLum : targetScaleOtherLum);
        p_r = p_r / (p_r + (1 - eval.Fr_g.x) * (lobe == GLOSSY_R ? targetScaleOtherLum : targetScaleLum));
        if (lobe == GLOSSY_R)
        {
            ret.bsdfOverPdf /= p_r;
            ret.pdf *= p_r;
            return ret;
        }
        ret.bsdfOverPdf = ((!surface.invalid ? 1.0f : 0.0f) * (!surface.reflection ? 1.0f : 0.0f)) *
            TranslucentTrOverPdf(surface, eval.Fr_g.x);
        ret.bsdfOverPdf *= TransmittanceToDielectricBaseTr(surface);
        ret.bsdfOverPdf *= f3(1.0f);
        ret.bsdfOverPdf /= pdf_base;
        ret.bsdfOverPdf /= (1 - p_r);
        ret.pdf = 1 - p_r;
        ret.pdf *= surface.GlossSpecular() ? (surface.ndotwh >= MIN_N_DOT_H_SPECULAR ? 1.0f : 0.0f) : wh_pdf * surface.whdotwo;
        ret.pdf *= pdf_base;
        if (!surface.GlossSpecular())
        {
            float dwh_dwi = JacobianHalfVecToIncident_Tr(surface.eta, surface.whdotwo, surface.whdotwi);
            ret.pdf *= dwh_dwi;
        }
        return ret;
    }

    template<class SD>
    ZR_D BSDFSamplerEval EvalBSDFSampler(float3 normal, const SD& surface, float3 wi, LOBE lobe, RNG& rng)
    {
        float2 u_c = rng.Uniform2D();
        float2 u_g = rng.Uniform2D();
        float2 u_d = rng.Uniform2D();
        rng.Uniform(); rng.Uniform(); rng.Uniform();
        if (!surface.specTr)
            return EvalBSDFSampler_NoSpecTr(normal, surface, wi, lobe, u_c, u_g, u_d);
        return EvalBSDFSampler_NoDiffuse(normal, surface, wi, lobe);
    }

    template<class SD>
    ZR_D float BSDFSamplerPdf_NoDiffuse(float3 normal, SD surface, float3 wi)
    {
        float3 wh = surface.SetWi(wi, normal);
        float pdf_base = 1;
        float pdf_c = 0;
        if (surface.Coated())
        {
            float reflectance_c = GGXReflectance_Dielectric(surface.rho, surface.coat_alpha, surface.ndotwo, surface.coat_eta);
            float pdf_coat = reflectance_c * surface.coat_weight;
            pdf_base = 1 - pdf_coat;
            if (surface.reflection)
                pdf_c = CoatPdf(surface) * pdf_coat;
        }
        const float wh_pdf = GGXMicrofacetPdf(surface.alpha, surface.ndotwh, surface.ndotwo);
        if (surface.metallic || !surface.specTr)
        {
            float pdf_gr = surface.GlossSpecular() ? (surface.ndotwh >= MIN_N_DOT_H_SPECULAR ? 1.0f : 0.0f) : wh_pdf / 4.0f;
            pdf_gr *= pdf_base;
            return surface.reflection ? pdf_c + pdf_gr : 0;
        }
        float pdf_g = surface.GlossSpecular() ? (surface.ndotwh >= MIN_N_DOT_H_SPECULAR ? 1.0f : 0.0f) : 1;
        pdf_g *= pdf_base;
        float targetScaleLum = Math::Luminance(f3(1.0f));
        float targetScaleOtherLum = Math::Luminance(f3(1.0f));
        float Fr_g = surface.Fresnel().x;
        float pdf_r = Fr_g * (surface.reflection ? targetScaleLum : targetScaleOtherLum);
        pdf_r = pdf_r / (pdf_r + (1 - Fr_g) * (surface.reflection ? targetScaleOtherLum : targetScaleLum));
        if (surface.reflection)
        {
            pdf_g *= surface.GlossSpecular() ? 1 : (wh_pdf / 4.0f);
            pdf_g *= pdf_r;
            return pdf_g + pdf_c;
        }
        pdf_g *= 1 - pdf_r;
        if (!surface.GlossSpecular())
        {
            pdf_g *= wh_pdf * surface.whdotwo;
            float dwh_dwi = JacobianHalfVecToIncident_Tr(surface.eta, surface.whdotwo, surface.whdotwi);
            pdf_g *= dwh_dwi;
        }
        return pdf_g;
    }

    template<class SD>
    ZR_D float BSDFSamplerPdf(float3 normal, SD surface, float3 wi_z, RNG& rng)
    {
        if (surface.specTr)
            return BSDFSamplerPdf_NoDiffuse(normal, surface, wi_z);
        surface.SetWi(wi_z, normal);
        if (!surface.reflection && !surface.ThinWalled())
            return 0;
        BSDFEval eval_z = Unified(surface);
        float targetLum = Math::Luminance(eval_z.f);
        if (targetLum == 0)
            return 0;
        float w_sum_c, w_sum_g, w_sum_dr, w_sum_dt;
        {
            float pdf_g = GlossPdf(surface);
            float pdf_d = !surface.metallic ? DiffusePdf(surface) : 0;
            float pdf_c = surface.Coated() ? CoatPdf(surface) : 0;
            float w = surface.reflection ? RT::BalanceHeuristic3(pdf_g, pdf_d, pdf_c, targetLum) :
                (targetLum / pdf_d) * (!surface.metallic ? 1.0f : 0.0f);
            w_sum_g = w; w_sum_dr = w; w_sum_dt = w; w_sum_c = w;
        }
        if (w_sum_g == 0)
            return 0;
        float pdf_d;
        float3 wi_d = SampleDiffuse(normal, rng.Uniform2D(), pdf_d);
        float Fr_g = 0;
        if (!surface.metallic)
        {
            surface.SetWi_Refl(wi_d, normal);
            BSDFEval eval = Unified(surface);
            Fr_g = eval.Fr_g.x;
            float targetLum_dr = Math::Luminance(eval.f);
            float pdf_g = GlossPdf(surface);
            float pdf_c = surface.Coated() ? CoatPdf(surface) : 0;
            float w = RT::BalanceHeuristic3(pdf_d, pdf_g, pdf_c, targetLum_dr);
            w_sum_g += w; w_sum_dt += w; w_sum_c += w;
        }
        if (!surface.metallic && surface.ThinWalled())
        {
            float3 target_dt = DielectricBaseDiffuseTr(surface, Fr_g);
            float targetLum_dt = Math::Luminance(target_dt);
            float w = targetLum_dt / pdf_d;
            w_sum_g += w; w_sum_dr += w; w_sum_c += w;
        }
        {
            float3 wi_g = SampleGloss(surface, normal, rng.Uniform2D());
            surface.SetWi_Refl(wi_g, normal);
            float targetLum_g = Math::Luminance(Unified(surface).f);
            float pdf_g = GlossPdf(surface);
            float pdf_dd = !surface.metallic ? DiffusePdf(surface) : 0;
            float pdf_c = surface.Coated() ? CoatPdf(surface) : 0;
            float w = RT::BalanceHeuristic3(pdf_g, pdf_dd, pdf_c, targetLum_g);
            w_sum_dr += w; w_sum_dt += w; w_sum_c += w;
        }
        if (surface.Coated())
        {
            float3 wi_c = SampleCoat(surface, normal, rng.Uniform2D());
            surface.SetWi_Refl(wi_c, normal);
            float targetLum_c = Math::Luminance(Unified(surface).f);
            float pdf_g = GlossPdf(surface);
            float pdf_dd = !surface.metallic ? DiffusePdf(surface) : 0;
            float pdf_c = CoatPdf(surface);
            float w = RT::BalanceHeuristic3(pdf_g, pdf_dd, pdf_c, targetLum_c);
            w_sum_g += w; w_sum_dr += w; w_sum_dt += w;
        }
        float pdf = w_sum_g > 0 ? targetLum / w_sum_g : 0;
        pdf += w_sum_dr > 0 ? targetLum / w_sum_dr : 0;
        pdf += w_sum_c > 0 ? targetLum / w_sum_c : 0;
        pdf += surface.ThinWalled() && (w_sum_dt > 0) ? targetLum / w_sum_dt : 0;
        return pdf;
    }
}
} // namespace zr
