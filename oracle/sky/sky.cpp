// ORACLE -- test infrastructure, not product code (see orc_math.h header).
//
// The sky-view LUT and the sky behind geometry (sky_api.h), restated from the reference shaders:
//   Common/Volumetric.hlsli      densities, Altitude, IntersectRayAtmosphere / IntersectRayPlanet, EstimateTransmittance,
//                                EstimateLs, RayleighPhaseFunction, SchlickPhaseFunction
//   Common/Math.hlsli:104-134    ArcCos, SphericalToCartesian, SphericalFromCartesian
//   Sky/SkyViewLUT.hlsl:19-54    one texel per thread, NON_LINEAR_LATITUDE 1, max(0, Ls) into R11G11B10F
//   Common/LightSource.hlsli     Le_Sky (:158-175), Le_SkyWithSunDisk (:177-199)
//   Compositing.hlsl:43-47, ReSTIR_DI_Temporal.hlsl:274-281   the two write points
// Numerics as orc_math.h: mad / dot are fmaf chains, other products and sums are rounded one at a time in HLSL text order.
// SampleLevel(g_samLinearWrap) is bilinear at texel-centre mapping with wrap on both axes and float weights (DESIGN §6 item 13).
#include "sky_api.h"
#include "../orc_gbuffer.h"

using namespace orc;

namespace
{
    constexpr float ONE_OVER_4_PI = 0.079577472f;

    float3 V3(const float v[3]) { return f3(v[0], v[1], v[2]); }
    float3 Exp3(float3 v) { return f3(zr_expf(v.x), zr_expf(v.y), zr_expf(v.z)); }

    // ---- Volumetric.hlsli ----
    float RayleighPhase(float cosTheta) { return 0.0596831f * (1.0f + cosTheta * cosTheta); }
    float SchlickPhase(float cosTheta, float g)
    {
        const float k = 1.55f * g - 0.55f * g * g * g;
        const float denom = 1.0f - k * cosTheta;
        return ONE_OVER_4_PI * (1.0f - k * k) / (denom * denom);
    }
    float3 Density(float altitude)
    {
        return f3(zr_expf(-fmaxf(0.0f, altitude / 8.0f)), zr_expf(-fmaxf(0.0f, altitude / 1.2f)),
            fmaxf(0.0f, 1.0f - fabsf(altitude - 25.0f) / 15.0f));
    }
    float Altitude(float3 pos, float planetRadius) { return length(pos) - planetRadius; }
    float IntersectAtmosphere(float radius, float3 o, float3 d)
    {
        const float m = dot(d, o);
        const float delta = sqrtf(m * m - dot(o, o) + radius * radius);
        return -m + delta;
    }
    bool IntersectPlanet(float radius, float3 o, float3 d, float& t)
    {
        const float m = dot(d, o);
        float delta = m * m - dot(o, o) + radius * radius;
        if (delta < 0.0f) { t = 0.0f; return false; }
        delta = sqrtf(delta);
        t = fminf(-m - delta, -m + delta);
        return t >= 0.0f;
    }
    float3 Transmittance(float R, float3 o, float3 d, float t, float3 sr, float sm, float3 so, int n)
    {
        if (t <= 1e-5f) return f3(1.0f);
        const float step = t / (float)n;
        float3 pos = o + 0.5f * step * d;
        float3 tau = f3(0.0f);
        for (int s = 0; s < n; s++)
        {
            tau += Density(Altitude(pos, R));
            pos += step * d;
        }
        tau = sr * tau.x + sm * tau.y + so * tau.z;
        tau *= step;
        return Exp3(-tau);
    }
    float3 Ls(float R, float3 o, float3 d, float3 l, float Hatm, float g, float3 sr, float ssm, float stm, float3 so, int n)
    {
        float t = IntersectAtmosphere(R + Hatm, o, d);
        float tp;
        if (IntersectPlanet(R, o, d, tp)) t = tp;
        const float step = t / (float)n;
        float3 pos = o + 0.5f * step * d;
        float3 tau = f3(0.0f), lr = f3(0.0f), lm = f3(0.0f);
        for (int s = 0; s < n; s++)
        {
            const float3 dens = Density(Altitude(pos, R));
            tau += dens * step;
            const float3 tr = Exp3(-(sr * tau.x + stm * tau.y + so * tau.z));
            const float tl = IntersectAtmosphere(R + Hatm, pos, -l);
            const float3 trl = Transmittance(R, pos, -l, tl, sr, stm, so, 8);
            lr += tr * dens.x * trl;
            lm += tr * dens.y * trl;
            pos += step * d;
        }
        const float c = dot(l, -d);
        float3 L = lr * sr * RayleighPhase(c);
        L += lm * ssm * SchlickPhase(c, g);
        L *= step;
        return L;
    }

    // ---- SkyViewLUT.hlsl ----
    uint32_t LutTexel(const zr_frame_constants& fc, uint32_t x, uint32_t y, uint32_t lw, uint32_t lh)
    {
        float phi = (float)x / (float)lw;
        phi *= TWO_PI;
        const float v = (float)y / (float)lh;
        const float s = v >= 0.5f ? 1.0f : -1.0f;
        const float a = v - 0.5f;
        const float theta = a * a * TWO_PI * s + PI_OVER_2;
        const float sinTheta = zr_sinf(theta);
        const float3 w = f3(1.0f * sinTheta * zr_cosf(phi), 1.0f * zr_cosf(theta), -1.0f * sinTheta * zr_sinf(phi));
        const float3 sr = V3(fc.RayleighSigmaSColor) * fc.RayleighSigmaSScale;
        const float stm = fc.MieSigmaA + fc.MieSigmaS;
        const float3 so = V3(fc.OzoneSigmaAColor) * fc.OzoneSigmaAScale;
        const float3 o = f3(0.0f, fc.PlanetRadius + 0.2f, 0.0f);
        float3 L = Ls(fc.PlanetRadius, o, w, V3(fc.SunDir), fc.AtmosphereAltitude, fc.g, sr, fc.MieSigmaS, stm, so, 32);
        L *= fc.SunIlluminance;
        return pack_r11g11b10(max3(L, 0.0f));
    }

    // ---- LightSource.hlsli ----
    struct Lut { const uint32_t* t; uint32_t w, h; };
    float3 Sample(const Lut& lut, float2 uv)
    {
        const float tx = uv.x * (float)lut.w - 0.5f, ty = uv.y * (float)lut.h - 0.5f;
        const float fx0 = floorf(tx), fy0 = floorf(ty);
        const float fx = tx - fx0, fy = ty - fy0;
        const int W = (int)lut.w, H = (int)lut.h;
        const int x0 = (((int)fx0 % W) + W) % W, y0 = (((int)fy0 % H) + H) % H;
        const int x1 = (x0 + 1) % W, y1 = (y0 + 1) % H;
        const float3 c00 = unpack_r11g11b10(lut.t[(size_t)y0 * W + x0]), c10 = unpack_r11g11b10(lut.t[(size_t)y0 * W + x1]);
        const float3 c01 = unpack_r11g11b10(lut.t[(size_t)y1 * W + x0]), c11 = unpack_r11g11b10(lut.t[(size_t)y1 * W + x1]);
        return c00 * ((1.0f - fx) * (1.0f - fy)) + c10 * (fx * (1.0f - fy)) + c01 * ((1.0f - fx) * fy) + c11 * (fx * fy);
    }
    float3 LeSky(float3 wi, const Lut& lut)
    {
        const float theta = Math::ArcCos(wi.y);
        float phi = zr_atan2f(-wi.z, wi.x);
        phi = phi < 0 ? phi + TWO_PI : phi;
        float2 uv = f2(phi * ONE_OVER_2_PI, theta * ONE_OVER_PI);
        const float sn = theta >= PI_OVER_2 ? 1.0f : -1.0f;
        uv.y = mad(0.5f, theta, -PI_OVER_4);
        uv.y = 0.5f + sn * sqrtf(fabsf(uv.y) * ONE_OVER_PI);
        return Sample(lut, uv);
    }
    float3 LeSkyWithSunDisk(const zr_frame_constants& fc, const Lut& lut, uint32_t x, uint32_t y, bool* sun)
    {
        const float2 dim = f2((float)fc.RenderWidth, (float)fc.RenderHeight);
        const float2 uv = (f2((float)x, (float)y) + 0.5f + f2(fc.CurrCameraJitter[0], fc.CurrCameraJitter[1])) / dim;
        const float2 ndc = Math::NDCFromUV(uv);
        const float3 dv = f3(ndc.x * fc.AspectRatio * fc.TanHalfFOV, ndc.y * fc.TanHalfFOV, 1.0f);
        const float3 bx = f3(fc.CurrView[0][0], fc.CurrView[0][1], fc.CurrView[0][2]);
        const float3 by = f3(fc.CurrView[1][0], fc.CurrView[1][1], fc.CurrView[1][2]);
        const float3 bz = f3(fc.CurrView[2][0], fc.CurrView[2][1], fc.CurrView[2][2]);
        const float3 wc = normalize(mad(dv.x, bx, mad(dv.y, by, dv.z * bz)));
        float3 o = f3(0.0f, 1e-1f, 0.0f);
        o.y += fc.PlanetRadius;
        float3 wt = wc;
        wt.y = wt.y * fc.SunCosAngularRadius + sqrtf(1.0f - wc.y * wc.y) * fc.SunSinAngularRadius;
        float t;
        const bool hit = IntersectPlanet(fc.PlanetRadius, o, wt, t);
        *sun = dot(-wc, V3(fc.SunDir)) >= fc.SunCosAngularRadius && !hit;
        return *sun ? f3(fc.SunIlluminance) : LeSky(wc, lut);
    }
    bool Invalid(const uint32_t* core, size_t i) { return DecodeFlags(core[i * 4 + 3] & 0xff).invalid; }
}

extern "C"
{
    void sky_atan2f(const float* y, const float* x, uint32_t n, float* out)
    {
        for (uint32_t i = 0; i < n; i++) out[i] = zr_atan2f(y[i], x[i]);
    }
    void sky_view_lut(const zr_frame_constants* fc, uint32_t lut_w, uint32_t lut_h, uint32_t* out)
    {
        for (uint32_t y = 0; y < lut_h; y++)
            for (uint32_t x = 0; x < lut_w; x++)
                out[(size_t)y * lut_w + x] = LutTexel(*fc, x, y, lut_w, lut_h);
    }
    void sky_le_sky(const uint32_t* lut, uint32_t lut_w, uint32_t lut_h, const float* wi, uint32_t n, float* out)
    {
        const Lut l{ lut, lut_w, lut_h };
        for (uint32_t i = 0; i < n; i++)
        {
            const float3 c = LeSky(f3(wi[3 * i], wi[3 * i + 1], wi[3 * i + 2]), l);
            out[3 * i] = c.x; out[3 * i + 1] = c.y; out[3 * i + 2] = c.z;
        }
    }
    void sky_background(const zr_frame_constants* fc, const uint32_t* lut, uint32_t lut_w, uint32_t lut_h, float* out, uint8_t* sun)
    {
        const Lut l{ lut, lut_w, lut_h };
        for (uint32_t y = 0; y < fc->RenderHeight; y++)
            for (uint32_t x = 0; x < fc->RenderWidth; x++)
            {
                const size_t i = (size_t)y * fc->RenderWidth + x;
                bool s;
                const float3 c = LeSkyWithSunDisk(*fc, l, x, y, &s);
                out[3 * i] = c.x; out[3 * i + 1] = c.y; out[3 * i + 2] = c.z;
                if (sun) sun[i] = s ? 1 : 0;
            }
    }
    void sky_composite(const zr_frame_constants* fc, const uint32_t* core, const uint32_t* lut, uint32_t lut_w, uint32_t lut_h,
        uint32_t emissive_di, float* composited)
    {
        if (fc->Accumulate && fc->CameraStatic) return;
        const Lut l{ lut, lut_w, lut_h };
        for (uint32_t y = 0; y < fc->RenderHeight; y++)
            for (uint32_t x = 0; x < fc->RenderWidth; x++)
            {
                const size_t i = (size_t)y * fc->RenderWidth + x;
                if (!Invalid(core, i)) continue;
                bool s;
                const float3 c = emissive_di ? LeSkyWithSunDisk(*fc, l, x, y, &s) : f3(0.0f);
                composited[4 * i] = c.x; composited[4 * i + 1] = c.y; composited[4 * i + 2] = c.z; composited[4 * i + 3] = 0.0f;
            }
    }
    void sky_di_accumulate(const zr_frame_constants* fc, const uint32_t* core, const uint32_t* lut, uint32_t lut_w, uint32_t lut_h,
        const float* before, float* final_img)
    {
        if (!(fc->Accumulate && fc->CameraStatic)) return;
        const Lut l{ lut, lut_w, lut_h };
        const float keep = fc->NumFramesCameraStatic > 1 ? 1.0f : 0.0f;
        for (uint32_t y = 0; y < fc->RenderHeight; y++)
            for (uint32_t x = 0; x < fc->RenderWidth; x++)
            {
                const size_t i = (size_t)y * fc->RenderWidth + x;
                if (!Invalid(core, i)) continue;
                bool s;
                const float3 c = f3(before[4 * i], before[4 * i + 1], before[4 * i + 2]) * keep + LeSkyWithSunDisk(*fc, l, x, y, &s);
                final_img[4 * i] = c.x; final_img[4 * i + 1] = c.y; final_img[4 * i + 2] = c.z; final_img[4 * i + 3] = before[4 * i + 3];
            }
    }
}
