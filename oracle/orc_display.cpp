// ORACLE -- test infrastructure, not product code (see orc_math.h header).
//
// CPU restatement of the post-processing after TAA:
//   luminance histogram    ZetaRenderPass/AutoExposure/AutoExposure_Histogram.hlsl:22-74 (CalculateeBin)
//   exposure               AutoExposure_WeightedAvg.hlsl:20-110, SKIP_OUTSIDE_PERCENTILE_RANGE 0
//   display                Display/Display.hlsl:42-77 (DisplayOption::DEFAULT), Tonemap.hlsli, R8G8B8A8_UNORM_SRGB store
// Defined here (DESIGN 6): the bin values are summed in one pairwise tree (h = 128, 64, ..., 1), the LUT is filtered with
// float weights, the sRGB OETF is the exact IEC 61966-2-1 curve. Transcendentals are zr_fpmath.h's, as on the device.
#include "orc_api.h"
#include "orc_math.h"

using namespace orc;

namespace
{
    constexpr uint32_t BINS = 256;
    constexpr uint32_t LUT_N = 48;

    uint32_t Bin(const float* rgba, const zr_auto_exposure_params& p)
    {
        // Texture2D<half4> view of the RGBA32F signal
        const float3 c = f3(to_half(rgba[0]), to_half(rgba[1]), to_half(rgba[2]));
        const float lum = Math::Luminance(c);
        if (lum <= 1e-4f)
            return 0;
        const float range = p.max_lum - p.min_lum;
        float t = saturate((lum - p.min_lum) / range);
        t = zr_powf(t, p.lum_map_exp);
        uint32_t bin = (uint32_t)(t * 254.0f) + 1;
        if (bin > BINS - 1) bin = BINS - 1;
        return bin;
    }

    float Exposure(float avgLum)
    {
        const float ev100 = zr_log2f((avgLum * 100.0f) / 12.5f);
        const float lumMax = (78.0f / (0.65f * 100.0f)) * zr_powf(2.0f, ev100);
        return 1.0f / lumMax;
    }

    float Rgb9e5(uint32_t v, int channel)
    {
        const int e = (int)(v >> 27);
        const uint32_t m = (v >> (9 * channel)) & 0x1ff;
        return (float)m * ldexpf(1.0f, e - 15 - 9);
    }

    // Texture3D SampleLevel, linear filter, clamp addressing, float weights: x, then y, then z
    float3 SampleLut(const uint32_t* lut, float3 uv)
    {
        float t[3] = { uv.x * 48.0f - 0.5f, uv.y * 48.0f - 0.5f, uv.z * 48.0f - 0.5f };
        uint32_t i0[3], i1[3];
        float f[3];
        for (int a = 0; a < 3; a++)
        {
            t[a] = fminf(fmaxf(t[a], 0.0f), 47.0f);
            i0[a] = (uint32_t)floorf(t[a]);
            i1[a] = i0[a] + 1 < LUT_N ? i0[a] + 1 : LUT_N - 1;
            f[a] = t[a] - (float)i0[a];
        }
        float out[3];
        for (int ch = 0; ch < 3; ch++)
        {
            auto T = [&](uint32_t x, uint32_t y, uint32_t z) { return Rgb9e5(lut[((size_t)z * LUT_N + y) * LUT_N + x], ch); };
            const float c00 = Math::Lerp(T(i0[0], i0[1], i0[2]), T(i1[0], i0[1], i0[2]), f[0]);
            const float c10 = Math::Lerp(T(i0[0], i1[1], i0[2]), T(i1[0], i1[1], i0[2]), f[0]);
            const float c01 = Math::Lerp(T(i0[0], i0[1], i1[2]), T(i1[0], i0[1], i1[2]), f[0]);
            const float c11 = Math::Lerp(T(i0[0], i1[1], i1[2]), T(i1[0], i1[1], i1[2]), f[0]);
            out[ch] = Math::Lerp(Math::Lerp(c00, c10, f[1]), Math::Lerp(c01, c11, f[1]), f[2]);
        }
        return f3(out[0], out[1], out[2]);
    }

    float3 TonyMcMapface(float3 s, const uint32_t* lut)
    {
        const float3 encoded = s / (s + 1.0f);
        const float3 uv = encoded * (47.0f / 48.0f) + 0.5f / 48.0f;
        return SampleLut(lut, uv);
    }

    // mul(v, M) for a float3x3 written row by row: out_j = v.x M[0][j] + v.y M[1][j] + v.z M[2][j]
    float3 Mul(float3 v, const float M[9])
    {
        float o[3];
        for (int j = 0; j < 3; j++)
            o[j] = fmaf(v.z, M[6 + j], fmaf(v.y, M[3 + j], v.x * M[j]));
        return f3(o[0], o[1], o[2]);
    }

    float Contrast(float x)
    {
        const float x2 = x * x;
        const float x4 = x2 * x2;
        const float x6 = x4 * x2;
        float r = -17.86f * x6 * x;
        r = r + 78.01f * x6;
        r = r - 126.7f * x4 * x;
        r = r + 92.06f * x4;
        r = r - 28.72f * x2 * x;
        r = r + 4.361f * x2;
        r = r - 0.1718f * x;
        return r + 0.002857f;
    }

    float3 AgxInset(float3 v)
    {
        static const float M[9] = { 0.842479062253094f, 0.0423282422610123f, 0.0423756549057051f,
                                    0.0784335999999992f, 0.878468636469772f, 0.0784336f,
                                    0.0792237451477643f, 0.0791661274605434f, 0.879142973793104f };
        const float minEv = -12.47393f, maxEv = 4.026069f;
        v = Mul(v, M);
        float c[3] = { v.x, v.y, v.z };
        for (int a = 0; a < 3; a++)
        {
            float l = fminf(fmaxf(zr_log2f(c[a]), minEv), maxEv);
            c[a] = Contrast((l - minEv) / (maxEv - minEv));
        }
        return f3(c[0], c[1], c[2]);
    }

    float3 AgxEotf(float3 v)
    {
        static const float M[9] = { 1.19687900512017f, -0.0528968517574562f, -0.0529716355144438f,
                                    -0.0980208811401368f, 1.15190312990417f, -0.0980434501171241f,
                                    -0.0990297440797205f, -0.0989611768448433f, 1.15107367264116f };
        v = Mul(v, M);
        return f3(zr_powf(v.x, 2.2f), zr_powf(v.y, 2.2f), zr_powf(v.z, 2.2f));
    }

    float3 AgxLook(float3 v, float3 slope, float power, float sat)
    {
        const float luma = Math::Luminance(v);
        const float3 s = v * slope + 0.0f;
        const float3 p = f3(zr_powf(s.x, power), zr_powf(s.y, power), zr_powf(s.z, power));
        return f3(luma + sat * (p.x - luma), luma + sat * (p.y - luma), luma + sat * (p.z - luma));
    }

    float3 Tonemap(float3 c, const zr_display_params& p, const uint32_t* lut)
    {
        switch (p.tonemapper)
        {
        case ZR_TONEMAPPER_NEUTRAL:
        {
            const float3 t = TonyMcMapface(c, lut);
            const float l = Math::Luminance(t);
            return f3(Math::Lerp(l, t.x, p.saturation), Math::Lerp(l, t.y, p.saturation), Math::Lerp(l, t.z, p.saturation));
        }
        case ZR_TONEMAPPER_AGX_DEFAULT: return AgxEotf(AgxInset(c));
        case ZR_TONEMAPPER_AGX_GOLDEN: return AgxEotf(AgxLook(AgxInset(c), f3(1.0f, 0.9f, 0.5f), 0.8f, 0.8f));
        case ZR_TONEMAPPER_AGX_PUNCHY: return AgxEotf(AgxLook(AgxInset(c), f3(1.0f), 1.35f, 1.4f));
        case ZR_TONEMAPPER_AGX_CUSTOM: return AgxEotf(AgxLook(AgxInset(c), f3(1.0f), p.agx_exp, p.saturation));
        default: return c;
        }
    }

    float Oetf(float v)
    {
        if (v <= 0.0031308f)
            return 12.92f * v;
        return 1.055f * zr_powf(v, 1.0f / 2.4f) - 0.055f;
    }
}

extern "C"
{
    // signal: float4[n]; bins[n]
    void orc_lum_bins(const float* signal, int64_t n, const zr_auto_exposure_params* p, uint32_t* bins)
    {
        for (int64_t i = 0; i < n; i++)
            bins[i] = Bin(signal + 4 * i, *p);
    }

    // adds the pixels of rows [y0, y1) of a W-wide float4 image to hist[256]
    void orc_lum_histogram(const float* signal, uint32_t W, uint32_t y0, uint32_t y1, const zr_auto_exposure_params* p, uint32_t* hist)
    {
        for (size_t i = (size_t)y0 * W; i < (size_t)y1 * W; i++)
            hist[Bin(signal + 4 * i, *p)]++;
    }

    // one k_exposure: state = {exposure, adapted luminance} in and out; numPixels = RenderWidth * RenderHeight
    void orc_exposure(const uint32_t* hist, uint32_t numPixels, const zr_auto_exposure_params* p, float dt, float* state)
    {
        float s[BINS];
        for (uint32_t i = 0; i < BINS; i++)
            s[i] = i == 0 ? 0.0f : ((float)hist[i] * ((float)(i - 1) + 0.5f)) / 256.0f;
        for (uint32_t h = BINS / 2; h > 0; h /= 2)
            for (uint32_t i = 0; i < h; i++)
                s[i] = s[i] + s[i + h];
        uint32_t numSamples = numPixels - hist[0];
        if (numSamples < 1) numSamples = 1;
        const float mean = s[0] / (float)numSamples;
        float result = zr_powf(mean, 1.0f / p->lum_map_exp);
        result = result * (p->max_lum - p->min_lum) + p->min_lum;
        const float prev = state[1];
        if (prev < 1e8f)
            result = prev + (result - prev) * (1.0f - zr_expf(-dt * 1000.0f * p->adaptation_rate));
        state[0] = Exposure(result);
        state[1] = result;
    }

    // rows [y0, y1) of a W-wide half4 image -> RGBA8 (alpha 255); exposure: float2 state or null (auto exposure off)
    void orc_display(const uint16_t* taa, uint32_t W, uint32_t y0, uint32_t y1, const zr_display_params* p, const float* exposure,
        const uint32_t* lut, uint32_t* out)
    {
        for (size_t i = (size_t)y0 * W; i < (size_t)y1 * W; i++)
        {
            float3 c = f3(zr_f16_to_f32(taa[4 * i]), zr_f16_to_f32(taa[4 * i + 1]), zr_f16_to_f32(taa[4 * i + 2]));
            if (p->auto_exposure)
                c = c * exposure[0];
            c = saturate(Tonemap(c, *p, lut));
            out[i] = Math::FloatToUNorm8(Oetf(c.x)) | Math::FloatToUNorm8(Oetf(c.y)) << 8 | Math::FloatToUNorm8(Oetf(c.z)) << 16 |
                0xff000000u;
        }
    }

    // building blocks for the independent float64 checks
    void orc_rgb9e5_decode(const uint32_t* v, int64_t n, float* rgb)
    {
        for (int64_t i = 0; i < n; i++)
            for (int ch = 0; ch < 3; ch++)
                rgb[3 * i + ch] = Rgb9e5(v[i], ch);
    }
    void orc_srgb_oetf(const float* v, int64_t n, float* out)
    {
        for (int64_t i = 0; i < n; i++)
            out[i] = Oetf(v[i]);
    }
    // the tone mapper alone (after exposure, before saturate): rgb[n][3] -> out[n][3]
    void orc_tonemap(const float* rgb, int64_t n, const zr_display_params* p, const uint32_t* lut, float* out)
    {
        for (int64_t i = 0; i < n; i++)
        {
            const float3 c = Tonemap(f3(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]), *p, lut);
            out[3 * i] = c.x; out[3 * i + 1] = c.y; out[3 * i + 2] = c.z;
        }
    }
}
