// ORACLE -- test infrastructure, not product code (see orc_math.h header).
//
// CPU restatement of the post stencils (SURVEY 8a-18):
//   Compositing            ZetaRenderPass/Compositing/Compositing.hlsl:30-126
//   FilterFirefly          ZetaRenderPass/Compositing/FireflyFilter.hlsl:35-124
//   TAA                    ZetaRenderPass/TAA/TAA.hlsl:29-189, Common/Common.hlsli:65-102 (Catmull-Rom)
// The reference has no tests or golden images for these passes; oracle/indep_post.py is an independent float64 truth of them,
// and tests/test_post_oracle.py holds this file to it.
// Documented deviations (DESIGN.md): sky/sun-disk background for invalid pixels is out of scope
// (writes 0); the firefly filter reads an input image and writes a separate output (the reference
// filters in place and races with itself); bilinear history taps use exact float weights.
#include "orc_api.h"
#include "orc_gbuffer.h"

using namespace orc;

extern "C"
{
    // direct / indirect: float4[w*h] or null; out: float4[w*h]
    void orc_compositing(const zr_frame_constants* fc, const uint32_t* core_, const float* direct_,
        const float* indirect_, float* out_)
    {
        const uint4* core = (const uint4*)core_;
        const float4* direct = (const float4*)direct_;
        const float4* indirect = (const float4*)indirect_;
        float4* out = (float4*)out_;
        const uint32_t W = fc->RenderWidth, H = fc->RenderHeight;
        const bool accumulate = fc->Accumulate && fc->CameraStatic;
        const uint32_t numFramesAccumulated = accumulate ? fc->NumFramesCameraStatic : 1;
        for (uint32_t y = 0; y < H; y++)
            for (uint32_t x = 0; x < W; x++)
            {
                size_t i = (size_t)y * W + x;
                GFlags flags = DecodeFlags(core[i].w & 0xff);
                if (flags.invalid && !accumulate)
                {
                    out[i] = f4(0, 0, 0, 0);
                    continue;
                }
                float3 color = f3(0);
                if (direct)
                    color += f3(direct[i].x, direct[i].y, direct[i].z);
                if (indirect && !flags.emissive)
                    color += f3(indirect[i].x, indirect[i].y, indirect[i].z);
                color = color / (float)numFramesAccumulated;
                out[i] = f4(color.x, color.y, color.z, 0);
            }
    }

    void orc_firefly(const zr_frame_constants* fc, const uint32_t* core_, const float* in_, float* out_)
    {
        const uint4* core = (const uint4*)core_;
        const float4* in = (const float4*)in_;
        float4* out = (float4*)out_;
        const int W = (int)fc->RenderWidth, H = (int)fc->RenderHeight;
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++)
            {
                size_t idx = (size_t)y * W + x;
                const float z_view = asfloat(core[idx].x);
                float3 currColor = f3(in[idx].x, in[idx].y, in[idx].z);
                if (z_view == FLT_MAX_)
                {
                    out[idx] = f4(currColor.x, currColor.y, currColor.z, 0);
                    continue;
                }
                float minLum = FLT_MAX_;
                float maxLum = 0.0f;
                float3 minColor = currColor;
                float3 maxColor = f3(0);
                float currLum = Math::Luminance(currColor);
                for (int i = -1; i <= 1; i++)
                    for (int j = -1; j <= 1; j++)
                    {
                        if (i == 0 && j == 0)
                            continue;
                        int ax = x + j, ay = y + i;
                        // int2 >= uint2 compares as unsigned: negative addresses are skipped too
                        if ((uint32_t)ax >= (uint32_t)W || (uint32_t)ay >= (uint32_t)H)
                            continue;
                        size_t n = (size_t)ay * W + ax;
                        const float neighborLinearDepth = asfloat(core[n].x);
                        if (neighborLinearDepth == FLT_MAX_)
                            continue;
                        float3 neighborColor = f3(in[n].x, in[n].y, in[n].z);
                        float neighborLum = Math::Luminance(neighborColor);
                        if (neighborLum < minLum) { minLum = neighborLum; minColor = neighborColor; }
                        else if (neighborLum > maxLum) { maxLum = neighborLum; maxColor = neighborColor; }
                    }
                float3 ret = currLum < minLum ? minColor : (currLum > maxLum ? maxColor : currColor);
                ret = minLum <= maxLum ? ret : currColor;
                out[idx] = f4(ret.x, ret.y, ret.z, 0);
            }
    }

    static float Mitchell1D(float x, float B, float C)
    {
        x = fabsf(2.0f * x);
        const float oneDivSix = 1.0f / 6.0f;
        if (x > 1)
            return ((-B - 6.0f * C) * x * x * x + (6.0f * B + 30.0f * C) * x * x +
                (-12.0f * B - 48.0f * C) * x + (8.0f * B + 24.0f * C)) * oneDivSix;
        else
            return ((12.0f - 9.0f * B - 6.0f * C) * x * x * x + (-18.0f + 12.0f * B + 6.0f * C) * x * x +
                (6.0f - 2.0f * B)) * oneDivSix;
    }

    static float3 LoadHalf4(const uint2* img, int W, int H, int x, int y)
    {
        x = x < 0 ? 0 : (x > W - 1 ? W - 1 : x);
        y = y < 0 ? 0 : (y > H - 1 ? H - 1 : y);
        uint2 p = img[(size_t)y * W + x];
        return f3(half_lo(p.x), half_hi(p.x), half_lo(p.y));
    }

    // Common::SampleTextureCatmullRom (Common.hlsli:65-102): nine g_samLinearClamp SampleLevel taps on the RGBA16F history. By
    // construction every tap lies either at a texel centre (texPos0 = texPos1 - 1, texPos3 = texPos1 + 2: the sampler returns that texel)
    // or between the two middle texels at the fraction offset12 (texPos12 = texPos1 + offset12: the sampler's bilinear weight). That is
    // what is restated here -- centre taps are the texel, the 1|2 taps blend the two middle texels with the float fraction offset12 (the
    // hardware quantises it to 8 fractional bits; not modelled) -- instead of pushing the positions through uv = pos / texSize and back,
    // whose rounding would turn exact texel centres into 4-texel blends with weights of 1e-7. Clamp addressing on the texel indices.
    static float3 SampleTextureCatmullRom(const uint2* img, int W, int H, float2 uv, float2 texSize)
    {
        float2 samplePos = uv * texSize;
        const float fx1 = floorf(samplePos.x - 0.5f), fy1 = floorf(samplePos.y - 0.5f);
        float2 texPos1 = f2(fx1 + 0.5f, fy1 + 0.5f);
        float2 f = samplePos - texPos1;
        auto w0f = [](float f) { return f * (-0.5f + f * (1.0f - 0.5f * f)); };
        auto w1f = [](float f) { return 1.0f + f * f * (-2.5f + 1.5f * f); };
        auto w2f = [](float f) { return f * (0.5f + f * (2.0f - 1.5f * f)); };
        auto w3f = [](float f) { return f * f * (-0.5f + 0.5f * f); };
        float2 w0 = f2(w0f(f.x), w0f(f.y)), w1 = f2(w1f(f.x), w1f(f.y));
        float2 w2 = f2(w2f(f.x), w2f(f.y)), w3 = f2(w3f(f.x), w3f(f.y));
        float2 w12 = w1 + w2;
        float2 offset12 = w2 / (w1 + w2);
        const int ix = (int)fx1, iy = (int)fy1;       // texel under texPos1
        auto T = [&](int i, int j) { return LoadHalf4(img, W, H, ix + i, iy + j); };
        auto lerp = [](float3 a, float3 b, float t) { return a * (1.0f - t) + b * t; };
        const float ox = offset12.x, oy = offset12.y;
        float3 result = f3(0);
        result += T(-1, -1) * w0.x * w0.y;
        result += lerp(T(0, -1), T(1, -1), ox) * w12.x * w0.y;
        result += T(2, -1) * w3.x * w0.y;
        result += lerp(T(-1, 0), T(-1, 1), oy) * w0.x * w12.y;
        result += lerp(lerp(T(0, 0), T(1, 0), ox), lerp(T(0, 1), T(1, 1), ox), oy) * w12.x * w12.y;
        result += lerp(T(2, 0), T(2, 1), oy) * w3.x * w12.y;
        result += T(-1, 2) * w0.x * w3.y;
        result += lerp(T(0, 2), T(1, 2), ox) * w12.x * w3.y;
        result += T(2, 2) * w3.x * w3.y;
        return result;
    }

    static float3 ClipAABB(float3 aabbMin, float3 aabbMax, float3 histSample)
    {
        float3 center = 0.5f * (aabbMax + aabbMin);
        float3 extents = 0.5f * (aabbMax - aabbMin);
        float3 rayToCenter = histSample - center;
        float3 rayToCenterUnit = abs3(rayToCenter / extents);
        float m = fmaxf(rayToCenterUnit.x, fmaxf(rayToCenterUnit.y, rayToCenterUnit.z));
        if (m > 1.0f)
            return center + rayToCenter / m;
        return histSample;
    }

    // signal: float4[w*h]; prevOut / out: half4 as uint2[w*h]
    void orc_taa(const zr_frame_constants* fc, const uint32_t* core_, const uint32_t* motionEmissive_,
        const float* signal_, const uint32_t* prevOut_, uint32_t* out_, float blendWeight, int temporalIsValid)
    {
        const uint4* core = (const uint4*)core_;
        const uint2* motionEmissive = (const uint2*)motionEmissive_;
        const float4* signal = (const float4*)signal_;
        const uint2* prevOut = (const uint2*)prevOut_;
        uint2* out = (uint2*)out_;
        const int W = (int)fc->RenderWidth, H = (int)fc->RenderHeight;
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++)
            {
                size_t idx = (size_t)y * W + x;
                const float depth = asfloat(core[idx].x);
                const float3 currColor = f3(signal[idx].x, signal[idx].y, signal[idx].z);
                auto store = [&](float3 c) { out[idx] = uint2{ pack_half2(c.x, c.y), pack_half2(c.z, 0.0f) }; };
                if (!temporalIsValid || depth == FLT_MAX_) { store(currColor); continue; }

                float weightSum = Mitchell1D(0, 0.33f, 0.33f) * Mitchell1D(0, 0.33f, 0.33f);
                float3 reconstructed = currColor * weightSum;
                float3 firstMoment = currColor;
                float3 secondMoment = currColor * currColor;
                float closestDepth = depth;
                int cdx = 0, cdy = 0;
                int numNeighbors = 1;
                for (int i = -1; i < 2; i++)
                    for (int j = -1; j < 2; j++)
                    {
                        if (i == 0 && j == 0) continue;
                        int nx = x + i, ny = y + j;
                        if (nx < 0 || ny < 0 || nx >= W || ny >= H) continue;
                        size_t n = (size_t)ny * W + nx;
                        float3 neighborColor = max3(f3(signal[n].x, signal[n].y, signal[n].z), 0.0f);
                        float weight = Mitchell1D((float)i, 0.33f, 0.33f) * Mitchell1D((float)j, 0.33f, 0.33f);
                        weight *= 1.0f / (1.0f + Math::Luminance(neighborColor));
                        reconstructed += neighborColor * weight;
                        weightSum += weight;
                        firstMoment += neighborColor;
                        secondMoment += neighborColor * neighborColor;
                        float neighborDepth = asfloat(core[n].x);
                        if (neighborDepth < closestDepth) { closestDepth = neighborDepth; cdx = i; cdy = j; }
                        numNeighbors += 1;
                    }
                reconstructed = reconstructed / fmaxf(weightSum, 1e-5f);
                const float2 motionVec = unpack_snorm16x2(motionEmissive[(size_t)(y + cdy) * W + (x + cdx)].x);
                const float2 renderDim = f2((float)W, (float)H);
                const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / renderDim;
                const float2 prevUV = currUV - motionVec;
                if (prevUV.x < 0.0f || prevUV.y < 0.0f || prevUV.x > 1.0f || prevUV.y > 1.0f) { store(reconstructed); continue; }

                float3 history = SampleTextureCatmullRom(prevOut, W, H, prevUV, renderDim);
                const float3 mean = firstMoment / (float)numNeighbors;
                float3 std = abs3(secondMoment - (firstMoment * firstMoment) / (float)numNeighbors);
                std = std / ((float)numNeighbors - 1.0f);
                std = sqrt3(std);
                const float3 clippedHistory = ClipAABB(mean - std, mean + std, history);
                const float currWeight = saturate(blendWeight * (1.0f / (1.0f + Math::Luminance(reconstructed))));
                const float histWeight = saturate((1.0f - blendWeight) * (1.0f / (1.0f + Math::Luminance(clippedHistory))));
                float3 result = (currWeight * reconstructed + histWeight * clippedHistory) / (currWeight + histWeight);
                result = isnan3(result) ? reconstructed : result;
                store(result);
            }
    }
}
