// post.cu -- compositing, firefly filter and TAA stencils (HBM-bound kernels).
//
// Replaces Compositing/Compositing.hlsl:30-126, Compositing/FireflyFilter.hlsl:35-124 and
// TAA/TAA.hlsl:29-189 (+ Common.hlsli:65-102 Catmull-Rom history fetch) and their host passes
// (Compositing.cpp:83-145, TAA.cpp:87-123).
//
// Notes: these kernels move bytes and nothing else. Compositing is elementwise, so when the
// firefly filter is on it is fused into the 3x3 stencil (each tap recomposites from the two lighting
// images; the neighbour taps are L1/L2 hits) which removes one 16 B/px write + one 16 B/px read of
// the reference's two-dispatch sequence. The filter writes a second image instead of filtering in
// place (the reference's in-place UAV update races with its own neighbour reads).
#include "zr_common.cuh"
#include "zr_planes.h"
#include "zr_sky.cuh"
#include "zr_schedule.h"

namespace zr
{
namespace
{
    struct PostParams
    {
        uint32_t W, H;
        uint32_t accumulate;            // Accumulate && CameraStatic
        uint32_t numFramesAccumulated;
        float blendWeight;
        uint32_t temporalIsValid;
        uint32_t rowBegin, rowEnd;      // rows this device owns (strip-sharded frames); the whole image by default
    };

    // The sky behind geometry (zr_compositing_pass_set_sky); only the SKY instantiations read it
    struct SkyArgs
    {
        Sky::LutView lut;
        uint32_t emissiveDI;
        zr_frame_constants fc;
    };

    // SKY: invalid pixels of non-accumulating frames show Le_SkyWithSunDisk when emissive direct lighting is on (Compositing.hlsl:43-47)
    template<bool SKY>
    ZR_D float3 composite_px(const uint4* __restrict__ core, const float4* __restrict__ direct,
        const float4* __restrict__ indirect, size_t i, const PostParams& p, const SkyArgs& sky, uint32_t x, uint32_t y)
    {
        const uint32_t flags = __ldg(&core[i].w) & 0xffu;
        if ((flags & ZR_GBUFFER_FLAG_INVALID) && !p.accumulate)
        {
            if constexpr (SKY)
                return sky.emissiveDI ? Sky::Le_SkyWithSunDisk(sky.fc, sky.lut, x, y) : f3(0);
            return f3(0);
        }
        float3 color = f3(0);
        if (direct)
        {
            float4 d = __ldg(&direct[i]);
            color += f3(d.x, d.y, d.z);
        }
        if (indirect && !(flags & ZR_GBUFFER_FLAG_EMISSIVE))
        {
            float4 d = __ldg(&indirect[i]);
            color += f3(d.x, d.y, d.z);
        }
        return color / (float)p.numFramesAccumulated;
    }

    template<bool SKY>
    __global__ void __launch_bounds__(256) k_compositing(const uint4* __restrict__ core,
        const float4* __restrict__ direct, const float4* __restrict__ indirect, float4* __restrict__ out, PostParams p, SkyArgs sky)
    {
        const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31);
        const uint32_t y = p.rowBegin + blockIdx.y * 8 + (threadIdx.x >> 5);
        if (x >= p.W || y >= p.rowEnd) return;
        const size_t i = (size_t)y * p.W + x;
        float3 c = composite_px<SKY>(core, direct, indirect, i, p, sky, x, y);
        out[i] = f4(c.x, c.y, c.z, 0.0f);
    }

    // Shared-memory-tiled fused compositing + firefly stencil. A block owns a 32 x 16 pixel tile: every pixel
    // of the 34 x 18 halo'd tile is composited ONCE (1.2 composites per output pixel instead of 9 -- an untiled kernel
    // re-composites each tap, 27 IEEE divisions per pixel, and is issue-bound, not bandwidth-bound), its luminance and
    // "has geometry" flag are staged next to it, and the 3 x 3 min / max search then runs out of shared memory in the
    // reference's tap order, so the result is bit-identical to the oracle. Rows are read as contiguous 34-pixel segments
    // (coalesced 128-bit loads).
    constexpr int FF_TW = 32, FF_TH = 16, FF_SW = FF_TW + 2, FF_SH = FF_TH + 2;
    template<bool SKY>
    __global__ void __launch_bounds__(FF_TW * FF_TH) k_firefly_tiled(const uint4* __restrict__ core, const float* __restrict__ depth,
        const float4* __restrict__ direct, const float4* __restrict__ indirect, float4* __restrict__ out, PostParams p, SkyArgs sky)
    {
        __shared__ float4 tile[FF_SH][FF_SW];           // xyz = (composited) colour, w = its luminance
        __shared__ uint8_t geom[FF_SH][FF_SW];          // 1 = inside the image and depth != FLT_MAX
        const int W = (int)p.W, H = (int)p.H;
        const int x0 = blockIdx.x * FF_TW;
        const int y0 = (int)p.rowBegin + blockIdx.y * FF_TH;
        for (int e = threadIdx.x; e < FF_SW * FF_SH; e += FF_TW * FF_TH)
        {
            const int ty = e / FF_SW, tx = e - ty * FF_SW;
            const int gx = x0 - 1 + tx, gy = y0 - 1 + ty;
            float4 v = f4(0.0f, 0.0f, 0.0f, 0.0f);
            uint8_t g = 0;
            if ((uint32_t)gx < (uint32_t)W && (uint32_t)gy < (uint32_t)H)
            {
                const size_t i = (size_t)gy * W + gx;
                const float3 c = composite_px<SKY>(core, direct, indirect, i, p, sky, (uint32_t)gx, (uint32_t)gy);
                v = f4(c.x, c.y, c.z, Math::Luminance(c));
                g = __ldg(&depth[i]) != FLT_MAX_ ? 1 : 0;
            }
            tile[ty][tx] = v;
            geom[ty][tx] = g;
        }
        __syncthreads();
        const int lx = threadIdx.x & (FF_TW - 1), ly = threadIdx.x / FF_TW;
        const int x = x0 + lx, y = y0 + ly;
        if (x >= W || y >= (int)p.rowEnd) return;
        const size_t idx = (size_t)y * W + x;
        const float4 c4 = tile[ly + 1][lx + 1];
        const float3 currColor = f3(c4.x, c4.y, c4.z);
        if (!geom[ly + 1][lx + 1])
        {
            out[idx] = f4(currColor.x, currColor.y, currColor.z, 0.0f);
            return;
        }
        float minLum = FLT_MAX_;
        float maxLum = 0.0f;
        float3 minColor = currColor;
        float3 maxColor = f3(0);
        const float currLum = c4.w;
#pragma unroll
        for (int i = -1; i <= 1; i++)
        {
#pragma unroll
            for (int j = -1; j <= 1; j++)
            {
                if (i == 0 && j == 0) continue;
                if (!geom[ly + 1 + i][lx + 1 + j]) continue;
                const float4 n4 = tile[ly + 1 + i][lx + 1 + j];
                const float3 neighborColor = f3(n4.x, n4.y, n4.z);
                const float neighborLum = n4.w;
                if (neighborLum < minLum) { minLum = neighborLum; minColor = neighborColor; }
                else if (neighborLum > maxLum) { maxLum = neighborLum; maxColor = neighborColor; }
            }
        }
        float3 ret = currLum < minLum ? minColor : (currLum > maxLum ? maxColor : currColor);
        ret = minLum <= maxLum ? ret : currColor;
        out[idx] = f4(ret.x, ret.y, ret.z, 0.0f);
    }

    ZR_D float Mitchell1D(float x, float B, float C)
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

    ZR_D float3 LoadHalf4(const uint2* __restrict__ img, int W, int H, int x, int y)
    {
        x = x < 0 ? 0 : (x > W - 1 ? W - 1 : x);
        y = y < 0 ? 0 : (y > H - 1 ? H - 1 : y);
        const uint2 p = __ldg(&img[(size_t)y * W + x]);
        return f3(half_lo(p.x), half_hi(p.x), half_lo(p.y));
    }

    // Common::SampleTextureCatmullRom (Common.hlsli:65-102) on the RGBA16F history. The reference's nine bilinear taps lie at texel
    // centres (texPos0, texPos3: the sampler returns the texel) or between the two middle texels at the fraction offset12 (texPos12), so
    // they cover a 4 x 4 texel footprint: 16 loads (clamp addressing), the 1|2 taps blended with offset12, then the nine weighted taps
    // in the reference's order (oracle/orc_post.cpp restates exactly this).
    ZR_D float3 HalfRGB(uint2 p) { return f3(half_lo(p.x), half_hi(p.x), half_lo(p.y)); }
    ZR_D float3 Lerp3(float3 a, float3 b, float t) { return a * (1.0f - t) + b * t; }

    ZR_D float3 SampleTextureCatmullRom(const uint2* __restrict__ img, int W, int H, float2 uv, float2 texSize)
    {
        const float2 samplePos = uv * texSize;
        const float fx1 = floorf(samplePos.x - 0.5f), fy1 = floorf(samplePos.y - 0.5f);
        const float2 texPos1 = f2(fx1 + 0.5f, fy1 + 0.5f);
        const float2 f = samplePos - texPos1;
        const float2 w0 = f2(f.x * (-0.5f + f.x * (1.0f - 0.5f * f.x)), f.y * (-0.5f + f.y * (1.0f - 0.5f * f.y)));
        const float2 w1 = f2(1.0f + f.x * f.x * (-2.5f + 1.5f * f.x), 1.0f + f.y * f.y * (-2.5f + 1.5f * f.y));
        const float2 w2 = f2(f.x * (0.5f + f.x * (2.0f - 1.5f * f.x)), f.y * (0.5f + f.y * (2.0f - 1.5f * f.y)));
        const float2 w3 = f2(f.x * f.x * (-0.5f + 0.5f * f.x), f.y * f.y * (-0.5f + 0.5f * f.y));
        const float2 w12 = w1 + w2;
        const float2 offset12 = w2 / (w1 + w2);
        const int ix = (int)fx1, iy = (int)fy1;
        int cx[4]; size_t row[4];
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            const int tx = ix - 1 + k, ty = iy - 1 + k;
            cx[k] = tx < 0 ? 0 : (tx > W - 1 ? W - 1 : tx);
            row[k] = (size_t)(ty < 0 ? 0 : (ty > H - 1 ? H - 1 : ty)) * W;
        }
        uint2 t[4][4];
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int i = 0; i < 4; i++)
                t[j][i] = __ldg(&img[row[j] + cx[i]]);
        const float ox = offset12.x, oy = offset12.y;
        float3 result = f3(0);
        result += HalfRGB(t[0][0]) * w0.x * w0.y;
        result += Lerp3(HalfRGB(t[0][1]), HalfRGB(t[0][2]), ox) * w12.x * w0.y;
        result += HalfRGB(t[0][3]) * w3.x * w0.y;
        result += Lerp3(HalfRGB(t[1][0]), HalfRGB(t[2][0]), oy) * w0.x * w12.y;
        result += Lerp3(Lerp3(HalfRGB(t[1][1]), HalfRGB(t[1][2]), ox), Lerp3(HalfRGB(t[2][1]), HalfRGB(t[2][2]), ox), oy) * w12.x * w12.y;
        result += Lerp3(HalfRGB(t[1][3]), HalfRGB(t[2][3]), oy) * w3.x * w12.y;
        result += HalfRGB(t[3][0]) * w0.x * w3.y;
        result += Lerp3(HalfRGB(t[3][1]), HalfRGB(t[3][2]), ox) * w12.x * w3.y;
        result += HalfRGB(t[3][3]) * w3.x * w3.y;
        return result;
    }

    ZR_D float3 ClipAABB(float3 aabbMin, float3 aabbMax, float3 histSample)
    {
        const float3 center = 0.5f * (aabbMax + aabbMin);
        const float3 extents = 0.5f * (aabbMax - aabbMin);
        const float3 rayToCenter = histSample - center;
        const float3 u = abs3(rayToCenter / extents);
        const float m = fmaxf(u.x, fmaxf(u.y, u.z));
        if (m > 1.0f)
            return center + rayToCenter / m;
        return histSample;
    }

    // TAA.hlsl:29-189. A block owns 32 x 8 pixels. The 3 x 3 neighbourhood is staged once per tile: every pixel of the 34 x 10 halo'd tile is
    // clamped to >= 0 and gets its tone-mapping weight 1 / (1 + luminance) ONCE (the per-tap form costs eight IEEE divisions per output
    // pixel), depth beside it; the taps then run out of shared memory in the reference's order with the reference's arithmetic.
    // 5 blocks per SM = 48 registers, chosen over 62 (4 blocks) and 40 (6 blocks)
    __global__ void __launch_bounds__(256, 5) k_taa(const float* __restrict__ depthPlane,
        const uint2* __restrict__ motionEmissive, const float4* __restrict__ signal,
        const uint2* __restrict__ prevOut, uint2* __restrict__ out, PostParams p)
    {
        constexpr int SW = 34, SH = 10;
        __shared__ float4 s_c[SH * SW];     // {max(rgb, 0), 1 / (1 + luminance)}
        __shared__ float s_d[SH * SW];
        const int W = (int)p.W, H = (int)p.H;
        const int bx = blockIdx.x * 32, by = (int)p.rowBegin + blockIdx.y * 8;
        if (p.temporalIsValid)
        {
            for (int e = (int)threadIdx.x; e < SW * SH; e += 256)
            {
                const int gx = bx + e % SW - 1, gy = by + e / SW - 1;
                float4 v = f4(0, 0, 0, 0);
                float d = FLT_MAX_;
                if (gx >= 0 && gy >= 0 && gx < W && gy < H)
                {
                    const size_t n = (size_t)gy * W + gx;
                    const float4 c4 = __ldg(&signal[n]);
                    const float3 c = max3(f3(c4.x, c4.y, c4.z), 0.0f);
                    v = f4(c.x, c.y, c.z, 1.0f / (1.0f + Math::Luminance(c)));
                    d = __ldg(&depthPlane[n]);
                }
                s_c[e] = v; s_d[e] = d;
            }
            __syncthreads();
        }
        const int lx = (int)(threadIdx.x & 31), ly = (int)(threadIdx.x >> 5);
        const int x = bx + lx, y = by + ly;
        if (x >= W || y >= (int)p.rowEnd) return;
        const size_t idx = (size_t)y * W + x;
        const float depth = __ldg(&depthPlane[idx]);
        const float4 s4 = __ldg(&signal[idx]);
        const float3 currColor = f3(s4.x, s4.y, s4.z);
        if (!p.temporalIsValid || depth == FLT_MAX_)
        {
            out[idx] = make_uint2(pack_half2(currColor.x, currColor.y), pack_half2(currColor.z, 0.0f));
            return;
        }
        float weightSum = Mitchell1D(0, 0.33f, 0.33f) * Mitchell1D(0, 0.33f, 0.33f);
        float3 reconstructed = currColor * weightSum;
        float3 firstMoment = currColor;
        float3 secondMoment = currColor * currColor;
        float closestDepth = depth;
        int cdx = 0, cdy = 0;
        int numNeighbors = 1;
#pragma unroll
        for (int i = -1; i < 2; i++)
        {
#pragma unroll
            for (int j = -1; j < 2; j++)
            {
                if (i == 0 && j == 0) continue;
                const int nx = x + i, ny = y + j;
                if (nx < 0 || ny < 0 || nx >= W || ny >= H) continue;
                const int sidx = (ly + 1 + j) * SW + lx + 1 + i;
                const float4 c4 = s_c[sidx];
                const float3 neighborColor = f3(c4.x, c4.y, c4.z);
                float weight = Mitchell1D((float)i, 0.33f, 0.33f) * Mitchell1D((float)j, 0.33f, 0.33f);
                weight *= c4.w;
                reconstructed += neighborColor * weight;
                weightSum += weight;
                firstMoment += neighborColor;
                secondMoment += neighborColor * neighborColor;
                const float neighborDepth = s_d[sidx];
                if (neighborDepth < closestDepth) { closestDepth = neighborDepth; cdx = i; cdy = j; }
                numNeighbors += 1;
            }
        }
        reconstructed = reconstructed / fmaxf(weightSum, 1e-5f);
        const float2 motionVec = unpack_snorm16x2(__ldg(&motionEmissive[(size_t)(y + cdy) * W + (x + cdx)].x));
        const float2 renderDim = f2((float)W, (float)H);
        const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / renderDim;
        const float2 prevUV = currUV - motionVec;
        if (prevUV.x < 0.0f || prevUV.y < 0.0f || prevUV.x > 1.0f || prevUV.y > 1.0f)
        {
            out[idx] = make_uint2(pack_half2(reconstructed.x, reconstructed.y), pack_half2(reconstructed.z, 0.0f));
            return;
        }
        const float3 history = SampleTextureCatmullRom(prevOut, W, H, prevUV, renderDim);
        const float3 mean = firstMoment / (float)numNeighbors;
        float3 std = abs3(secondMoment - (firstMoment * firstMoment) / (float)numNeighbors);
        std = std / ((float)numNeighbors - 1.0f);
        std = sqrt3(std);
        const float3 clippedHistory = ClipAABB(mean - std, mean + std, history);
        const float currWeight = saturate(p.blendWeight * (1.0f / (1.0f + Math::Luminance(reconstructed))));
        const float histWeight = saturate((1.0f - p.blendWeight) * (1.0f / (1.0f + Math::Luminance(clippedHistory))));
        float3 result = (currWeight * reconstructed + histWeight * clippedHistory) / (currWeight + histWeight);
        result = isnan3(result) ? reconstructed : result;
        out[idx] = make_uint2(pack_half2(result.x, result.y), pack_half2(result.z, 0.0f));
    }

    PostParams make_params(const zr_frame_constants& fc)
    {
        PostParams p;
        p.W = fc.RenderWidth;
        p.H = fc.RenderHeight;
        p.accumulate = (fc.Accumulate && fc.CameraStatic) ? 1u : 0u;
        p.numFramesAccumulated = p.accumulate ? fc.NumFramesCameraStatic : 1u;
        p.blendWeight = 0.1f;
        p.temporalIsValid = 0;
        p.rowBegin = 0; p.rowEnd = p.H;
        return p;
    }
}
} // namespace zr

// ------------------------------------------------------------------------------------------------
// Host-side pass objects: same verbs as the reference's structs
// ------------------------------------------------------------------------------------------------
struct zr_compositing_pass
{
    // Compositing (Compositing/Compositing.h): owns the LIGHT_ACCUM image (RGBA32F)
    uint32_t width = 0, height = 0;
    struct Sized
    {
        zr::Planes planes{ "zr_compositing_pass" };
        float4* d_composited = nullptr;     // output of compositing (fused with the firefly filter when it is on); never cleared
    } sz;
    zr_compositing_params params{ 1, 1, 1 };
    zr::StripRows strip{ "zr_compositing_pass" };
    zr::Sky::LutView sky{ nullptr, 0, 0 };     // zr_compositing_pass_set_sky; not owned

    zr_status Setup() { return ZR_OK; }
    zr_status OnWindowResized(uint32_t w, uint32_t h)
    {
        Sized next;
        ZR_TRY(next.planes.Alloc(next.d_composited, (size_t)w * h, false));
        sz = std::move(next);
        width = w; height = h;
        strip.ForgetRows();
        return ZR_OK;
    }
    zr_status Render(const zr_frame_inputs* in, const void* d_direct, const void* d_indirect, cudaStream_t stream)
    {
        using namespace zr;
        if (!in || !in->curr.d_core || !in->curr.d_depth)
        {
            set_error("zr_compositing_pass_render: missing G-buffer");
            return ZR_ERR_INVALID_ARG;
        }
        const zr_status st = check_frame_size("zr_compositing_pass", in->frame, width, height);
        if (st != ZR_OK) return st;
        PostParams p = make_params(in->frame);
        const float4* direct = params.emissive_di ? (const float4*)d_direct : nullptr;
        const float4* indirect = params.indirect ? (const float4*)d_indirect : nullptr;
        p.rowBegin = strip.rowBegin; p.rowEnd = strip.ClampedRowEnd(height);
        const bool withSky = sky.texels != nullptr;
        SkyArgs skyArgs;
        skyArgs.lut = sky;
        skyArgs.emissiveDI = params.emissive_di;
        skyArgs.fc = in->frame;
        if (params.firefly_filter)
        {
            const dim3 tgrid((width + FF_TW - 1) / FF_TW, (p.rowEnd - p.rowBegin + FF_TH - 1) / FF_TH);
            ZR_PROF("k_firefly", stream);
            (withSky ? k_firefly_tiled<true> : k_firefly_tiled<false>)<<<tgrid, FF_TW * FF_TH, 0, stream>>>((const uint4*)in->curr.d_core,
                (const float*)in->curr.d_depth, direct, indirect, sz.d_composited, p, skyArgs);
            ZR_LAUNCH_CHECK();
        }
        else
        {
            ZR_PROF("k_compositing", stream);
            const dim3 grid((width + 31) / 32, (p.rowEnd - p.rowBegin + 7) / 8);
            (withSky ? k_compositing<true> : k_compositing<false>)<<<grid, 256, 0, stream>>>((const uint4*)in->curr.d_core, direct, indirect,
                sz.d_composited, p, skyArgs);
            ZR_LAUNCH_CHECK();
        }
        return ZR_OK;
    }
};

struct zr_taa_pass
{
    // TAA (TAA/TAA.h): two RGBA16F images, ping-ponged every Render (TAA.cpp:99-104)
    uint32_t width = 0, height = 0;
    struct Sized
    {
        zr::Planes planes{ "zr_taa_pass" };
        uint2* d_tex[2] = { nullptr, nullptr };
    } sz;
    int outIdx = 0;
    bool isTemporalTexValid = false;
    float blendWeight = 0.1f;       // DefaultParamVals::BlendWeight
    zr::StripRows strip{ "zr_taa_pass" };

    zr_status Setup() { return ZR_OK; }
    zr_status OnWindowResized(uint32_t w, uint32_t h)
    {
        Sized next;
        for (int i = 0; i < 2; i++) ZR_TRY(next.planes.Alloc(next.d_tex[i], (size_t)w * h));
        ZR_TRY(next.planes.Clear());
        sz = std::move(next);
        width = w; height = h;
        strip.ForgetRows();
        isTemporalTexValid = false;
        return ZR_OK;
    }
    zr_status Render(const zr_frame_inputs* in, const void* d_signal, cudaStream_t stream)
    {
        using namespace zr;
        if (!in || !in->curr.d_depth || !in->curr.d_motion_emissive || !d_signal)
        {
            set_error("zr_taa_pass_render: missing input");
            return ZR_ERR_INVALID_ARG;
        }
        const zr_status st = check_frame_size("zr_taa_pass", in->frame, width, height);
        if (st != ZR_OK) return st;
        PostParams p = make_params(in->frame);
        p.blendWeight = blendWeight;
        p.temporalIsValid = isTemporalTexValid ? 1u : 0u;
        p.rowBegin = strip.rowBegin; p.rowEnd = strip.ClampedRowEnd(height);
        dim3 grid((width + 31) / 32, (p.rowEnd - p.rowBegin + 7) / 8);
        outIdx ^= 1;
        ZR_PROF("k_taa", stream);
        k_taa<<<grid, 256, 0, stream>>>((const float*)in->curr.d_depth, (const uint2*)in->curr.d_motion_emissive,
            (const float4*)d_signal, sz.d_tex[outIdx ^ 1], sz.d_tex[outIdx], p);
        ZR_LAUNCH_CHECK();
        isTemporalTexValid = true;
        return ZR_OK;
    }
};

extern "C"
{
    zr_status zr_compositing_pass_create(uint32_t width, uint32_t height, zr_compositing_pass** out) { return zr::CreatePass("zr_compositing_pass", width, height, out); }
    zr_status zr_compositing_pass_resize(zr_compositing_pass* p, uint32_t width, uint32_t height) { return zr::ResizePass("zr_compositing_pass", p, width, height); }
    zr_status zr_compositing_pass_set_params(zr_compositing_pass* p, const zr_compositing_params* params)
    {
        if (!p || !params) return ZR_ERR_INVALID_ARG;
        p->params = *params;
        return ZR_OK;
    }
    zr_status zr_compositing_pass_set_sky(zr_compositing_pass* p, const zr_image2d* lut)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return zr::Sky::ViewOf("zr_compositing_pass_set_sky", lut, p->sky);
    }
    zr_status zr_compositing_pass_render(zr_compositing_pass* p, const zr_frame_inputs* in, const void* d_direct,
        const void* d_indirect, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, d_direct, d_indirect, (cudaStream_t)stream);
    }
    zr_status zr_compositing_pass_set_rows(zr_compositing_pass* p, uint32_t y0, uint32_t y1) { return p ? p->strip.SetRows(y0, y1, p->height) : ZR_ERR_INVALID_ARG; }
    zr_status zr_compositing_pass_get_output(zr_compositing_pass* p, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        *out = zr_image2d{ p->sz.d_composited, p->width, p->height, p->width * 16u, 16u };
        return ZR_OK;
    }
    void zr_compositing_pass_destroy(zr_compositing_pass* p) { delete p; }

    zr_status zr_taa_pass_create(uint32_t width, uint32_t height, zr_taa_pass** out) { return zr::CreatePass("zr_taa_pass", width, height, out); }
    zr_status zr_taa_pass_resize(zr_taa_pass* p, uint32_t width, uint32_t height) { return zr::ResizePass("zr_taa_pass", p, width, height); }
    zr_status zr_taa_pass_set_rows(zr_taa_pass* p, uint32_t y0, uint32_t y1) { return p ? p->strip.SetRows(y0, y1, p->height) : ZR_ERR_INVALID_ARG; }
    zr_status zr_taa_pass_set_blend_weight(zr_taa_pass* p, float w)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        p->blendWeight = w;
        return ZR_OK;
    }
    zr_status zr_taa_pass_render(zr_taa_pass* p, const zr_frame_inputs* in, const void* d_signal, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, d_signal, (cudaStream_t)stream);
    }
    zr_status zr_taa_pass_get_output(zr_taa_pass* p, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        *out = zr_image2d{ p->sz.d_tex[p->outIdx], p->width, p->height, p->width * 8u, 8u };
        return ZR_OK;
    }
    void zr_taa_pass_destroy(zr_taa_pass* p) { delete p; }
}
