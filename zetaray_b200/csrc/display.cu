// display.cu -- post-processing after TAA: histogram auto exposure and the tone-mapped sRGB display image.
//
// Replaces AutoExposure/AutoExposure_Histogram.hlsl, AutoExposure_WeightedAvg.hlsl (SKIP_OUTSIDE_PERCENTILE_RANGE 0) and the
// default path of Display/Display.hlsl with Tonemap.hlsli, and their host passes (AutoExposure.cpp:100-140, Display.cpp). The
// oracle's restatement is oracle/orc_display.cpp; DESIGN 6 lists where these kernels deliberately differ from the reference.
//
//   k_lum_histogram   owned rows of the composited signal (16 B/px read) -> 256 luminance bins; a persistent grid of two blocks
//                     per SM, warp aggregation with __match_any_sync and one global atomic per non-empty bin per block (a block
//                     per 16 x 16 tile, as the reference dispatches it, would issue ~2 M atomics on 256 addresses at 1080p)
//   k_exposure        one block: weighted mean of bins 1..255 in a fixed pairwise order, inverse mapping, temporal adaptation,
//                     EV100 exposure -> float2 {exposure, adapted luminance}; clears the bins for the next frame
//   k_display         TAA output (8 B/px) x exposure -> tone mapper -> saturate -> sRGB OETF -> RGBA8 (4 B/px)
//   k_display_view    a G-buffer debug view (Display.hlsl:79-170) in place of k_display
//   k_pick_mask       picked instance k's triangles -> bit k of a per-pixel mask (DrawPicked.hlsl), a warp per triangle
//   k_outline         the mask's Sobel outline over the displayed image (Sobel.hlsl:27-105)
#include <cmath>
#include "zr_common.cuh"
#include "zr_pixel.cuh"
#include "zr_planes.h"
#include "zr_schedule.h"

namespace zr
{
namespace
{
    constexpr int HIST_BINS = 256;              // HIST_BIN_COUNT, AutoExposure_Common.h
    constexpr int HIST_THREADS = 512;
    constexpr int HIST_UNROLL = 4;              // independent 16-byte loads in flight per thread
    constexpr uint32_t LUT_DIM = 48;            // Tony McMapface, Tonemap.hlsli:16

    struct LumMap { float minLum, lumRange, lumMapExp; };

    // CalculateeBin (AutoExposure_Histogram.hlsl:22-40). The reference reads the RGBA32F signal through Texture2D<half4>, so every
    // channel is rounded to binary16 first. NaN luminance fails the EPS test and saturates to 0: bin 1.
    ZR_D uint32_t LumBin(float4 c, const LumMap& m)
    {
        const float3 rgb = f3(zr_f16_to_f32(zr_f32_to_f16(c.x)), zr_f16_to_f32(zr_f32_to_f16(c.y)), zr_f16_to_f32(zr_f32_to_f16(c.z)));
        const float lum = Math::Luminance(rgb);
        if (lum <= 1e-4f)
            return 0;
        const float t = zr_powf(saturate((lum - m.minLum) / m.lumRange), m.lumMapExp);
        const uint32_t bin = (uint32_t)(t * (float)(HIST_BINS - 2)) + 1u;
        return bin < HIST_BINS - 1 ? bin : HIST_BINS - 1;
    }

    // Pixels [begin, end) of the signal (the pass's rows). Every block walks the range in strides of HIST_THREADS * HIST_UNROLL
    // pixels; the loop bounds are uniform over the block, so every lane reaches __match_any_sync (out-of-range lanes carry no bin).
    __global__ void __launch_bounds__(HIST_THREADS, 2) k_lum_histogram(const float4* __restrict__ signal, uint32_t* __restrict__ hist,
        size_t begin, size_t end, LumMap m)
    {
        __shared__ uint32_t s_hist[HIST_BINS];
        for (int b = threadIdx.x; b < HIST_BINS; b += HIST_THREADS)
            s_hist[b] = 0;
        __syncthreads();
        const uint32_t lane = threadIdx.x & 31;
        const size_t chunk = (size_t)HIST_THREADS * HIST_UNROLL;
        for (size_t base = begin + blockIdx.x * chunk; base < end; base += (size_t)gridDim.x * chunk)
        {
            float4 v[HIST_UNROLL];
#pragma unroll
            for (int k = 0; k < HIST_UNROLL; k++)
            {
                const size_t i = base + (size_t)k * HIST_THREADS + threadIdx.x;
                v[k] = i < end ? __ldg(&signal[i]) : f4(0, 0, 0, 0);
            }
#pragma unroll
            for (int k = 0; k < HIST_UNROLL; k++)
            {
                const size_t i = base + (size_t)k * HIST_THREADS + threadIdx.x;
                const uint32_t bin = i < end ? LumBin(v[k], m) : 0xffffffffu;
                const uint32_t peers = __match_any_sync(0xffffffffu, bin);
                if (bin != 0xffffffffu && lane == (uint32_t)(__ffs(peers) - 1))
                    atomicAdd(&s_hist[bin], (uint32_t)__popc(peers));
            }
        }
        __syncthreads();
        for (int b = threadIdx.x; b < HIST_BINS; b += HIST_THREADS)
            if (s_hist[b])
                atomicAdd(&hist[b], s_hist[b]);
    }

    // ComputeAutoExposure (AutoExposure_WeightedAvg.hlsl:20-28)
    ZR_D float ComputeAutoExposure(float avgLum)
    {
        const float S = 100.0f, K = 12.5f, q = 0.65f;
        const float EV100 = zr_log2f((avgLum * S) / K);
        const float luminanceMax = (78.0f / (q * S)) * zr_powf(2.0f, EV100);
        return 1.0f / luminanceMax;
    }

    // AutoExposure_WeightedAvg.hlsl:42-110. The reference sums with WaveActiveSum, whose order is unspecified; here the sum is a
    // pairwise tree over the 256 bin values (s[i] += s[i + h] for h = 128, 64, ..., 1), which the oracle restates exactly.
    // numPixels is the whole frame's RenderWidth * RenderHeight, also in sharded frames (the bins then hold every rank's counts).
    __global__ void __launch_bounds__(HIST_BINS) k_exposure(uint32_t* __restrict__ hist, float2* __restrict__ state, uint32_t numPixels,
        LumMap m, float adaptationRate, float dt)
    {
        __shared__ float s_sum[HIST_BINS];
        __shared__ uint32_t s_bin0;
        const uint32_t i = threadIdx.x;
        const uint32_t binSize = hist[i];
        if (i == 0)
            s_bin0 = binSize;
        s_sum[i] = i == 0 ? 0.0f : ((float)binSize * ((float)(i - 1) + 0.5f)) / (float)HIST_BINS;
        __syncthreads();
        hist[i] = 0;        // the next frame's histogram starts empty (no separate clear)
        for (uint32_t h = HIST_BINS / 2; h > 0; h >>= 1)
        {
            if (i < h)
                s_sum[i] = s_sum[i] + s_sum[i + h];
            __syncthreads();
        }
        if (i != 0)
            return;
        const uint32_t numSamples = numPixels - s_bin0;
        const float mean = s_sum[0] / (float)(numSamples > 1u ? numSamples : 1u);
        float result = zr_powf(mean, 1.0f / m.lumMapExp);
        result = result * m.lumRange + m.minLum;
        const float prev = state->y;
        if (prev < 1e8f)
            result = prev + (result - prev) * (1.0f - zr_expf(-dt * 1000.0f * adaptationRate));
        *state = make_float2(ComputeAutoExposure(result), result);
    }

    // ---- Tonemap.hlsli ----
    // R9G9B9E5_SHAREDEXP: 9-bit mantissas (R low), 5-bit shared exponent, value = m * 2^(e - 15 - 9)
    ZR_D float3 DecodeRGB9E5(uint32_t v)
    {
        const float scale = __uint_as_float(((v >> 27) + 127u - 24u) << 23);
        return f3((float)(v & 0x1ffu) * scale, (float)((v >> 9) & 0x1ffu) * scale, (float)((v >> 18) & 0x1ffu) * scale);
    }
    ZR_D float3 LutTexel(const uint32_t* __restrict__ lut, uint32_t x, uint32_t y, uint32_t z)
    {
        return DecodeRGB9E5(__ldg(&lut[(z * LUT_DIM + y) * LUT_DIM + x]));
    }

    // tony_mc_mapface (Tonemap.hlsli:10-22): the LUT stays packed (48^3 x 4 B, L2-resident) and is filtered here with float
    // weights (the sampler's are 8-bit fixed point), x then y then z, at the linear sampler's texel-centre mapping with clamp
    // addressing. The coordinate is clamped before its floor, which also maps NaN to texel 0.
    ZR_D float3 TonyMcMapface(float3 stimulus, const uint32_t* __restrict__ lut)
    {
        const float3 encoded = stimulus / (stimulus + 1.0f);
        const float3 uv = encoded * ((float)(LUT_DIM - 1) / (float)LUT_DIM) + 0.5f / (float)LUT_DIM;
        const float3 t = uv * (float)LUT_DIM - 0.5f;
        const float hi = (float)(LUT_DIM - 1);
        const float tx = fminf(fmaxf(t.x, 0.0f), hi), ty = fminf(fmaxf(t.y, 0.0f), hi), tz = fminf(fmaxf(t.z, 0.0f), hi);
        const uint32_t x0 = (uint32_t)floorf(tx), y0 = (uint32_t)floorf(ty), z0 = (uint32_t)floorf(tz);
        const uint32_t x1 = min(x0 + 1, LUT_DIM - 1), y1 = min(y0 + 1, LUT_DIM - 1), z1 = min(z0 + 1, LUT_DIM - 1);
        const float fx = tx - (float)x0, fy = ty - (float)y0, fz = tz - (float)z0;
        const float3 c00 = Math::Lerp(LutTexel(lut, x0, y0, z0), LutTexel(lut, x1, y0, z0), fx);
        const float3 c10 = Math::Lerp(LutTexel(lut, x0, y1, z0), LutTexel(lut, x1, y1, z0), fx);
        const float3 c01 = Math::Lerp(LutTexel(lut, x0, y0, z1), LutTexel(lut, x1, y0, z1), fx);
        const float3 c11 = Math::Lerp(LutTexel(lut, x0, y1, z1), LutTexel(lut, x1, y1, z1), fx);
        return Math::Lerp(Math::Lerp(c00, c10, fy), Math::Lerp(c01, c11, fy), fz);
    }

    // HLSL mul(row, M) with M filled row by row: out_j = sum_i v_i M[i][j]
    ZR_D float3 MulRow(float3 v, const float (&M)[3][3])
    {
        return f3(fmaf(v.z, M[2][0], fmaf(v.y, M[1][0], v.x * M[0][0])),
                  fmaf(v.z, M[2][1], fmaf(v.y, M[1][1], v.x * M[0][1])),
                  fmaf(v.z, M[2][2], fmaf(v.y, M[1][2], v.x * M[0][2])));
    }
    ZR_D float3 pow3(float3 v, float e) { return f3(zr_powf(v.x, e), zr_powf(v.y, e), zr_powf(v.z, e)); }

    ZR_D float AgxContrast(float x)
    {
        const float x2 = x * x, x4 = x2 * x2, x6 = x4 * x2;
        return -17.86f * x6 * x + 78.01f * x6 - 126.7f * x4 * x + 92.06f * x4 - 28.72f * x2 * x + 4.361f * x2 - 0.1718f * x + 0.002857f;
    }
    ZR_D float AgxLog(float v)
    {
        const float minEv = -12.47393f, maxEv = 4.026069f;
        return (fminf(fmaxf(zr_log2f(v), minEv), maxEv) - minEv) / (maxEv - minEv);
    }
    ZR_D float3 AgxInset(float3 v)
    {
        const float M[3][3] = { { 0.842479062253094f, 0.0423282422610123f, 0.0423756549057051f },
                                { 0.0784335999999992f, 0.878468636469772f, 0.0784336f },
                                { 0.0792237451477643f, 0.0791661274605434f, 0.879142973793104f } };
        v = MulRow(v, M);
        return f3(AgxContrast(AgxLog(v.x)), AgxContrast(AgxLog(v.y)), AgxContrast(AgxLog(v.z)));
    }
    ZR_D float3 AgxEotf(float3 v)
    {
        const float M[3][3] = { { 1.19687900512017f, -0.0528968517574562f, -0.0529716355144438f },
                                { -0.0980208811401368f, 1.15190312990417f, -0.0980434501171241f },
                                { -0.0990297440797205f, -0.0989611768448433f, 1.15107367264116f } };
        return pow3(MulRow(v, M), 2.2f);
    }
    ZR_D float3 AgxLook(float3 v, float3 slope, float e, float saturation)
    {
        const float luma = Math::Luminance(v);
        v = pow3(v * slope + 0.0f, e);
        return f3(luma + saturation * (v.x - luma), luma + saturation * (v.y - luma), luma + saturation * (v.z - luma));
    }

    ZR_D float SrgbOetf(float v) { return v <= 0.0031308f ? 12.92f * v : 1.055f * zr_powf(v, 1.0f / 2.4f) - 0.055f; }

    // saturated linear RGB -> the R8G8B8A8_UNORM_SRGB store's RGB bytes
    ZR_D uint32_t EncodeSrgb8(float3 c)
    {
        return Math::FloatToUNorm8(SrgbOetf(c.x)) | Math::FloatToUNorm8(SrgbOetf(c.y)) << 8 | Math::FloatToUNorm8(SrgbOetf(c.z)) << 16;
    }

    struct DisplayArgs { uint32_t tonemapper, autoExposure; float saturation, agxExp; };

    ZR_D float3 Tonemap(float3 c, const DisplayArgs& a, const uint32_t* __restrict__ lut)
    {
        switch (a.tonemapper)
        {
        case ZR_TONEMAPPER_NEUTRAL:
        {
            c = TonyMcMapface(c, lut);
            return Math::Lerp(f3(Math::Luminance(c)), c, a.saturation);
        }
        case ZR_TONEMAPPER_AGX_DEFAULT: return AgxEotf(AgxInset(c));
        case ZR_TONEMAPPER_AGX_GOLDEN: return AgxEotf(AgxLook(AgxInset(c), f3(1.0f, 0.9f, 0.5f), 0.8f, 0.8f));
        case ZR_TONEMAPPER_AGX_PUNCHY: return AgxEotf(AgxLook(AgxInset(c), f3(1.0f), 1.35f, 1.4f));
        case ZR_TONEMAPPER_AGX_CUSTOM: return AgxEotf(AgxLook(AgxInset(c), f3(1.0f), a.agxExp, a.saturation));
        default: return c;
        }
    }

    // Display.hlsl:42-77 (DisplayOption::DEFAULT) and the R8G8B8A8_UNORM_SRGB store, pixels [begin, end)
    __global__ void __launch_bounds__(256) k_display(const uint2* __restrict__ in, const float2* __restrict__ exposure,
        const uint32_t* __restrict__ lut, uint32_t* __restrict__ out, size_t begin, size_t end, DisplayArgs a)
    {
        const size_t i = begin + (size_t)blockIdx.x * 256 + threadIdx.x;
        if (i >= end)
            return;
        const uint2 p = __ldg(&in[i]);
        float3 c = f3(half_lo(p.x), half_hi(p.x), half_lo(p.y));
        if (a.autoExposure)
            c = c * __ldg(&exposure->x);
        c = saturate(Tonemap(c, a, lut));
        out[i] = EncodeSrgb8(c) | 0xff000000u;
    }

    // Display.hlsl:53-54, 79-170: one G-buffer channel in place of the tone-mapped signal, pixels [begin, end). The reference
    // tone-maps first and then overwrites the result, so a view reads no signal, exposure or LUT.
    __global__ void __launch_bounds__(256) k_display_view(const uint4* __restrict__ core, const uint2* __restrict__ me,
        const uint2* __restrict__ coat, uint32_t* __restrict__ out, size_t begin, size_t end, uint32_t view, float roughnessTh,
        float cameraNear)
    {
        const size_t i = begin + (size_t)blockIdx.x * 256 + threadIdx.x;
        if (i >= end)
            return;
        const uint4 c = ld128(&core[i]);
        const float z = asfloat(c.x);
        if (z == FLT_MAX_)
        {
            out[i] = 0u;        // background: (0, 0, 0, 0), alpha included
            return;
        }
        const GFlags fl = DecodeFlags(c.w & 0xff);
        const float roughness = Math::UNorm8ToFloat((c.w >> 8) & 0xff);
        const float3 baseColor = Math::UnpackRGB8(c.z & 0xffffff);
        float3 d = f3(0.0f);
        switch (view)
        {
        case ZR_DISPLAY_VIEW_BASE_COLOR: d = baseColor; break;
        case ZR_DISPLAY_VIEW_NORMAL: d = Math::DecodeUnitVector(Math::DecodeUNorm2(c.y)) * 0.5f + 0.5f; break;
        case ZR_DISPLAY_VIEW_METALNESS_ROUGHNESS: d = f3(fl.metallic ? 1.0f : 0.0f, roughness, 0.0f); break;
        case ZR_DISPLAY_VIEW_COAT_WEIGHT:
        case ZR_DISPLAY_VIEW_COAT_COLOR:
            if (fl.coated)
            {
                // GBuffer::UnpackCoat, as LoadPixel (zr_pixel.cuh) reads the coat plane
                const uint2 cc = __ldg(&coat[i]);
                const uint32_t px = cc.x & 0xffff, py = cc.x >> 16;
                d = view == ZR_DISPLAY_VIEW_COAT_WEIGHT ? f3(Math::UNorm8ToFloat((py >> 8) & 0xff)) : Math::UnpackRGB8(px | ((py & 0xff) << 16));
            }
            break;
        case ZR_DISPLAY_VIEW_ROUGHNESS_TH: d = roughness >= roughnessTh ? f3(0.26f, 0.014f, 0.021f) : f3(0.0f); break;
        case ZR_DISPLAY_VIEW_EMISSIVE: d = fl.emissive ? unpack_r11g11b10(__ldg(&me[i].y)) : baseColor * 0.005f; break;
        case ZR_DISPLAY_VIEW_TRANSMISSION: d = f3(fl.transmissive ? 1.0f : 0.0f, fl.transmissive ? 0.0f : 1.0f, 0.0f); break;
        case ZR_DISPLAY_VIEW_DEPTH: d = f3(cameraNear / z); break;
        default: break;
        }
        out[i] = EncodeSrgb8(saturate(d)) | 0xff000000u;
    }

    // ---- picked-instance outline (Display.cpp:293-400, DrawPicked.hlsl, Sobel.hlsl); DESIGN 6b states the rasteriser's rules ----
    // The picked instances and the running sum of their triangle counts: warp w rasterises triangle w - triEnd[k - 1] of inst[k].
    struct PickList { uint32_t n; uint32_t inst[ZR_DISPLAY_MAX_PICKED]; uint32_t triEnd[ZR_DISPLAY_MAX_PICKED]; };

    // Clips a view-space triangle to z >= near, the one clip plane of a reverse-Z projection with an infinite far plane: 0, 3 or 4
    // vertices of a convex polygon, in order. A crossing point is computed from the edge's inside vertex, so the two triangles
    // that share an edge clip it to the same point.
    ZR_D int ClipNear(const float3 (&v)[3], float nearZ, float3 (&out)[4])
    {
        int n = 0;
        for (int e = 0; e < 3; e++)
        {
            const float3 a = v[e], b = v[e == 2 ? 0 : e + 1];
            const bool ina = a.z >= nearZ, inb = b.z >= nearZ;
            if (ina)
                out[n++] = a;
            if (ina != inb)
            {
                const float3 p = ina ? a : b, q = ina ? b : a;
                const float t = (nearZ - p.z) / (q.z - p.z);
                out[n++] = f3(p.x + t * (q.x - p.x), p.y + t * (q.y - p.y), nearZ);
            }
        }
        return n;
    }

    // The inverse of k_gbuffer's camera-ray mapping (Math::NDCFromUV, jitter included): a view-space point on the ray of pixel
    // (x, y) lands on (x + 0.5, y + 0.5).
    ZR_D float2 ProjectToPixel(float3 p, const zr_frame_constants& fc)
    {
        const float2 ndc = f2(p.x / p.z / fc.TanHalfFOV / fc.AspectRatio, p.y / p.z / fc.TanHalfFOV);
        const float2 uv = Math::UVFromNDC(ndc);
        return f2(uv.x * (float)fc.RenderWidth - fc.CurrCameraJitter[0], uv.y * (float)fc.RenderHeight - fc.CurrCameraJitter[1]);
    }

    // Edge function of a -> b at p, evaluated with the endpoints in one fixed order, so the two triangles that share an edge get
    // exactly opposite values
    ZR_D float EdgeFn(float2 a, float2 b, float2 p)
    {
        const bool swap = b.y < a.y || (b.y == a.y && b.x < a.x);
        const float2 s = swap ? b : a, t = swap ? a : b;
        const float e = (t.x - s.x) * (p.y - s.y) - (t.y - s.y) * (p.x - s.x);
        return swap ? -e : e;
    }
    // Inside is E > 0 on every edge of an oriented triangle (rows grow downwards). A centre on an edge is inside when the edge is
    // a left edge (b.y < a.y) or a top edge (horizontal, b.x > a.x): the D3D top-left rule.
    ZR_D bool EdgeIn(float2 a, float2 b, float2 p)
    {
        const float e = EdgeFn(a, b, p);
        return e > 0.0f || (e == 0.0f && (b.y < a.y || (b.y == a.y && b.x > a.x)));
    }
    // Either winding: no back-face culling (the DrawPicked PSO, Display.cpp:452-470). A degenerate triangle covers nothing.
    ZR_D bool InTriangle(float2 a, float2 b, float2 c, float2 p)
    {
        const float area = EdgeFn(a, b, c);
        if (area == 0.0f)
            return false;
        if (area < 0.0f) { const float2 t = b; b = c; c = t; }
        return EdgeIn(a, b, p) && EdgeIn(b, c, p) && EdgeIn(c, a, p);
    }

    // Rows [y0, y1) of the mask; no depth test, so hidden parts of an instance are marked too
    __global__ void __launch_bounds__(256) k_pick_mask(SceneDev sc, zr_frame_constants fc, PickList pl, uint32_t* __restrict__ mask,
        uint32_t y0, uint32_t y1)
    {
        const uint32_t w = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
        if (w >= pl.triEnd[pl.n - 1])
            return;
        uint32_t k = 0;
        while (w >= pl.triEnd[k])
            k++;
        const uint32_t prim = w - (k ? pl.triEnd[k - 1] : 0u);
        const zr_mesh_instance md = LoadInstance(sc, pl.inst[k]);
        const float4 q = normalize(Math::DecodeNormalized4(md.Rotation));
        const float3 scale = h3(md.Scale);
        const float3 translation = f3(md.Translation[0], md.Translation[1], md.Translation[2]);
        float3 v[3];
        for (int j = 0; j < 3; j++)
        {
            const VertexD V = LoadVertex(sc, __ldg(&sc.indices[prim * 3 + md.BaseIdxOffset + j]) + md.BaseVtxOffset);
            v[j] = Math::mul3x4(fc.CurrView, Math::TransformTRS(V.pos, translation, q, scale));
        }
        float3 c[4];
        const int n = ClipNear(v, fc.CameraNear, c);
        if (n < 3)
            return;
        float2 s[4];
        float x0 = FLT_MAX_, x1 = -FLT_MAX_, ya = FLT_MAX_, yb = -FLT_MAX_;
        for (int j = 0; j < n; j++)
        {
            s[j] = ProjectToPixel(c[j], fc);
            x0 = fminf(x0, s[j].x); x1 = fmaxf(x1, s[j].x); ya = fminf(ya, s[j].y); yb = fmaxf(yb, s[j].y);
        }
        // pixels whose centre can lie inside, clamped to the frame's columns and the rows asked for
        const float xs = fmaxf(ceilf(x0 - 0.5f), 0.0f), xe = fminf(floorf(x1 - 0.5f), (float)fc.RenderWidth - 1.0f);
        const float ys = fmaxf(ceilf(ya - 0.5f), (float)y0), ye = fminf(floorf(yb - 0.5f), (float)y1 - 1.0f);
        if (!(xs <= xe && ys <= ye))
            return;
        const uint32_t bx = (uint32_t)xs, by = (uint32_t)ys, bw = (uint32_t)xe - bx + 1, bh = (uint32_t)ye - by + 1;
        const uint32_t bit = 1u << k;
        for (uint32_t j = lane; j < bw * bh; j += 32)
        {
            const uint32_t x = bx + j % bw, y = by + j / bw;
            const float2 p = f2((float)x + 0.5f, (float)y + 0.5f);
            if (InTriangle(s[0], s[1], s[2], p) || (n == 4 && InTriangle(s[0], s[2], s[3], p)))
                atomicOr(&mask[(size_t)y * fc.RenderWidth + x], bit);
        }
    }

    // Sobel.hlsl, for each bit k of the mask: a pixel with bit k somewhere in its in-frame 3 x 3 neighbourhood (CheckNeighborHood)
    // and a non-zero Sobel gradient of bit k (taps outside the frame read 0) takes the outline colour. The gradients are small
    // integers, exact in float, and Luminance(sqrt(gx^2 + gy^2)) > 0 exactly when one of them is non-zero. Pixels [begin, end).
    __global__ void __launch_bounds__(256) k_outline(const uint32_t* __restrict__ mask, uint32_t* __restrict__ out, uint32_t W,
        uint32_t H, size_t begin, size_t end)
    {
        const size_t i = begin + (size_t)blockIdx.x * 256 + threadIdx.x;
        if (i >= end)
            return;
        const int x = (int)(i % W), y = (int)(i / W);
        uint32_t m[3][3];
        uint32_t any = 0;
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 3; c++)
            {
                const int xx = x - 1 + c, yy = y - 1 + r;
                m[r][c] = xx >= 0 && xx < (int)W && yy >= 0 && yy < (int)H ? __ldg(&mask[(size_t)yy * W + xx]) : 0u;
                any |= m[r][c];
            }
        for (uint32_t b = any; b; b &= b - 1)
        {
            const uint32_t bit = b & (0u - b);
            int t[3][3];
            for (int r = 0; r < 3; r++)
                for (int c = 0; c < 3; c++)
                    t[r][c] = (m[r][c] & bit) ? 1 : 0;
            const int gx = -t[0][0] - 2 * t[1][0] - t[2][0] + t[0][2] + 2 * t[1][2] + t[2][2];
            const int gy = t[0][0] + 2 * t[0][1] + t[0][2] - t[2][0] - 2 * t[2][1] - t[2][2];
            if (gx != 0 || gy != 0)
            {
                // the reference writes this linear colour into its _SRGB back buffer
                out[i] = EncodeSrgb8(f3(0.913098693f, 0.332451582f, 0.048171822f)) | 0xff000000u;
                return;
            }
        }
    }

    bool is_finite(float v) { return std::isfinite(v); }
}
} // namespace zr

// ------------------------------------------------------------------------------------------------
// Host-side pass objects
// ------------------------------------------------------------------------------------------------
struct zr_auto_exposure_pass
{
    // AutoExposure (AutoExposure/AutoExposure.h): the 256-bin histogram and the 1 x 1 RG32F exposure texture (INIT_TO_ZERO)
    uint32_t width = 0, height = 0;
    struct Sized
    {
        zr::Planes planes{ "zr_auto_exposure_pass" };
        uint32_t* d_hist = nullptr;         // all zero between frames: k_exposure clears it
        float2* d_state = nullptr;          // {exposure, adapted luminance}
    } sz;
    zr_auto_exposure_params params = Defaults();
    zr::StripRows strip{ "zr_auto_exposure_pass" };
    bool hasHistory = false;                // a frame ran since create / resize / reset
    zr_reduce_u32_fn reduce = nullptr;
    void* reduceUser = nullptr;
    uint32_t maxBlocks = 0;

    static zr_auto_exposure_params Defaults() { return zr_auto_exposure_params{ 5e-3f, 4.0f, 0.5f, 1.0f }; }     // AutoExposure.h:73-80
    zr_status Setup()
    {
        int dev = 0, sms = 0;
        ZR_CUDA(cudaGetDevice(&dev));
        ZR_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        maxBlocks = 2u * (uint32_t)sms;
        return ZR_OK;
    }
    zr_status OnWindowResized(uint32_t w, uint32_t h)
    {
        Sized next;
        ZR_TRY(next.planes.Alloc(next.d_hist, zr::HIST_BINS));
        ZR_TRY(next.planes.Alloc(next.d_state, 1));
        ZR_TRY(next.planes.Clear());
        sz = std::move(next);
        width = w; height = h;
        strip.ForgetRows();
        hasHistory = false;
        return ZR_OK;
    }
    zr_status ResetTemporal()
    {
        ZR_TRY(sz.planes.Clear());
        hasHistory = false;
        return ZR_OK;
    }
    zr_status Render(const zr_frame_inputs* in, const void* d_signal, cudaStream_t stream)
    {
        using namespace zr;
        if (!in || !d_signal)
        {
            set_error("zr_auto_exposure_pass_render: missing input");
            return ZR_ERR_INVALID_ARG;
        }
        ZR_TRY(check_frame_size("zr_auto_exposure_pass", in->frame, width, height));
        const float dt = in->frame.dt;
        if (!is_finite(dt) || dt < 0.0f)
        {
            set_error("zr_auto_exposure_pass_render: dt must be a finite number of seconds >= 0 (got %g)", (double)dt);
            return ZR_ERR_INVALID_ARG;
        }
        if (dt == 0.0f && !hasHistory)
        {
            set_error("zr_auto_exposure_pass_render: dt == 0 on the first frame would leave the adapted luminance at 0 and the exposure infinite");
            return ZR_ERR_INVALID_ARG;
        }
        const LumMap m{ params.min_lum, params.max_lum - params.min_lum, params.lum_map_exp };
        const size_t begin = (size_t)strip.rowBegin * width, end = (size_t)strip.ClampedRowEnd(height) * width;
        const size_t chunk = (size_t)HIST_THREADS * HIST_UNROLL;
        const size_t blocksNeeded = (end - begin + chunk - 1) / chunk;
        const uint32_t blocks = (uint32_t)(blocksNeeded < maxBlocks ? blocksNeeded : maxBlocks);
        ZR_PROF("k_lum_histogram", stream);
        k_lum_histogram<<<blocks, HIST_THREADS, 0, stream>>>((const float4*)d_signal, sz.d_hist, begin, end, m);
        ZR_LAUNCH_CHECK();
        if (reduce)
            reduce(reduceUser, sz.d_hist, HIST_BINS, stream);
        ZR_PROF("k_exposure", stream);
        k_exposure<<<1, HIST_BINS, 0, stream>>>(sz.d_hist, sz.d_state, width * height, m, params.adaptation_rate, dt);
        ZR_LAUNCH_CHECK();
        hasHistory = true;
        return ZR_OK;
    }
};

struct zr_display_pass
{
    // DisplayPass (Display/Display.h): the R8G8B8A8 image it presents, its debug view and the outline of the picked instances
    uint32_t width = 0, height = 0;
    struct Sized
    {
        zr::Planes planes{ "zr_display_pass" };
        uint32_t* d_out = nullptr;
        uint32_t* d_mask = nullptr;         // bit k: picked instance k covers the pixel (rows of the frame with picks)
    } sz;
    zr::Planes lutPlanes{ "zr_display_pass" };
    uint32_t* d_lut = nullptr;              // Tony McMapface, packed R9G9B9E5; NULL until set_lut
    zr_display_params params = Defaults();
    zr::StripRows strip{ "zr_display_pass" };
    uint32_t view = ZR_DISPLAY_VIEW_DEFAULT;
    float roughnessTh = 1.0f;               // Display.cpp:73
    uint32_t picked[ZR_DISPLAY_MAX_PICKED] = {};
    uint32_t numPicked = 0;

    static zr_display_params Defaults() { return zr_display_params{ ZR_TONEMAPPER_NEUTRAL, 1u, 1.0f, 1.0f }; }     // Display.cpp:70-74
    zr_status Setup() { return ZR_OK; }
    zr_status OnWindowResized(uint32_t w, uint32_t h)
    {
        Sized next;
        ZR_TRY(next.planes.Alloc(next.d_out, (size_t)w * h));
        ZR_TRY(next.planes.Alloc(next.d_mask, (size_t)w * h));
        ZR_TRY(next.planes.Clear());
        sz = std::move(next);
        width = w; height = h;
        strip.ForgetRows();
        return ZR_OK;
    }
    zr_status SetLut(const uint32_t* h_lut, uint32_t dim)
    {
        using namespace zr;
        if (!h_lut || dim != LUT_DIM)
        {
            set_error("zr_display_pass_set_lut: expected the %u^3 R9G9B9E5 Tony McMapface LUT (got %s, dim %u)", LUT_DIM,
                h_lut ? "data" : "NULL", dim);
            return ZR_ERR_INVALID_ARG;
        }
        Planes next{ "zr_display_pass" };
        uint32_t* d = nullptr;
        const size_t n = (size_t)LUT_DIM * LUT_DIM * LUT_DIM;
        ZR_TRY(next.Alloc(d, n, false));
        ZR_CLEAR_BEGIN();       // a frame still in flight may read the old LUT
        ZR_CUDA(cudaMemcpy(d, h_lut, n * sizeof(uint32_t), cudaMemcpyHostToDevice));
        ZR_CLEAR_END();
        lutPlanes = std::move(next);
        d_lut = d;
        return ZR_OK;
    }
    zr_status Render(const zr_frame_inputs* in, const void* d_signal, const void* d_exposure, cudaStream_t stream)
    {
        using namespace zr;
        const bool defaultView = view == ZR_DISPLAY_VIEW_DEFAULT;
        if (!in || (defaultView && !d_signal))
        {
            set_error("zr_display_pass_render: missing input");
            return ZR_ERR_INVALID_ARG;
        }
        ZR_TRY(check_frame_size("zr_display_pass", in->frame, width, height));
        if (in->frame.DisplayWidth != in->frame.RenderWidth || in->frame.DisplayHeight != in->frame.RenderHeight)
        {
            set_error("zr_display_pass_render: display size %ux%u differs from the render size %ux%u (no upscaler in this build)",
                in->frame.DisplayWidth, in->frame.DisplayHeight, in->frame.RenderWidth, in->frame.RenderHeight);
            return ZR_ERR_INVALID_ARG;
        }
        if (defaultView && params.auto_exposure && !d_exposure)
        {
            set_error("zr_display_pass_render: auto exposure is on but no exposure state was given");
            return ZR_ERR_INVALID_ARG;
        }
        if (defaultView && params.tonemapper == ZR_TONEMAPPER_NEUTRAL && !d_lut)
        {
            set_error("zr_display_pass_render: the NEUTRAL tone mapper needs the Tony McMapface LUT (zr_display_pass_set_lut)");
            return ZR_ERR_INVALID_ARG;
        }
        if (!defaultView && (!in->curr.d_core || !in->curr.d_motion_emissive || !in->curr.d_coat))
        {
            set_error("zr_display_pass_render: debug view %u reads the current G-buffer, which is missing", view);
            return ZR_ERR_INVALID_ARG;
        }
        PickList pl{};
        if (numPicked)
        {
            if (!in->scene)
            {
                set_error("zr_display_pass_render: picked instances need the scene");
                return ZR_ERR_INVALID_ARG;
            }
            if (!(in->frame.CameraNear > 0.0f))
            {
                set_error("zr_display_pass_render: picked instances need CameraNear > 0 (got %g)", (double)in->frame.CameraNear);
                return ZR_ERR_INVALID_ARG;
            }
            uint32_t total = 0;
            for (uint32_t k = 0; k < numPicked; k++)
            {
                if (picked[k] >= in->scene->dev.numInstances)
                {
                    set_error("zr_display_pass_render: picked instance %u is not in the scene (%u instances)", picked[k],
                        in->scene->dev.numInstances);
                    return ZR_ERR_INVALID_ARG;
                }
                pl.inst[k] = picked[k];
                total += in->scene->hostInstances[picked[k]].numTris;
                pl.triEnd[k] = total;
            }
            pl.n = numPicked;
        }
        const uint32_t y0 = strip.rowBegin, y1 = strip.ClampedRowEnd(height);
        const size_t begin = (size_t)y0 * width, end = (size_t)y1 * width;
        const uint32_t blocks = (uint32_t)((end - begin + 255) / 256);
        if (defaultView)
        {
            const DisplayArgs a{ params.tonemapper, params.auto_exposure ? 1u : 0u, params.saturation, params.agx_exp };
            ZR_PROF("k_display", stream);
            k_display<<<blocks, 256, 0, stream>>>((const uint2*)d_signal, (const float2*)d_exposure, d_lut, sz.d_out, begin, end, a);
            ZR_LAUNCH_CHECK();
        }
        else
        {
            ZR_PROF("k_display_view", stream);
            k_display_view<<<blocks, 256, 0, stream>>>((const uint4*)in->curr.d_core, (const uint2*)in->curr.d_motion_emissive,
                (const uint2*)in->curr.d_coat, sz.d_out, begin, end, view, roughnessTh, in->frame.CameraNear);
            ZR_LAUNCH_CHECK();
        }
        if (numPicked)
        {
            // the outline of row y reads the mask rows y - 1 .. y + 1: each strip rasterises its rows and one on either side
            const uint32_t m0 = y0 ? y0 - 1 : 0u, m1 = y1 < height ? y1 + 1 : height;
            ZR_CUDA(cudaMemsetAsync(sz.d_mask + (size_t)m0 * width, 0, (size_t)(m1 - m0) * width * sizeof(uint32_t), stream));
            const uint32_t tris = pl.triEnd[numPicked - 1];
            if (tris)
            {
                ZR_PROF("k_pick_mask", stream);
                k_pick_mask<<<(uint32_t)(((uint64_t)tris * 32 + 255) / 256), 256, 0, stream>>>(in->scene->dev, in->frame, pl, sz.d_mask, m0, m1);
                ZR_LAUNCH_CHECK();
            }
            ZR_PROF("k_outline", stream);
            k_outline<<<blocks, 256, 0, stream>>>(sz.d_mask, sz.d_out, width, height, begin, end);
            ZR_LAUNCH_CHECK();
        }
        return ZR_OK;
    }
};

extern "C"
{
    zr_status zr_auto_exposure_pass_create(uint32_t width, uint32_t height, zr_auto_exposure_pass** out) { return zr::CreatePass("zr_auto_exposure_pass", width, height, out); }
    zr_status zr_auto_exposure_pass_resize(zr_auto_exposure_pass* p, uint32_t width, uint32_t height) { return zr::ResizePass("zr_auto_exposure_pass", p, width, height); }
    zr_status zr_auto_exposure_pass_reset_temporal(zr_auto_exposure_pass* p) { return zr::ResetPass(p); }
    zr_status zr_auto_exposure_pass_default_params(zr_auto_exposure_params* out) { return zr::DefaultParams<zr_auto_exposure_pass>(out); }
    zr_status zr_auto_exposure_pass_set_params(zr_auto_exposure_pass* p, const zr_auto_exposure_params* params)
    {
        if (!p || !params) return ZR_ERR_INVALID_ARG;
        const zr_auto_exposure_params& q = *params;
        if (!zr::is_finite(q.min_lum) || !zr::is_finite(q.max_lum) || !zr::is_finite(q.lum_map_exp) || !zr::is_finite(q.adaptation_rate) ||
            q.min_lum < 0.0f || q.max_lum <= q.min_lum || q.lum_map_exp <= 0.0f)
        {
            zr::set_error("zr_auto_exposure_pass_set_params: need finite values with 0 <= min_lum < max_lum and lum_map_exp > 0");
            return ZR_ERR_INVALID_ARG;
        }
        p->params = q;
        return ZR_OK;
    }
    zr_status zr_auto_exposure_pass_render(zr_auto_exposure_pass* p, const zr_frame_inputs* in, const void* d_signal, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, d_signal, (cudaStream_t)stream);
    }
    zr_status zr_auto_exposure_pass_set_rows(zr_auto_exposure_pass* p, uint32_t y0, uint32_t y1) { return p ? p->strip.SetRows(y0, y1, p->height) : ZR_ERR_INVALID_ARG; }
    zr_status zr_auto_exposure_pass_set_reduce(zr_auto_exposure_pass* p, zr_reduce_u32_fn fn, void* user)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        p->reduce = fn; p->reduceUser = user;
        return ZR_OK;
    }
    zr_status zr_auto_exposure_pass_get_output(zr_auto_exposure_pass* p, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        *out = zr_image2d{ p->sz.d_state, 1, 1, 8u, 8u };
        return ZR_OK;
    }
    void zr_auto_exposure_pass_destroy(zr_auto_exposure_pass* p) { delete p; }

    zr_status zr_display_pass_create(uint32_t width, uint32_t height, zr_display_pass** out) { return zr::CreatePass("zr_display_pass", width, height, out); }
    zr_status zr_display_pass_resize(zr_display_pass* p, uint32_t width, uint32_t height) { return zr::ResizePass("zr_display_pass", p, width, height); }
    zr_status zr_display_pass_default_params(zr_display_params* out) { return zr::DefaultParams<zr_display_pass>(out); }
    zr_status zr_display_pass_set_params(zr_display_pass* p, const zr_display_params* params)
    {
        if (!p || !params) return ZR_ERR_INVALID_ARG;
        if (params->tonemapper > ZR_TONEMAPPER_AGX_CUSTOM || !zr::is_finite(params->saturation) || !zr::is_finite(params->agx_exp))
        {
            zr::set_error("zr_display_pass_set_params: tonemapper must be 0..%d and saturation / agx_exp finite", (int)ZR_TONEMAPPER_AGX_CUSTOM);
            return ZR_ERR_INVALID_ARG;
        }
        p->params = *params;
        return ZR_OK;
    }
    zr_status zr_display_pass_set_lut(zr_display_pass* p, const uint32_t* h_rgb9e5, uint32_t dim)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->SetLut(h_rgb9e5, dim);
    }
    zr_status zr_display_pass_render(zr_display_pass* p, const zr_frame_inputs* in, const void* d_signal, const void* d_exposure, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, d_signal, d_exposure, (cudaStream_t)stream);
    }
    zr_status zr_display_pass_set_rows(zr_display_pass* p, uint32_t y0, uint32_t y1) { return p ? p->strip.SetRows(y0, y1, p->height) : ZR_ERR_INVALID_ARG; }
    zr_status zr_display_pass_set_view(zr_display_pass* p, uint32_t view, float roughness_th)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        if (view > ZR_DISPLAY_VIEW_DEPTH || !zr::is_finite(roughness_th))
        {
            zr::set_error("zr_display_pass_set_view: view must be 0..%d and roughness_th finite (got %u, %g)", (int)ZR_DISPLAY_VIEW_DEPTH,
                view, (double)roughness_th);
            return ZR_ERR_INVALID_ARG;
        }
        p->view = view; p->roughnessTh = roughness_th;
        return ZR_OK;
    }
    zr_status zr_display_pass_set_picked(zr_display_pass* p, const uint32_t* h_instances, uint32_t n)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        if (n > ZR_DISPLAY_MAX_PICKED || (n && !h_instances))
        {
            zr::set_error("zr_display_pass_set_picked: need n <= %u instance indices (got n = %u, %s)", ZR_DISPLAY_MAX_PICKED, n,
                h_instances ? "data" : "NULL");
            return ZR_ERR_INVALID_ARG;
        }
        for (uint32_t k = 0; k < n; k++) p->picked[k] = h_instances[k];
        p->numPicked = n;
        return ZR_OK;
    }
    zr_status zr_display_pass_get_output(zr_display_pass* p, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        *out = zr_image2d{ p->sz.d_out, p->width, p->height, p->width * 4u, 4u };
        return ZR_OK;
    }
    void zr_display_pass_destroy(zr_display_pass* p) { delete p; }
}
