// ORACLE -- test infrastructure, not product code (see orc_math.h header).
//
// Scalar restatement of the SVGF denoiser of zetaray_b200/csrc/svgf.cu. NO REFERENCE COUNTERPART: ZetaRay ships no SVGF pass
// (SURVEY.md:24-28; BASELINE.json's north_star and config 3 name it), so this file DEFINES the algorithm and the CUDA kernels are
// held to it bit for bit. Parity unpinned by construction (nothing in the reference to pin against).
//
// The filter (after Schied et al. 2017, "Spatiotemporal Variance-Guided Filtering", with arithmetic chosen so that every operation is
// an IEEE + - x / sqrt or an explicit fmaf -- no transcendental -- and the kernel stays close to its bandwidth bound):
//   temporal pass   reproject with the G-buffer motion vector (nearest), accept on relative depth (10 %) and normal (n.n' >= 0.9),
//                   blend colour and the first two luminance moments with alpha = max(1 / N, 0.2), N = history length <= 32;
//                   variance = max(0, m2 - m1^2), replaced by the 3x3 spatial estimate while N < 4
//   a-trous passes  step 1, 2, 4, 8, 16; B3-spline taps (5x5, radius 2) or the 3x3 binomial (radius 1);
//                   w = h_i h_j * max(0, 1 - |dz| / (sigma_z z_c step)) * max(0, k_n n.n_c + (1 - k_n)) * max(0, 1 - |dl| / (sigma_l sqrt(var_c) + 1e-4));
//                   colour' = sum w c / sum w, variance' = sum w^2 var / (sum w)^2, taps in row-major order, centre first
// Storage: colour + variance as 4 x binary16 (variance in alpha), guide = {view depth f32, oct32 normal}.
#include "orc_api.h"
#include "orc_gbuffer.h"
#include <thread>
#include <vector>

using namespace orc;

namespace
{
    struct SvgfParams { float sigma_z, k_n, sigma_l; uint32_t radius; };

    inline void unpack_cv(uint2 p, float3& c, float& var)
    {
        c = f3(half_lo(p.x), half_hi(p.x), half_lo(p.y));
        var = half_hi(p.y);
    }
    inline uint2 pack_cv(float3 c, float var)
    {
        uint2 r; r.x = pack_half2(c.x, c.y); r.y = pack_half2(c.z, var);
        return r;
    }
    template<class F>
    void rows(int H, int nthreads, F fn)
    {
        std::vector<std::thread> th;
        for (int t = 0; t < nthreads; t++)
            th.emplace_back([=] { for (int y = t; y < H; y += nthreads) fn(y); });
        for (auto& t : th) t.join();
    }
}

extern "C"
{
    // color: float4[w*h] noisy input; core / me: current G-buffer; prevGuide: uint2[w*h] {z, oct normal} of the previous frame;
    // histPrev / histCurr: uint4[w*h] {half4 colour | half m1, m2, N, 0}; cv: uint2[w*h]; guide: uint2[w*h]
    void orc_svgf_temporal(const zr_frame_constants* fc, const uint32_t* core_, const uint32_t* me_, const float* color_, const uint32_t* prevGuide_,
        const uint32_t* histPrev_, int historyValid, uint32_t* histCurr_, uint32_t* cv_, uint32_t* guide_, int nthreads)
    {
        const uint4* core = (const uint4*)core_;
        const uint2* me = (const uint2*)me_;
        const float4* color = (const float4*)color_;
        const uint2* prevGuide = (const uint2*)prevGuide_;
        const uint4* histPrev = (const uint4*)histPrev_;
        uint4* histCurr = (uint4*)histCurr_;
        uint2* cv = (uint2*)cv_;
        uint2* guide = (uint2*)guide_;
        const int W = (int)fc->RenderWidth, H = (int)fc->RenderHeight;
        rows(H, nthreads, [=](int y)
        {
            for (int x = 0; x < W; x++)
            {
                const size_t idx = (size_t)y * W + x;
                const float z = asfloat(core[idx].x);
                const float3 c = f3(color[idx].x, color[idx].y, color[idx].z);
                if (z == FLT_MAX_)
                {
                    cv[idx] = pack_cv(c, 0.0f);
                    guide[idx] = uint2{ asuint(FLT_MAX_), 0u };
                    histCurr[idx] = uint4{ 0u, 0u, 0u, 0u };
                    continue;
                }
                const float3 n = Math::DecodeUnitVector(Math::DecodeUNorm2(core[idx].y));
                const float l = Math::Luminance(c);
                float3 col = c; float m1 = l, m2 = l * l, N = 1.0f;
                if (historyValid)
                {
                    const float2 renderDim = f2((float)W, (float)H);
                    const float2 motionVec = unpack_snorm16x2(me[idx].x);
                    const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / renderDim;
                    const float2 prevUV = currUV - motionVec;
                    const float2 pp = prevUV * renderDim;
                    const int ppx = (int)pp.x, ppy = (int)pp.y;
                    if (!(prevUV.x < 0.0f || prevUV.y < 0.0f || prevUV.x > 1.0f || prevUV.y > 1.0f) && ppx < W && ppy < H)
                    {
                        const size_t pidx = (size_t)ppy * W + ppx;
                        const float zp = asfloat(prevGuide[pidx].x);
                        if (zp != FLT_MAX_ && fabsf(zp - z) <= 0.1f * z)
                        {
                            const float3 np = Math::DecodeUnitVector(Math::DecodeUNorm2(prevGuide[pidx].y));
                            if (dot(np, n) >= 0.9f)
                            {
                                const uint4 h = histPrev[pidx];
                                const float3 hc = f3(half_lo(h.x), half_hi(h.x), half_lo(h.y));
                                const float hm1 = half_lo(h.z), hm2 = half_hi(h.z), hN = half_lo(h.w);
                                N = fminf(hN + 1.0f, 32.0f);
                                const float alpha = fmaxf(1.0f / N, 0.2f);
                                col = f3(fmaf(alpha, c.x - hc.x, hc.x), fmaf(alpha, c.y - hc.y, hc.y), fmaf(alpha, c.z - hc.z, hc.z));
                                m1 = fmaf(alpha, l - hm1, hm1);
                                m2 = fmaf(alpha, l * l - hm2, hm2);
                            }
                        }
                    }
                }
                float var = fmaxf(0.0f, m2 - m1 * m1);
                if (N < 4.0f)
                {
                    // spatial estimate over the 3x3 neighbourhood of the noisy input (valid depth only), row-major
                    float s1 = 0, s2 = 0, cnt = 0;
                    for (int j = -1; j <= 1; j++)
                        for (int i = -1; i <= 1; i++)
                        {
                            const int tx = x + i, ty = y + j;
                            if (tx < 0 || ty < 0 || tx >= W || ty >= H) continue;
                            const size_t t = (size_t)ty * W + tx;
                            if (asfloat(core[t].x) == FLT_MAX_) continue;
                            const float lt = Math::Luminance(f3(color[t].x, color[t].y, color[t].z));
                            s1 += lt; s2 = fmaf(lt, lt, s2); cnt += 1.0f;
                        }
                    const float mean = s1 / cnt;
                    var = fmaxf(var, fmaxf(0.0f, s2 / cnt - mean * mean));
                }
                cv[idx] = pack_cv(col, var);
                guide[idx] = uint2{ core[idx].x, core[idx].y };
                uint4 h;
                h.x = pack_half2(col.x, col.y); h.y = pack_half2(col.z, 0.0f); h.z = pack_half2(m1, m2); h.w = pack_half2(N, 0.0f);
                histCurr[idx] = h;
            }
        });
    }

    // one a-trous iteration: in -> out (both uint2[w*h]); outF (float4[w*h], optional) receives the unquantised result as well
    void orc_svgf_atrous(uint32_t W_, uint32_t H_, const uint32_t* guide_, const uint32_t* in_, uint32_t* out_, float* outF_, uint32_t step,
        const float* params4, int nthreads)
    {
        const uint2* guide = (const uint2*)guide_;
        const uint2* in = (const uint2*)in_;
        uint2* out = (uint2*)out_;
        float4* outF = (float4*)outF_;
        const int W = (int)W_, H = (int)H_, s = (int)step;
        const SvgfParams prm{ params4[0], params4[1], params4[2], (uint32_t)params4[3] };
        const int R = (int)prm.radius;
        static const float h5[5] = { 1.0f / 16, 1.0f / 4, 3.0f / 8, 1.0f / 4, 1.0f / 16 };
        static const float h3[3] = { 1.0f / 4, 1.0f / 2, 1.0f / 4 };
        const float* hk = R == 2 ? h5 : h3;
        rows(H, nthreads, [=](int y)
        {
            for (int x = 0; x < W; x++)
            {
                const size_t idx = (size_t)y * W + x;
                const float zc = asfloat(guide[idx].x);
                float3 cc; float varc;
                unpack_cv(in[idx], cc, varc);
                if (zc == FLT_MAX_)
                {
                    out[idx] = in[idx];
                    if (outF) outF[idx] = f4(cc.x, cc.y, cc.z, varc);
                    continue;
                }
                const float3 nc = Math::DecodeUnitVector(Math::DecodeUNorm2(guide[idx].y));
                const float lc = Math::Luminance(cc);
                const float invZ = 1.0f / (prm.sigma_z * zc * (float)s);
                const float invL = 1.0f / fmaf(prm.sigma_l, sqrtf(fmaxf(varc, 0.0f)), 1e-4f);
                const float oneMinusK = 1.0f - prm.k_n;
                const float w0 = hk[R] * hk[R];
                float3 sumC = cc * w0;
                float sumV = (w0 * w0) * varc, sumW = w0;
                for (int j = -R; j <= R; j++)
                    for (int i = -R; i <= R; i++)
                    {
                        if (i == 0 && j == 0) continue;
                        const int tx = x + i * s, ty = y + j * s;
                        if (tx < 0 || ty < 0 || tx >= W || ty >= H) continue;
                        const size_t t = (size_t)ty * W + tx;
                        const float zt = asfloat(guide[t].x);
                        const float3 nt = Math::DecodeUnitVector(Math::DecodeUNorm2(guide[t].y));
                        float3 ct; float vart;
                        unpack_cv(in[t], ct, vart);
                        const float lt = Math::Luminance(ct);
                        const float wz = fmaf(-fabsf(zt - zc), invZ, 1.0f);
                        const float ndot = fmaf(nt.x, nc.x, fmaf(nt.y, nc.y, nt.z * nc.z));
                        const float wn = fmaf(ndot, prm.k_n, oneMinusK);
                        const float wl = fmaf(-fabsf(lt - lc), invL, 1.0f);
                        float w = (hk[i + R] * hk[j + R]) * fmaxf(wz, 0.0f);
                        w = w * fmaxf(wn, 0.0f);
                        w = w * fmaxf(wl, 0.0f);
                        sumC = f3(fmaf(w, ct.x, sumC.x), fmaf(w, ct.y, sumC.y), fmaf(w, ct.z, sumC.z));
                        sumV = fmaf(w * w, vart, sumV);
                        sumW = sumW + w;
                    }
                const float3 oc = sumC / sumW;
                const float ov = sumV / (sumW * sumW);
                out[idx] = pack_cv(oc, ov);
                if (outF) outF[idx] = f4(oc.x, oc.y, oc.z, ov);
            }
        });
    }
}
