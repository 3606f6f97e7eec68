// svgf.cu -- SVGF denoiser: temporal accumulation + variance estimate, then a-trous wavelet passes as TMA-tiled stencils.
//
// No counterpart in the reference (ZetaRay ships no SVGF; BASELINE.json's north_star and config 3 name it): the algorithm is
// defined by oracle/orc_svgf.cpp and this file is held to it bit for bit (tests/test_svgf_gpu.py).
//
// Execution model of an a-trous pass with step s. A tap pattern with stride s never leaves its sub-lattice
// {(x, y) : x = u s + px, y = v s + py}, so the image is VIEWED as a 4-D tensor {px, u, py, v} (strides 8 B, 8 s B, pitch, s pitch) and a
// block filters a dense 32 x 16 box of lattice points for two adjacent x-phases: one cp.async.bulk.tensor.4d brings the (32 + 2R) x
// (16 + 2R) x 2 lattice box of colour + variance, a second one the guide box {depth, normal}, both land as dense tiles in shared memory
// whatever the step (SASS: UTMALDG.4D), are expanded once to float (normal decode and luminance once per staged pixel, not once per
// tap), filtered from shared memory, and the result tile leaves through one cp.async.bulk.tensor.4d store (UTMASTG.4D). Every pass
// therefore reads 1.2-1.4x and writes 1.0x its algorithmic bytes from L2 / HBM at any step, with no strided global access.
// Step 1 is the same kernel over a plain 2-D map (64 x 16 pixel tiles).
//
// Strip-sharded frames (zr_svgf_pass_set_rows / set_halo_exchange): the temporal stage computes the strip's rows, every a-trous
// pass launches only the tiles whose output rows meet the strip, and the pass calls the halo hook after each stage on the planes
// the next stage reads beyond the strip. One pass reaches at most R * 2^k <= 32 rows, so the exchange before it fits the halo.
#include "zr_common.cuh"
#include "zr_planes.h"
#include "zr_schedule.h"
#include "zr_tma.cuh"
#include <cstdlib>

namespace zr
{
namespace
{
    struct SvgfParamsDev { float sigma_z, k_n, sigma_l; };

    ZR_D void UnpackCV(uint2 p, float3& c, float& var)
    {
        c = f3(half_lo(p.x), half_hi(p.x), half_lo(p.y));
        var = half_hi(p.y);
    }
    ZR_D uint2 PackCV(float3 c, float var) { return make_uint2(pack_half2(c.x, c.y), pack_half2(c.z, var)); }

    // -----------------------------------------------------------------------------------------------------------------
    // temporal accumulation + variance (orc_svgf_temporal) of rows [rowBegin, rowEnd), rowEnd <= height. Internal planes are padded
    // to `pitch` pixels per row. The 3x3 variance fallback reads `core` and `color` one row beyond the rows it computes.
    // -----------------------------------------------------------------------------------------------------------------
    __global__ void __launch_bounds__(256) k_svgf_temporal(zr_frame_constants fc, const uint4* __restrict__ core, const uint2* __restrict__ me,
        const float4* __restrict__ color, const uint2* __restrict__ prevGuide, const uint4* __restrict__ histPrev, int historyValid,
        uint4* __restrict__ histCurr, uint2* __restrict__ cv, uint2* __restrict__ guide, uint32_t pitch, uint32_t rowBegin, uint32_t rowEnd)
    {
        const int W = (int)fc.RenderWidth, H = (int)fc.RenderHeight;
        const int x = (int)(blockIdx.x * 32 + (threadIdx.x & 31)), y = (int)(rowBegin + blockIdx.y * 8 + (threadIdx.x >> 5));
        if (x >= W || y >= (int)rowEnd) return;
        const size_t idx = (size_t)y * W + x, pidxOut = (size_t)y * pitch + x;
        const uint4 cr = ld128(&core[idx]);
        const float z = asfloat(cr.x);
        const float4 c4 = __ldg(&color[idx]);
        const float3 c = f3(c4.x, c4.y, c4.z);
        if (z == FLT_MAX_)
        {
            cv[pidxOut] = PackCV(c, 0.0f);
            guide[pidxOut] = make_uint2(asuint(FLT_MAX_), 0u);
            histCurr[pidxOut] = make_uint4(0u, 0u, 0u, 0u);
            return;
        }
        const float3 n = Math::DecodeUnitVector(Math::DecodeUNorm2(cr.y));
        const float l = Math::Luminance(c);
        float3 col = c; float m1 = l, m2 = l * l, N = 1.0f;
        if (historyValid)
        {
            const float2 renderDim = f2((float)W, (float)H);
            const float2 motionVec = unpack_snorm16x2(__ldg(&me[idx].x));
            const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / renderDim;
            const float2 prevUV = currUV - motionVec;
            const float2 pp = prevUV * renderDim;
            const int ppx = (int)pp.x, ppy = (int)pp.y;
            if (!(prevUV.x < 0.0f || prevUV.y < 0.0f || prevUV.x > 1.0f || prevUV.y > 1.0f) && ppx < W && ppy < H)
            {
                const size_t pidx = (size_t)ppy * pitch + ppx;
                const uint2 pg = __ldg(&prevGuide[pidx]);
                const float zp = asfloat(pg.x);
                if (zp != FLT_MAX_ && fabsf(zp - z) <= 0.1f * z)
                {
                    const float3 np = Math::DecodeUnitVector(Math::DecodeUNorm2(pg.y));
                    if (dot(np, n) >= 0.9f)
                    {
                        const uint4 h = ld128(&histPrev[pidx]);
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
            float s1 = 0, s2 = 0, cnt = 0;
            for (int j = -1; j <= 1; j++)
                for (int i = -1; i <= 1; i++)
                {
                    const int tx = x + i, ty = y + j;
                    if (tx < 0 || ty < 0 || tx >= W || ty >= H) continue;
                    const size_t t = (size_t)ty * W + tx;
                    if (asfloat(__ldg(&core[t].x)) == FLT_MAX_) continue;
                    const float4 ct = __ldg(&color[t]);
                    const float lt = Math::Luminance(f3(ct.x, ct.y, ct.z));
                    s1 += lt; s2 = fmaf(lt, lt, s2); cnt += 1.0f;
                }
            const float mean = s1 / cnt;
            var = fmaxf(var, fmaxf(0.0f, s2 / cnt - mean * mean));
        }
        cv[pidxOut] = PackCV(col, var);
        guide[pidxOut] = make_uint2(cr.x, cr.y);
        st128(&histCurr[pidxOut], make_uint4(pack_half2(col.x, col.y), pack_half2(col.z, 0.0f), pack_half2(m1, m2), pack_half2(N, 0.0f)));
    }

    // -----------------------------------------------------------------------------------------------------------------
    // one a-trous pass. R = tap radius (1: 3x3, 2: 5x5); P = 2: strided lattice through 4-D maps (step >= 2), P = 1: step 1
    // -----------------------------------------------------------------------------------------------------------------
    template<int R, int P>
    struct AtrousTile
    {
        static constexpr int TU = P == 2 ? 32 : 64;                 // lattice columns of the output tile (x P phases each)
        static constexpr int TV = 16;
        // apron columns left and right. A TMA box must start on a 16-byte boundary in global memory: with 8-byte pixels the step-1
        // map needs an EVEN start column, so its apron is 2 even for the 3x3 taps (an odd start is an illegal-instruction fault,
        // r2i); in the lattice maps the innermost dimension is the 16-byte phase pair, so any lattice column will do.
        static constexpr int AX = P == 2 ? R : 2;
        static constexpr int ROW = (TU + 2 * AX) * P;               // staged elements per lattice row
        static constexpr int SV = TV + 2 * R;
        static constexpr int NS = ROW * SV;
        static constexpr int OUT = TU * P * TV;                     // 1024
        // shared memory layout (bytes)
        static constexpr int OFF_RAWC = 0;
        static constexpr int OFF_RAWG = OFF_RAWC + ((NS * 8 + 127) / 128) * 128;
        static constexpr int OFF_OUT = OFF_RAWG + ((NS * 8 + 127) / 128) * 128;
        static constexpr int OFF_F = OFF_OUT + OUT * 8;             // expanded box: 2 x float4 + 1 float per staged pixel
        static constexpr int OFF_BAR = OFF_F + 9 * NS * 4;
        static constexpr int BYTES = ((OFF_BAR + 8 + 127) / 128) * 128;
    };

    template<int R, int P, bool LAST>
    // The tensor maps are read from global memory (one address per (pass, plane), uploaded once when the pass is sized) instead of
    // travelling as 3 x 128 bytes of __grid_constant__ parameters with each of the five launches. The pass computes output rows
    // [rowBegin, rowEnd), rowEnd <= H; blockIdx.x = tile column + tilesU * (tile row - first tile row of the phase meeting those rows);
    // tilesV = tile rows of the whole frame.
    __global__ void __launch_bounds__(512, 2) k_svgf_atrous(const CUtensorMap* __restrict__ pMapIn, const CUtensorMap* __restrict__ pMapGuide,
        const CUtensorMap* __restrict__ pMapOut, float4* __restrict__ outF, uint32_t W, uint32_t H, uint32_t step, uint32_t tilesU,
        uint32_t tilesV, uint32_t rowBegin, uint32_t rowEnd, SvgfParamsDev prm)
    {
        using T = AtrousTile<R, P>;
        extern __shared__ __align__(128) unsigned char smem[];
        uint2* rawC = reinterpret_cast<uint2*>(smem + T::OFF_RAWC);
        uint2* rawG = reinterpret_cast<uint2*>(smem + T::OFF_RAWG);
        uint2* outT = reinterpret_cast<uint2*>(smem + T::OFF_OUT);
        // expanded box: {r, g, b, variance}, {depth, normal}, luminance -- two 128-bit and one 32-bit shared-memory load per tap
        float4* s_cv = reinterpret_cast<float4*>(smem + T::OFF_F);
        float4* s_zn = s_cv + T::NS;
        float* s_lum = reinterpret_cast<float*>(s_zn + T::NS);
        uint64_t* bar = reinterpret_cast<uint64_t*>(smem + T::OFF_BAR);
        const uint32_t t = threadIdx.x;
        // phase of the sub-lattice: x-phases 2 * pair, 2 * pair + 1; y-phase py
        const int pair = P == 2 ? (int)(blockIdx.y % (step / 2)) : 0, py = P == 2 ? (int)(blockIdx.y / (step / 2)) : 0;
        // Tile rows are selected per y-phase: from the phase's first tile row holding an image row >= rowBegin, as many as the phase
        // that needs most (the host's count), so a phase may run one tile row past the strip, but none past the frame. A strip's
        // tiles also hold rows outside the strip, and intermediate passes store them whole: those rows may be computed from stale
        // bands. That is harmless: before the next pass reads them the halo exchange overwrites the 32 rows either side of the
        // strip, and no pass reads further than 32 rows beyond it. The whole frame (rowBegin = 0, rowEnd = H) runs every tile.
        // (step is a power of two: a shift, not an integer division, in every block's prologue)
        const uint32_t vBegin = rowBegin > (uint32_t)py ? (rowBegin - (uint32_t)py + step - 1) >> (__ffs(step) - 1) : 0u;
        const int tu = (int)(blockIdx.x % tilesU), tv = (int)(vBegin / T::TV + blockIdx.x / tilesU);
        if (tv >= (int)tilesV) return;
        const int u0 = tu * T::TU, v0 = tv * T::TV;
        if (t == 0)
        {
            tma::MbarInit(bar, 1);
            tma::FenceBarrierInit();
        }
        __syncthreads();
        if (t == 0)
        {
            tma::MbarArriveExpectTx(bar, 2u * T::NS * 8u);
            if (P == 2)
            {
                tma::Load4D(rawC, pMapIn, bar, 2 * pair, u0 - T::AX, py, v0 - R);
                tma::Load4D(rawG, pMapGuide, bar, 2 * pair, u0 - T::AX, py, v0 - R);
            }
            else
            {
                tma::Load2D(rawC, pMapIn, bar, u0 - T::AX, v0 - R);
                tma::Load2D(rawG, pMapGuide, bar, u0 - T::AX, v0 - R);
            }
        }
        tma::MbarWait(bar, 0);
        // expand the staged box once: halves -> float, luminance, normal decode; outside the image -> depth = FLT_MAX (weight 0)
        for (int e = (int)t; e < T::NS; e += 512)
        {
            const int sv = e / T::ROW, col = e % T::ROW;
            int x, y;
            if (P == 2) { x = (u0 - T::AX + (col >> 1)) * (int)step + 2 * pair + (col & 1); y = (v0 - R + sv) * (int)step + py; }
            else { x = u0 - T::AX + col; y = v0 - R + sv; }
            const bool inImg = x >= 0 && y >= 0 && x < (int)W && y < (int)H;
            float3 c = f3(0); float var = 0, z = FLT_MAX_; float3 n = f3(0);
            if (inImg)
            {
                UnpackCV(rawC[e], c, var);
                const uint2 g = rawG[e];
                z = asfloat(g.x);
                n = Math::DecodeUnitVector(Math::DecodeUNorm2(g.y));
            }
            s_cv[e] = f4(c.x, c.y, c.z, var);
            s_zn[e] = f4(z, n.x, n.y, n.z);
            s_lum[e] = Math::Luminance(c);
        }
        __syncthreads();
        constexpr float h5[5] = { 1.0f / 16, 1.0f / 4, 3.0f / 8, 1.0f / 4, 1.0f / 16 };
        constexpr float h3[3] = { 1.0f / 4, 1.0f / 2, 1.0f / 4 };
#pragma unroll
        for (int k = 0; k < 2; k++)
        {
            const int o = (int)t + k * 512;
            const int ov = o / (T::TU * P), ocol = o % (T::TU * P);
            const int ci = (ov + R) * T::ROW + ocol + T::AX * P;
            const float4 cvc = s_cv[ci], znc = s_zn[ci];
            const float zc = znc.x;
            uint2 packed = rawC[ci];
            float4 res = cvc;
            if (zc != FLT_MAX_)
            {
                const float3 cc = f3(cvc.x, cvc.y, cvc.z);
                const float varc = cvc.w, lc = s_lum[ci];
                const float3 nc = f3(znc.y, znc.z, znc.w);
                const float invZ = 1.0f / (prm.sigma_z * zc * (float)step);
                const float invL = 1.0f / fmaf(prm.sigma_l, sqrtf(fmaxf(varc, 0.0f)), 1e-4f);
                const float oneMinusK = 1.0f - prm.k_n;
                const float w0 = (R == 2 ? h5[2] : h3[1]) * (R == 2 ? h5[2] : h3[1]);
                float3 sumC = cc * w0;
                float sumV = (w0 * w0) * varc, sumW = w0;
#pragma unroll
                for (int j = -R; j <= R; j++)
#pragma unroll
                    for (int i = -R; i <= R; i++)
                    {
                        if (i == 0 && j == 0) continue;
                        const int ti = ci + j * T::ROW + i * P;
                        const float hw = (R == 2 ? h5[i + R] : h3[i + R]) * (R == 2 ? h5[j + R] : h3[j + R]);
                        const float4 cvt = s_cv[ti], znt = s_zn[ti];
                        const float wz = fmaf(-fabsf(znt.x - zc), invZ, 1.0f);
                        const float ndot = fmaf(znt.y, nc.x, fmaf(znt.z, nc.y, znt.w * nc.z));
                        const float wn = fmaf(ndot, prm.k_n, oneMinusK);
                        const float wl = fmaf(-fabsf(s_lum[ti] - lc), invL, 1.0f);
                        // wz, wl <= 1 by construction (1 - |d| * inv, one rounding), so max(., 0) is a saturate: one FFMA.SAT each
                        float w = hw * __saturatef(wz);
                        w = w * fmaxf(wn, 0.0f);
                        w = w * __saturatef(wl);
                        sumC = f3(fmaf(w, cvt.x, sumC.x), fmaf(w, cvt.y, sumC.y), fmaf(w, cvt.z, sumC.z));
                        sumV = fmaf(w * w, cvt.w, sumV);
                        sumW = sumW + w;
                    }
                const float3 oc = sumC / sumW;
                const float ovar = sumV / (sumW * sumW);
                packed = PackCV(oc, ovar);
                res = f4(oc.x, oc.y, oc.z, ovar);
            }
            if (LAST)
            {
                int x, y;
                if (P == 2) { x = (u0 + (ocol >> 1)) * (int)step + 2 * pair + (ocol & 1); y = (v0 + ov) * (int)step + py; }
                else { x = u0 + ocol; y = v0 + ov; }
                if (x < (int)W && y >= (int)rowBegin && y < (int)rowEnd)
                    outF[(size_t)y * W + x] = res;
            }
            else
                outT[o] = packed;
        }
        if (!LAST)
        {
            tma::FenceProxyAsync();
            __syncthreads();
            if (t == 0)
            {
                if (P == 2) tma::Store4D(pMapOut, outT, 2 * pair, u0, py, v0);
                else tma::Store2D(pMapOut, outT, u0, v0);
                tma::StoreCommit();
                tma::StoreWaitAll();
            }
        }
    }
}
} // namespace zr

// ---------------------------------------------------------------------------------------------------------------------
// pass object
// ---------------------------------------------------------------------------------------------------------------------
struct zr_svgf_pass
{
    static constexpr int MAX_PASSES = 5;
    uint32_t width = 0, height = 0;
    struct Sized
    {
        zr::Planes planes{ "zr_svgf_pass" };
        uint32_t pitch = 0, rows = 0;       // padded plane size in pixels
        uint2* d_cv[2] = { nullptr, nullptr };
        uint2* d_guide[2] = { nullptr, nullptr };
        uint4* d_hist[2] = { nullptr, nullptr };
        float4* d_out = nullptr;
        CUtensorMap* d_maps = nullptr;      // [kind 0 = cv load, 1 = cv store, 2 = guide load][pass][plane]; load boxes depend on the radius
    } sz;
    int cur = 0;
    bool historyValid = false;
    zr_svgf_params params = Defaults();
    zr::StripRows strip{ "zr_svgf_pass" };
    const CUtensorMap* DevMap(int kind, int k, int plane) const { return sz.d_maps + ((kind * MAX_PASSES + k) * 2 + plane); }
    zr_image2d Padded(void* d_plane, uint32_t texelBytes) const { return zr_image2d{ d_plane, width, height, sz.pitch * texelBytes, texelBytes }; }

    static zr_svgf_params Defaults() { zr_svgf_params p{}; p.sigma_z = 0.02f; p.k_n = 16.0f; p.sigma_l = 4.0f; p.radius = 2; p.num_passes = 5; return p; }

    zr_status Setup()
    {
        using namespace zr;
        cudaError_t e = cudaSuccess;
#define ZR_SVGF_ATTR(R, P, LAST) \
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_svgf_atrous<R, P, LAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, AtrousTile<R, P>::BYTES)
        ZR_SVGF_ATTR(1, 1, false); ZR_SVGF_ATTR(1, 1, true); ZR_SVGF_ATTR(1, 2, false); ZR_SVGF_ATTR(1, 2, true);
        ZR_SVGF_ATTR(2, 1, false); ZR_SVGF_ATTR(2, 1, true); ZR_SVGF_ATTR(2, 2, false); ZR_SVGF_ATTR(2, 2, true);
#undef ZR_SVGF_ATTR
        if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(k_svgf_atrous)");
        return ZR_OK;
    }

    // writes the maps of s's planes for radius R to s.d_maps; on failure s.d_maps is unchanged
    static zr_status EncodeMaps(const Sized& s, uint32_t R)
    {
        using namespace zr;
        CUtensorMap host[3][MAX_PASSES][2];     // [cv load, cv store, guide load][pass][plane]
        for (int k = 0; k < MAX_PASSES; k++)
        {
            const uint64_t st = 1ull << k;
            for (int pl = 0; pl < 2; pl++)
            {
                bool ok = true;
                if (st == 1)
                {
                    const uint64_t dims[2] = { s.pitch, s.rows };
                    const uint64_t strides[1] = { (uint64_t)s.pitch * 8 };
                    const uint32_t boxL[2] = { 64 + 2 * 2, 16 + 2 * R }, boxS[2] = { 64, 16 };       // AtrousTile<R, 1>::AX == 2
                    ok = ok && tma::EncodeWords(&host[0][k][pl], s.d_cv[pl], 2, dims, strides, boxL);
                    ok = ok && tma::EncodeWords(&host[2][k][pl], s.d_guide[pl], 2, dims, strides, boxL);
                    ok = ok && tma::EncodeWords(&host[1][k][pl], s.d_cv[pl], 2, dims, strides, boxS);
                }
                else
                {
                    // {phase_x, u, phase_y, v}: pixel (u s + phase_x, v s + phase_y)
                    const uint64_t dims[4] = { st, s.pitch / st, st, s.rows / st };
                    const uint64_t strides[3] = { st * 8, (uint64_t)s.pitch * 8, st * (uint64_t)s.pitch * 8 };
                    const uint32_t boxL[4] = { 2, 32 + 2 * R, 1, 16 + 2 * R }, boxS[4] = { 2, 32, 1, 16 };
                    ok = ok && tma::EncodeWords(&host[0][k][pl], s.d_cv[pl], 4, dims, strides, boxL);
                    ok = ok && tma::EncodeWords(&host[2][k][pl], s.d_guide[pl], 4, dims, strides, boxL);
                    ok = ok && tma::EncodeWords(&host[1][k][pl], s.d_cv[pl], 4, dims, strides, boxS);
                }
                if (!ok)
                {
                    set_error("zr_svgf_pass: cuTensorMapEncodeTiled failed (step %u)", (unsigned)st);
                    return ZR_ERR_CUDA;
                }
            }
        }
        // no kernel may still be using the old maps, and the new ones are in place before the next launch
        ZR_CUDA(cudaDeviceSynchronize());
        ZR_CUDA(cudaMemcpy(s.d_maps, host, sizeof(host), cudaMemcpyHostToDevice));
        ZR_CUDA(cudaDeviceSynchronize());
        return ZR_OK;
    }

    zr_status OnWindowResized(uint32_t w, uint32_t h)
    {
        Sized next;
        // padded so that (a) every lattice view divides evenly (multiples of 32 >= 2 * 16) and (b) no TMA box is larger than the
        // tensor it is cut from, even for the coarsest lattice (step 16: 36 x 20 lattice points) of a small image
        next.pitch = (w + 31) / 32 * 32; next.rows = (h + 31) / 32 * 32;
        if (next.pitch < 16u * 36u) next.pitch = 16u * 36u;
        if (next.rows < 16u * 20u) next.rows = 16u * 20u;
        const size_t n = (size_t)next.pitch * next.rows;
        for (int i = 0; i < 2; i++)
        {
            ZR_TRY(next.planes.Alloc(next.d_cv[i], n));
            ZR_TRY(next.planes.Alloc(next.d_guide[i], n));
            ZR_TRY(next.planes.Alloc(next.d_hist[i], n));
        }
        ZR_TRY(next.planes.Alloc(next.d_out, (size_t)w * h));
        ZR_TRY(next.planes.Alloc(next.d_maps, 3 * MAX_PASSES * 2, false));
        ZR_TRY(next.planes.Clear());
        ZR_TRY(EncodeMaps(next, params.radius));
        sz = std::move(next);
        width = w; height = h;
        strip.ForgetRows();
        historyValid = false; cur = 0;
        return ZR_OK;
    }

    zr_status ResetTemporal()
    {
        ZR_TRY(sz.planes.Clear());
        historyValid = false; cur = 0;
        return ZR_OK;
    }

    // tile rows of `tileRows` lattice rows each that hold image rows [y0, y1) of y-phase py (lattice row v = image row v s + py),
    // counted from the first such tile row
    static uint32_t PhaseTileRows(uint32_t y0, uint32_t y1, uint32_t s, uint32_t py, uint32_t tileRows)
    {
        const uint32_t vBegin = y0 > py ? (y0 - py + s - 1) / s : 0, vEnd = y1 > py ? (y1 - py + s - 1) / s : 0;
        return vEnd > vBegin ? (vEnd + tileRows - 1) / tileRows - vBegin / tileRows : 0;
    }

    template<int R>
    zr_status LaunchAtrous(int k, int inPlane, bool last, uint32_t y0, uint32_t y1, cudaStream_t stream)
    {
        using namespace zr;
        const uint32_t s = 1u << k;
        const SvgfParamsDev prm{ params.sigma_z, params.k_n, params.sigma_l };
        const CUtensorMap* mIn = DevMap(0, k, inPlane);
        const CUtensorMap* mG = DevMap(2, k, cur);
        const CUtensorMap* mOut = DevMap(1, k, 1 - inPlane);
        ZR_PROF("k_svgf_atrous", stream);
        if (s == 1)
        {
            using T = AtrousTile<R, 1>;
            const uint32_t tilesU = (width + T::TU - 1) / T::TU, tilesV = (height + T::TV - 1) / T::TV;
            const dim3 grid(tilesU * PhaseTileRows(y0, y1, 1, 0, T::TV), 1);
            if (last) k_svgf_atrous<R, 1, true><<<grid, 512, T::BYTES, stream>>>(mIn, mG, mOut, sz.d_out, width, height, s, tilesU, tilesV, y0, y1, prm);
            else k_svgf_atrous<R, 1, false><<<grid, 512, T::BYTES, stream>>>(mIn, mG, mOut, sz.d_out, width, height, s, tilesU, tilesV, y0, y1, prm);
        }
        else
        {
            using T = AtrousTile<R, 2>;
            const uint32_t latW = (width + s - 1) / s, latH = (height + s - 1) / s;
            const uint32_t tilesU = (latW + T::TU - 1) / T::TU, tilesV = (latH + T::TV - 1) / T::TV;
            uint32_t rowsOfTiles = 0;
            for (uint32_t py = 0; py < s; py++) rowsOfTiles = std::max(rowsOfTiles, PhaseTileRows(y0, y1, s, py, T::TV));
            const dim3 grid(tilesU * rowsOfTiles, (s / 2) * s);
            if (last) k_svgf_atrous<R, 2, true><<<grid, 512, T::BYTES, stream>>>(mIn, mG, mOut, sz.d_out, width, height, s, tilesU, tilesV, y0, y1, prm);
            else k_svgf_atrous<R, 2, false><<<grid, 512, T::BYTES, stream>>>(mIn, mG, mOut, sz.d_out, width, height, s, tilesU, tilesV, y0, y1, prm);
        }
        ZR_LAUNCH_CHECK();
        if (getenv("ZR_SVGF_DEBUG"))
        {
            cudaError_t e = cudaStreamSynchronize(stream);
            if (e != cudaSuccess) { set_error("k_svgf_atrous pass %d (step %u, radius %d, last %d): %s", k, s, R, (int)last, cudaGetErrorString(e)); return ZR_ERR_CUDA; }
        }
        return ZR_OK;
    }

    zr_status Render(const zr_frame_inputs* in, const void* d_signal, cudaStream_t stream)
    {
        using namespace zr;
        if (!in || !in->curr.d_core || !in->curr.d_motion_emissive || !d_signal)
        {
            set_error("zr_svgf_pass_render: missing input");
            return ZR_ERR_INVALID_ARG;
        }
        const zr_status fs = check_frame_size("zr_svgf_pass", in->frame, width, height);
        if (fs != ZR_OK) return fs;
        cur = 1 - cur;
        const uint32_t y0 = strip.rowBegin, y1 = strip.ClampedRowEnd(height);
        {
            ZR_PROF("k_svgf_temporal", stream);
            k_svgf_temporal<<<dim3((width + 31) / 32, (y1 - y0 + 7) / 8), 256, 0, stream>>>(in->frame, (const uint4*)in->curr.d_core,
                (const uint2*)in->curr.d_motion_emissive, (const float4*)d_signal, sz.d_guide[1 - cur], sz.d_hist[1 - cur], historyValid ? 1 : 0,
                sz.d_hist[cur], sz.d_cv[0], sz.d_guide[cur], sz.pitch, y0, y1);
            ZR_LAUNCH_CHECK();
        }
        // the a-trous passes read colour + variance and the guide beyond the strip; next frame's reprojection reads guide + history
        const zr_image2d temporalOut[3] = { Padded(sz.d_cv[0], 8u), Padded(sz.d_guide[cur], 8u), Padded(sz.d_hist[cur], 16u) };
        strip.Exchange(temporalOut, 3, stream);
        int plane = 0;
        for (uint32_t k = 0; k < params.num_passes; k++)
        {
            const bool last = k + 1 == params.num_passes;
            zr_status st = params.radius == 2 ? LaunchAtrous<2>((int)k, plane, last, y0, y1, stream) : LaunchAtrous<1>((int)k, plane, last, y0, y1, stream);
            if (st != ZR_OK) return st;
            plane = 1 - plane;
            // the next pass reads the plane just written beyond the strip; after the last one, TAA reads the denoised signal there
            const zr_image2d written = last ? zr_image2d{ sz.d_out, width, height, width * 16u, 16u } : Padded(sz.d_cv[plane], 8u);
            strip.Exchange(&written, 1, stream);
        }
        historyValid = true;
        return ZR_OK;
    }
};

extern "C"
{
    zr_status zr_svgf_pass_create(uint32_t width, uint32_t height, zr_svgf_pass** out) { return zr::CreatePass("zr_svgf_pass", width, height, out); }
    zr_status zr_svgf_pass_resize(zr_svgf_pass* p, uint32_t width, uint32_t height) { return zr::ResizePass("zr_svgf_pass", p, width, height); }
    zr_status zr_svgf_pass_reset_temporal(zr_svgf_pass* p) { return zr::ResetPass(p); }
    zr_status zr_svgf_pass_default_params(zr_svgf_params* out) { return zr::DefaultParams<zr_svgf_pass>(out); }
    zr_status zr_svgf_pass_set_params(zr_svgf_pass* p, const zr_svgf_params* params)
    {
        if (!p || !params) return ZR_ERR_INVALID_ARG;
        if ((params->radius != 1 && params->radius != 2) || params->num_passes < 1 || params->num_passes > zr_svgf_pass::MAX_PASSES ||
            !(params->sigma_z > 0) || !(params->sigma_l > 0) || !(params->k_n >= 0))
        {
            zr::set_error("zr_svgf_pass_set_params: radius must be 1 or 2, 1..5 passes, positive sigmas");
            return ZR_ERR_INVALID_ARG;
        }
        if (params->radius != p->params.radius) ZR_TRY(zr_svgf_pass::EncodeMaps(p->sz, params->radius));
        p->params = *params;
        return ZR_OK;
    }
    zr_status zr_svgf_pass_set_rows(zr_svgf_pass* p, uint32_t y0, uint32_t y1) { return p ? p->strip.SetRows(y0, y1, p->height) : ZR_ERR_INVALID_ARG; }
    zr_status zr_svgf_pass_set_halo_exchange(zr_svgf_pass* p, zr_halo_exchange_fn fn, void* user) { return p ? p->strip.SetHaloExchange(fn, user) : ZR_ERR_INVALID_ARG; }
    zr_status zr_svgf_pass_render(zr_svgf_pass* p, const zr_frame_inputs* in, const void* d_signal, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, d_signal, (cudaStream_t)stream);
    }
    zr_status zr_svgf_pass_get_output(zr_svgf_pass* p, zr_svgf_output id, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        const uint32_t w = p->width, h = p->height;
        switch (id)
        {
        case ZR_SVGF_DENOISED: *out = zr_image2d{ p->sz.d_out, w, h, w * 16u, 16u }; break;
        case ZR_SVGF_ACCUMULATED: *out = p->Padded(p->sz.d_cv[0], 8u); break;       // only valid with num_passes == 1 .. see header
        case ZR_SVGF_GUIDE: *out = p->Padded(p->sz.d_guide[p->cur], 8u); break;
        case ZR_SVGF_HISTORY: *out = p->Padded(p->sz.d_hist[p->cur], 16u); break;
        default: zr::set_error("zr_svgf_pass_get_output: unknown output id"); return ZR_ERR_INVALID_ARG;
        }
        return ZR_OK;
    }
    void zr_svgf_pass_destroy(zr_svgf_pass* p) { delete p; }
}
