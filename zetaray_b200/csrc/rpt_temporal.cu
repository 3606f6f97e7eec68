// rpt_temporal.cu -- ReSTIR PT temporal reuse as classify -> per-case shift queues -> merge.
//
// Replaces Sort x2, Replay x2, ReSTIR_PT_Reconnect_CtT.hlsl and ReSTIR_PT_Reconnect_TtC.hlsl and produces the oracle's bytes;
// the execution model is the one of the spatial pass (rpt_spatial.cu, zr_rpt_shift.cuh):
//   k_temporal_classify  per pixel: reprojection + the validity tests both reconnection kernels start with (plane distance, roughness,
//                        transmissive flag; the replay's tighter plane test), which shifts are needed, their case / replay class;
//                        one flag byte per pixel for the merge, (pixel, direction) items for the queues
//   k_shift<.., true>    persistent blocks, one queue each
//   k_temporal_merge     per pixel: MIS weight of the current sample in the previous frame's domain, the reservoir update, the record
// None of the reference's temporal kernels has a wave-scope op, so the merge is a plain coalesced pass.
#include "zr_rpt_spatial.h"
#include "zr_rpt_shift.cuh"

namespace zr
{
namespace
{
    using namespace RPT;

    __global__ void __launch_bounds__(256) k_temporal_classify(SceneDev sc, FrameView f, RptParams prm, const zr_rpt_reservoir* __restrict__ resCurr,
        const zr_rpt_reservoir* __restrict__ resPrev, uint8_t* __restrict__ tflags, uint32_t* __restrict__ queue, uint32_t* __restrict__ counters,
        uint32_t capacity)
    {
        __shared__ uint32_t s_count[SpatialQueued::NUM_CLASSES], s_base[SpatialQueued::NUM_CLASSES];
        const int x = (int)(blockIdx.x * 32 + (threadIdx.x & 31));
        const int y = (int)(prm.rowBegin + blockIdx.y * 8 + (threadIdx.x >> 5));
        if (threadIdx.x < SpatialQueued::NUM_CLASSES) s_count[threadIdx.x] = 0;
        __syncthreads();
        uint32_t cls[2] = { NO_ITEM, NO_ITEM };     // [0] current -> previous frame (CtT), [1] previous frame -> current (TtC)
        uint32_t flagBits = 0;
        if (x < (int)f.W && y < (int)f.H && y < (int)prm.rowEnd)
        {
            const size_t idx = (size_t)y * f.W + x;
            const GFlags flags = DecodeFlags(ld128(&f.core[idx]).w & 0xff);
            bool ok = !(flags.invalid || flags.emissive), okReplay = false;
            int ppx = 0, ppy = 0;
            if (ok)
            {
                // temporal validity (identical tests in CtT, TtC and both replays; the replays use the tighter plane test)
                ok = PrevPixel(f, x, y, ppx, ppy);
                if (ok)
                    ok = asfloat(__ldg(&f.pcore[(size_t)ppy * f.W + ppx].x)) != FLT_MAX_;
            }
            if (ok)
            {
                const Pixel cur = LoadPixel(f, sc, f.core, f.coat, x, y, false, x, y);
                const Pixel prev = LoadPixel(f, sc, f.pcore, f.pcoat, ppx, ppy, true, x, y);
                ok = PlaneHeuristic(prev.pos, cur.normal, cur.pos, cur.z, 1.0f);
                okReplay = ok && PlaneHeuristic(prev.pos, cur.normal, cur.pos, cur.z, 0.01f);
                const bool matOk = !(prev.flags.emissive || (fabsf(prev.roughness - cur.roughness) > 0.3f) ||
                    (prev.flags.transmissive != cur.flags.transmissive));
                ok = ok && matOk;
                okReplay = okReplay && matOk;
            }
            if (ok)
            {
                flagBits = TF_OK | (okReplay ? TF_REPLAY_OK : 0);
                const uint4 q0 = ld128(&resCurr[idx]);
                const uint4 qp = ld128(&resPrev[(size_t)ppy * f.W + ppx]);
                const bool selfEmpty = (q0.x & 0xf) == Reconnection::EMPTY, pEmpty = (qp.x & 0xf) == Reconnection::EMPTY;
                const uint32_t M_p = (qp.x >> 4) & 0xf;
                if (asfloat(q0.y) != 0 && M_p > 0 && !selfEmpty) cls[0] = ShiftClass(q0.x);
                if (!pEmpty) cls[1] = ShiftClass(qp.x);
            }
            tflags[idx] = (uint8_t)flagBits;
        }
        const uint32_t base = (uint32_t)x | ((uint32_t)y << 16) | ((flagBits & TF_REPLAY_OK) ? (1u << 30) : 0u);
        const uint32_t item[2] = { base, base | (1u << 31) };
        AppendItems(cls, item, queue, counters, capacity, s_count, s_base);
    }

    // 4 blocks per SM = 64 registers (84 bytes of spills): a latency-bound streaming pass gains more from 32 resident warps than it loses
    // to the spills -- chosen over 80 registers (3 blocks) and 48 (5 blocks)
    __global__ void __launch_bounds__(256, 4) k_temporal_merge(SceneDev sc, FrameView f, RptParams prm, zr_rpt_reservoir* __restrict__ resCurr,
        const zr_rpt_reservoir* __restrict__ resPrev, float4* __restrict__ target, float4* __restrict__ finalImg,
        const uint8_t* __restrict__ tflags, const ShiftResult* __restrict__ shiftRes)
    {
        const zr_frame_constants& fc = f.fc;
        const int x = (int)(blockIdx.x * 32 + (threadIdx.x & 31));
        const int y = (int)(prm.rowBegin + blockIdx.y * 8 + (threadIdx.x >> 5));
        if (x >= (int)f.W || y >= (int)f.H || y >= (int)prm.rowEnd) return;
        const size_t idx = (size_t)y * f.W + x;
        {
            const GFlags flags = DecodeFlags(ld128(&f.core[idx]).w & 0xff);
            if (flags.invalid || flags.emissive) return;
        }
        zr_rpt_reservoir rec;
        LoadRecord(&resCurr[idx], rec);
        Reservoir r_curr = Reservoir::Load_NonReconnection(rec);
        const float4 tg = target[idx];
        r_curr.target = f3(tg.x, tg.y, tg.z);
        const bool ok = (__ldg(&tflags[idx]) & TF_OK) != 0;
        if (!ok)
        {
            if (!prm.spatialFlag)
                WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
            return;
        }
        int ppx = 0, ppy = 0;
        PrevPixel(f, x, y, ppx, ppy);
        const size_t pidx = (size_t)ppy * f.W + ppx;
        zr_rpt_reservoir recPrev;
        LoadRecord(&resPrev[pidx], recPrev);
        Reservoir r_prev = Reservoir::Load_NonReconnection(recPrev);
        const uint4* sp = reinterpret_cast<const uint4*>(&shiftRes[idx]);

        // ---- Reconnect_CtT: scale w_sum by the MIS weight of the current sample in the temporal domain ----
        if (r_curr.w_sum != 0 && r_prev.M > 0 && !r_curr.rc.Empty())
        {
            const float2 sh1 = __ldg(reinterpret_cast<const float2*>(&sp[1]));
            const float target_prev = sh1.x;
            if (target_prev > 0)
            {
                const float selfJ = (r_curr.rc.IsCase3() && r_curr.rc.lobe_k_min_1 == BSDF::ALL) ? 1.0f : asfloat(rec.jacobian_or_seed_nee);
                const float targetLum_curr = r_curr.W > 0 ? r_curr.w_sum / r_curr.W : 0;
                const float jacobian = selfJ > 0 ? sh1.y / selfJ : 0;
                const float m_curr = targetLum_curr / (targetLum_curr + (float)r_prev.M * target_prev * jacobian);
                r_curr.w_sum *= m_curr;
                rec.w_sum = r_curr.w_sum;
            }
        }

        // ---- Reconnect_TtC ----
        const uint32_t M_new = r_curr.M + r_prev.M;
        const uint32_t M_max = prm.M_max_temporal;
        if (r_prev.rc.Empty())
        {
            const float targetLum = Math::Luminance(r_curr.target);
            r_curr.W = targetLum > 0 ? r_curr.w_sum / targetLum : 0;
            r_curr.M = M_new;
            const uint32_t k = r_curr.rc.Empty() ? r_curr.rc.k : (r_curr.rc.k > 2 ? r_curr.rc.k : 2) - 2;
            const uint32_t mm = r_curr.M < M_max ? r_curr.M : M_max;
            rec.meta = (rec.meta & 0xffffff00u) | ((k | (mm << 4)) & 0xff);
            rec.W = r_curr.W;
            st128(&resCurr[idx], make_uint4(rec.meta, asuint(rec.w_sum), asuint(rec.W), rec.L_b));
            if (!prm.spatialFlag)
                WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
            return;
        }
        r_prev.Load_Reconnection(recPrev);
        if (r_prev.rc.IsCase1() || r_prev.rc.IsCase2())
            XkToCurr(sc, r_prev.rc);
        const uint4 sh0 = __ldg(&sp[0]);
        const float3 shTarget = f3(asfloat(sh0.x), asfloat(sh0.y), asfloat(sh0.z));
        const float shJ = asfloat(sh0.w);
        const float targetLum_curr = Math::Luminance(shTarget);
        const float jacobian = r_prev.rc.partialJacobian > 0 ? shJ / r_prev.rc.partialJacobian : 0;
        bool changed = false;
        if (targetLum_curr > 1e-6f && jacobian > 1e-5f)
        {
            RNG rng = RNG::Init((uint32_t)y, (uint32_t)x, fc.FrameNum + 31);
            const float targetLum_prev = r_prev.W > 0 ? r_prev.w_sum / r_prev.W : 0;
            const float numerator = (float)r_prev.M * targetLum_prev;
            const float denom = numerator / jacobian + targetLum_curr;
            const float m_prev = denom > 0 ? numerator / denom : 0;
            const float w_prev = m_prev * r_prev.W * targetLum_curr;
            if (r_curr.Update(w_prev, shTarget, r_prev.rc, rng))
            {
                r_curr.rc.partialJacobian = shJ;
                changed = true;
            }
        }
        const float targetLum = Math::Luminance(r_curr.target);
        r_curr.W = targetLum > 0 ? r_curr.w_sum / targetLum : 0;
        r_curr.M = M_new;
        if (changed)
        {
            zr_rpt_reservoir out;
            r_curr.Write(out, M_max);
            StoreRecord(&resCurr[idx], out);
            if (prm.spatialFlag)
            {
                r_curr.target = Math::Sanitize(r_curr.target);
                target[idx] = f4(r_curr.target.x, r_curr.target.y, r_curr.target.z, 0.0f);
            }
        }
        else
        {
            r_curr.WriteReservoirData(rec, M_max);
            st128(&resCurr[idx], make_uint4(rec.meta, asuint(rec.w_sum), asuint(rec.W), rec.L_b));
        }
        if (!prm.spatialFlag)
            WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
    }
}

zr_status SetupTemporalShifts()
{
    return SetupShifts<true>();
}

zr_status SpatialQueued::RunTemporal(const ShiftStreams& ss, const SceneDev& sc, const FrameView& f, const RptParams& prm, zr_rpt_reservoir* resCurr,
    const zr_rpt_reservoir* resPrev, float4* target, float4* finalImg, bool plain, cudaStream_t stream)
{
    const uint32_t rows = prm.rowEnd - prm.rowBegin;
    const dim3 grid((width + 31) / 32, (rows + 7) / 8);
    ZR_CUDA(cudaMemsetAsync(d_counters, 0, 16 * sizeof(uint32_t), stream));
    {
        ZR_PROF("k_temporal_classify", stream);
        k_temporal_classify<<<grid, 256, 0, stream>>>(sc, f, prm, resCurr, resPrev, d_flags, d_queue, d_counters, (uint32_t)capacity);
        ZR_LAUNCH_CHECK();
    }
    {
        ZR_PROF("k_shift_temporal", stream);
        const zr_status ls = LaunchShifts<true>(*this, ss, sc, f, prm, resCurr, resPrev, nullptr, plain, stream);
        zr::prof_after();
        if (ls != ZR_OK) return ls;
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return zr::cuda_fail(e, "k_shift (temporal) launch");
    }
    {
        ZR_PROF("k_temporal_merge", stream);
        k_temporal_merge<<<grid, 256, 0, stream>>>(sc, f, prm, resCurr, resPrev, target, finalImg, d_flags, d_shift);
        ZR_LAUNCH_CHECK();
    }
    return ZR_OK;
}
} // namespace zr
