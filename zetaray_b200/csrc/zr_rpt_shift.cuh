// zr_rpt_shift.cuh -- the shift engine of the queued reuse passes: persistent blocks drain one queue of (pixel, direction) items
// that all hold the same reconnection case and replay class, so every lane of every warp runs the same phases of the hybrid shift
// (zr_rpt.cuh Replay_kGt2_Sync / Shift2_Sync<CASE>) on real work. Used by the spatial pass (rpt_spatial.cu: current <-> neighbour
// pixel of the same frame) and by the temporal pass (rpt_temporal.cu: current <-> reprojected pixel of the previous frame).
//
// Block size: 512 threads x 2 blocks per SM (64 registers): the block-synchronous phases want many warps behind each
// instruction-cache line, so fewer, larger register budgets (256 x 2, 512 x 1 at 128 registers) or more, smaller blocks
// (256 x 4, 128 x 4) trade away the wrong resource. The choice has not been re-measured on H100 (same register file and
// thread limits per SM as the part it was tuned on).
#pragma once
#include "zr_rpt_spatial.h"

namespace zr
{
namespace
{
    using namespace RPT;
    constexpr int SHIFT_THREADS = 512, SHIFT_MINBLOCKS = 2;
    constexpr uint32_t NO_ITEM = 0xffffffffu;

    // queue class of a reservoir's sample from its metadata word: (case 1, 2, 3) x (k == 2, k > 2)
    ZR_D uint32_t ShiftClass(uint32_t meta)
    {
        const uint32_t kMin2 = meta & 0xf;                              // never EMPTY here
        const uint32_t lt_k = (meta >> 14) & 3, lt_k1 = (meta >> 16) & 3;
        const uint32_t c = lt_k1 != 0 ? 1u : (lt_k != 0 ? 2u : 0u);     // Reconnection::IsCase2 / IsCase3 / IsCase1
        return c * 2 + (kMin2 > 0 ? 1u : 0u);
    }


    // item = x | y << 16 | flag << 30 | direction << 31 (x < 65536, y < 16384); flag: temporal pass only, "the tighter plane test
    // of the replay passed" (ReSTIR_PT_Replay.hlsl:404)
    template<int CASE, bool REPLAY, bool TEMPORAL>
    __global__ void __launch_bounds__(SHIFT_THREADS, SHIFT_MINBLOCKS) k_shift(SceneDev sc, FrameView f, RptParams prm,
        const zr_rpt_reservoir* __restrict__ resIn, const zr_rpt_reservoir* __restrict__ resPrev, const uint16_t* __restrict__ neighbor,
        const uint32_t* __restrict__ queue, uint32_t* __restrict__ counters, uint32_t cls, ShiftResult* __restrict__ out)
    {
        __shared__ uint32_t s_base;
        const uint32_t total = counters[cls];
        for (;;)
        {
            __syncthreads();
            if (threadIdx.x == 0) s_base = atomicAdd(&counters[8 + cls], (uint32_t)SHIFT_THREADS);
            __syncthreads();
            const uint32_t base = s_base;
            if (base >= total) break;
            const bool act = base + threadIdx.x < total;
            int x = 0, y = 0;
            uint32_t dir = 0;
            bool replayOk = act;
            Reservoir r = Reservoir::Init();
            Pixel p, pr;
            if (act)
            {
                const uint32_t item = __ldg(&queue[base + threadIdx.x]);
                x = (int)(item & 0xffff); y = (int)((item >> 16) & 0x3fff); dir = item >> 31;
                zr_rpt_reservoir rec;
                if (!TEMPORAL)
                {
                    // spatial: direction 0 shifts this pixel's sample to the neighbour's primary vertex (coat parameters read at the
                    // centre pixel, Reconnect_CtS.hlsl:100), direction 1 the neighbour's sample to this pixel
                    int nx = 0, ny = 0;
                    NeighborOf(f, neighbor, x, y, nx, ny);
                    LoadRecord(dir == 0 ? &resIn[(size_t)y * f.W + x] : &resIn[(size_t)ny * f.W + nx], rec);
                    r = Reservoir::Load_NonReconnection(rec);
                    r.rc.x_k_in_motion = false;
                    r.Load_Reconnection(rec);
                    if (dir == 0) p = LoadPixel(f, sc, f.core, f.coat, nx, ny, false, x, y);
                    else p = LoadPixel(f, sc, f.core, f.coat, x, y, false, x, y);
                    if (REPLAY)
                    {
                        if (dir == 0) pr = LoadPixel(f, sc, f.core, f.coat, nx, ny, false, nx, ny);
                        else pr = p;
                    }
                }
                else
                {
                    // temporal: direction 0 shifts this frame's sample to the reprojected pixel of the previous frame (x_k moved to
                    // where its instance was, Reconnect_CtT.hlsl:258-272), direction 1 the previous frame's sample to this pixel
                    replayOk = ((item >> 30) & 1) != 0;
                    int ppx = 0, ppy = 0;
                    PrevPixel(f, x, y, ppx, ppy);
                    LoadRecord(dir == 0 ? &resIn[(size_t)y * f.W + x] : &resPrev[(size_t)ppy * f.W + ppx], rec);
                    r = Reservoir::Load_NonReconnection(rec);
                    r.Load_Reconnection(rec);
                    if (r.rc.IsCase1() || r.rc.IsCase2())
                    {
                        if (dir == 0) XkToPrev(sc, r.rc);
                        else XkToCurr(sc, r.rc);
                    }
                    if (dir == 0) p = LoadPixel(f, sc, f.pcore, f.pcoat, ppx, ppy, true, x, y);
                    else p = LoadPixel(f, sc, f.core, f.coat, x, y, false, x, y);
                    if (REPLAY) pr = p;
                }
            }
            OffsetPathContext ctx = OffsetPathContext::Init();
            if (REPLAY)
            {
                ZR_PHASE();
                ctx = Replay_kGt2_Sync(act && replayOk, sc, pr.pos, pr.normal, pr.eta_next, pr.surface, r.rc, prm.alpha_min);
                if (act && replayOk)
                    ctx = ctx.Quantize();
            }
            const OffsetPath shift = Shift2_Sync<CASE>(act, sc, p.pos, p.normal, p.eta_next, p.surface, r.rc, &ctx, prm.alpha_min);
            if (act)
            {
                ShiftResult* o = &out[(size_t)y * f.W + x];
                if (dir == 0)
                    *reinterpret_cast<float2*>(&o->ctsTargetLum) = f2(Math::Luminance(shift.target), shift.partialJacobian);
                else if (TEMPORAL)
                    st128(o, make_uint4(asuint(shift.target.x), asuint(shift.target.y), asuint(shift.target.z), asuint(shift.partialJacobian)));
                else
                {
                    // the spatial merge accepts the shifted sample only for 1e-5 < J / J_n < 100, so a Jacobian that is not positive
                    // is as good as zero; positive ones carry the "x_{k-1} transmissive" bit of the shifted path in the sign
                    const float J = shift.partialJacobian;
                    const float Jenc = J > 0 ? (shift.surfKMin1Tramsmissive ? -J : J) : 0.0f;
                    st128(o, make_uint4(asuint(shift.target.x), asuint(shift.target.y), asuint(shift.target.z), asuint(Jenc)));
                }
            }
        }
    }

    // One launch per class; a launch whose queue is empty costs a few microseconds (its blocks leave at the first claim). The launches
    // share nothing but read-only inputs -- each has its own queue and claim cursor, and the two items of a pixel write disjoint bytes of
    // its ShiftResult -- so they go to three streams (fork / join by events around the stage): a persistent block leaves as soon as its
    // queue is drained, which frees its slot for the next class's blocks. Measured on the strip-sharded frame, where every queue is a
    // fraction of the machine (DESIGN 7).
    template<bool TEMPORAL>
    zr_status LaunchShifts(SpatialQueued& q, const SceneDev& sc, const FrameView& f, const RptParams& prm, const zr_rpt_reservoir* resIn,
        const zr_rpt_reservoir* resPrev, const uint16_t* neighbor, cudaStream_t stream)
    {
        const uint32_t grid = (uint32_t)q.numSMs * SHIFT_MINBLOCKS;
        const bool fork = q.aux[0] && q.aux[1];
        cudaStream_t s1 = fork ? q.aux[0] : stream, s2 = fork ? q.aux[1] : stream;
        if (fork)
        {
            ZR_CUDA(cudaEventRecord(q.evFork, stream));
            ZR_CUDA(cudaStreamWaitEvent(s1, q.evFork, 0));
            ZR_CUDA(cudaStreamWaitEvent(s2, q.evFork, 0));
        }
#define ZR_LAUNCH_SHIFT(CASE, REPLAY, CLS, STREAM) \
        k_shift<CASE, REPLAY, TEMPORAL><<<grid, SHIFT_THREADS, 0, STREAM>>>(sc, f, prm, resIn, resPrev, neighbor, q.d_queue + (size_t)(CLS) * q.capacity, \
            q.d_counters, CLS, q.d_shift); \
        zr::count_launch()
        ZR_LAUNCH_SHIFT(1, false, 0, stream);
        ZR_LAUNCH_SHIFT(2, false, 2, s1);
        ZR_LAUNCH_SHIFT(3, false, 4, s2);
        ZR_LAUNCH_SHIFT(1, true, 1, s1);
        ZR_LAUNCH_SHIFT(2, true, 3, s2);
        ZR_LAUNCH_SHIFT(3, true, 5, stream);
#undef ZR_LAUNCH_SHIFT
        if (fork)
        {
            ZR_CUDA(cudaEventRecord(q.evJoin[0], s1));
            ZR_CUDA(cudaEventRecord(q.evJoin[1], s2));
            ZR_CUDA(cudaStreamWaitEvent(stream, q.evJoin[0], 0));
            ZR_CUDA(cudaStreamWaitEvent(stream, q.evJoin[1], 0));
        }
        return ZR_OK;
    }

    // block-aggregated append of up to two items per thread (cls[d] == NO_ITEM: none) to the per-class queues:
    // warp ballots -> shared counters -> one global atomic per class and block. Called by every thread of a 256-thread block.
    ZR_D void AppendItems(const uint32_t cls[2], const uint32_t item[2], uint32_t* __restrict__ queue, uint32_t* __restrict__ counters,
        uint32_t capacity, uint32_t* s_count, uint32_t* s_base)
    {
        const uint32_t lane = threadIdx.x & 31;
        uint32_t offs[2] = { 0, 0 };
        const uint32_t lt = (1u << lane) - 1;
#pragma unroll
        for (uint32_t c = 0; c < SpatialQueued::NUM_CLASSES; c++)
        {
            const uint32_t m0 = __ballot_sync(0xffffffffu, cls[0] == c), m1 = __ballot_sync(0xffffffffu, cls[1] == c);
            const uint32_t n0 = __popc(m0), n = n0 + __popc(m1);
            uint32_t base = 0;
            if (n && lane == 0) base = atomicAdd(&s_count[c], n);
            base = __shfl_sync(0xffffffffu, base, 0);
            if (cls[0] == c) offs[0] = base + __popc(m0 & lt);
            if (cls[1] == c) offs[1] = base + n0 + __popc(m1 & lt);
        }
        __syncthreads();
        if (threadIdx.x < SpatialQueued::NUM_CLASSES)
            s_base[threadIdx.x] = s_count[threadIdx.x] ? atomicAdd(&counters[threadIdx.x], s_count[threadIdx.x]) : 0;
        __syncthreads();
#pragma unroll
        for (uint32_t d = 0; d < 2; d++)
            if (cls[d] != NO_ITEM)
                queue[(size_t)cls[d] * capacity + s_base[cls[d]] + offs[d]] = item[d];
    }
}
} // namespace zr
