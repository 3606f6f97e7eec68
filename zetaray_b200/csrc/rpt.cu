// rpt.cu -- ReSTIR PT: path generation, temporal and spatial path reuse, and the IndirectLighting pass.
//
// Replaces IndirectLighting/ReSTIR_PT/*.hlsl (24 compiled variants, IndirectLighting.h:257-289) and the
// host sequencing of IndirectLighting.cpp:370-1025 for the emissive-light integrator.
//
// Dispatch structure (the reference records 1 + 6 + 7 dispatches per frame):
//   k_pathtrace        == ReSTIR_PT_PathTrace           one warp == one reference wave (16x2 pixels of a 16x8
//                                                        group), bounce loop in lock-step so the Russian-roulette
//                                                        wave-max is a warp max
//   k_temporal         == Sort x2 + Replay x2 + Reconnect_CtT + Reconnect_TtC fused. None of them has a
//                         wave-scope op, so the sorted thread maps cannot change results: the kernel runs in
//                         pixel order and keeps the replay context and the CtT-scaled w_sum in registers.
//   k_spatial_search   == ReSTIR_PT_SpatialSearch
//   k_sort             == ReSTIR_PT_Sort (only the StC map is needed: it defines which 32 pixels share the
//                         boiling-suppression wave sums)
//   k_spatial          == Replay x2 + Reconnect_CtS + Reconnect_StC fused, run in the StC-sorted order
// Per-pixel state moves as 128-bit accesses: 64-byte reservoir records, float4 target/final, uint4 G-buffer.
#include "zr_rpt_io.cuh"
#include "zr_rpt_spatial.h"
#include "zr_schedule.h"
#include <cstdio>
#include <string>
#include <vector>
#include <dlfcn.h>

namespace zr
{
namespace
{
    using namespace RPT;

    // accounts the cycles a block took to the tile of its first pixel
    ZR_D void AccountCost(unsigned long long* costMap, uint32_t W, uint32_t H, uint32_t x, uint32_t y, long long t0)
    {
        if (costMap && threadIdx.x == 0 && x < W && y < H)
            atomicAdd(&costMap[(size_t)(y >> 5) * ((W + 31) >> 5) + (x >> 5)], (unsigned long long)(clock64() - t0));
    }

    // 512 x float2, indexed per pixel by a random offset: a __constant__ table would serialise the 32 different addresses of a warp
    __device__ __align__(8) float c_disk512[1024];

    // -------------------------------------------------------------------------------------------
    // PathTrace
    // -------------------------------------------------------------------------------------------
// 768 threads at 80 registers with the parked state below (157 KB of shared memory per block). Measured on an H100 SXM (700 W):
// 3.33 ms per bench frame, against 3.65 ms at 1024 x 64 registers, 3.52 ms at 512 x 128 and 4.40 ms at 512 x 2 blocks x 64
// (DESIGN 4.1).
#ifndef ZR_PT_THREADS
#define ZR_PT_THREADS 768
#endif
    // The path's cold state: the reservoir under construction and the path's own reconnection vertex. Only reservoir updates,
    // SetCase1/2/3 and Clear touch them, yet held in registers they competed with the hot state and spilled to local memory,
    // whose reloads go to L2 once a full SM's spill area outgrows L1. They live in dynamic shared memory, one record per
    // thread; the record's odd number of 32-bit words puts the 32 lanes of a warp in 32 different banks.
    struct PtParked
    {
        Reservoir r;
        Reconnection rc;
        uint32_t pad;
    };
    static_assert(sizeof(PtParked) % 4 == 0 && (sizeof(PtParked) / 4) % 2 == 1, "PtParked must be an odd number of words");
    constexpr size_t PT_SMEM_BYTES = (size_t)ZR_PT_THREADS * sizeof(PtParked);

    // A block is ZR_PT_THREADS/128 consecutive 16x8 groups of the reference's swizzled dispatch; each warp is one
    // reference wave. The warps of a block walk the bounce phases together (zr_rpt.cuh "block-synchronous phases").
    // Dynamic shared memory: PT_SMEM_BYTES (PtParked per thread).
    __global__ void ZR_LB(ZR_PT_THREADS) k_pathtrace(SceneDev sc, FrameView f, RptParams prm, zr_rpt_reservoir* __restrict__ res,
        float4* __restrict__ target, float4* __restrict__ finalImg, uint32_t dispX, uint32_t dispY, const uint32_t* __restrict__ order)
    {
        extern __shared__ PtParked s_ptParked[];
        const zr_frame_constants& fc = f.fc;
        const long long t0 = clock64();
        uint2 sg = make_uint2(0, 0);
        const uint32_t groupFlat = order[blockIdx.x] * (ZR_PT_THREADS / 128) + (threadIdx.x >> 7);
        const uint32_t tInGroup = threadIdx.x & 127;
        uint2 px = make_uint2(0xffffffffu, 0xffffffffu);
        if (groupFlat < dispX * dispY)
            px = SwizzleThreadGroup(groupFlat, 0, tInGroup & 15, tInGroup >> 4, 16, 8, dispX, 16, 4, 16 * dispY, sg);
        bool inBounds = px.x < f.W && px.y < f.H && px.y >= prm.rowBegin && px.y < prm.rowEnd;
        const size_t idx = (size_t)px.y * f.W + px.x;
        bool alive = false;
        if (inBounds)
        {
            const GFlags flags = FlagsAt(f.core, f.W, px.x, px.y);
            if (flags.invalid || flags.emissive)
            {
                if (!fc.Accumulate || !fc.CameraStatic)
                    finalImg[idx] = f4(0, 0, 0, 0);
                inBounds = false;
            }
        }
        // loop-carried state
        float3 pos = f3(0), normal = f3(0), li = f3(0), throughput = f3(0), throughput_k = f3(1), tr = f3(1);
        BSDF::ShadingData surface;
        BSDF::BSDFSample bsdfSample = BSDF::BSDFSample::Init();
        HitEmissive nextHit;
        nextHit.hit = false;
        Reconnection& rc = s_ptParked[threadIdx.x].rc;
        Reservoir& r = s_ptParked[threadIdx.x].r;
        rc = Reconnection::Init();
        r = Reservoir::Init();
        PrevHit prevHit;
        prevHit.alpha_lobe = 0; prevHit.wi = f3(0); prevHit.pdf = 0; prevHit.lobe = BSDF::DIFFUSE_R;
        float eta_curr = BSDF::ETA_AIR, eta_next = BSDF::DEFAULT_ETA_MAT;
        bool inTranslucentMedium = false;
        int bounce = 0, maxNumBounces = 0;
        RNG rngReplay, rngThread, rngGroup;
        rngReplay.State = rngThread.State = rngGroup.State = 0;
        uint32_t sampleSetIdx = 0;
        uint32_t seedReplay0 = 0;

        if (inBounds)
        {
            const Pixel p = LoadPixel(f, sc, f.core, f.coat, px.x, px.y, false, px.x, px.y);
            rngGroup = RNG::Init4(sg.x, sg.y, fc.FrameNum, 1);
            const uint3 state = RNG::PCG3d(make_uint3(px.x, px.y, fc.FrameNum));
            rngReplay = RNG::InitSeed(state.x);
            rngThread = RNG::InitSeed(state.y);
            seedReplay0 = state.x;
            maxNumBounces = (int)(p.surface.specTr ? prm.maxGlossyTrBounces : prm.maxNonTrBounces);
            bsdfSample = BSDF::SampleBSDF(p.normal, p.surface, rngReplay);
            if (dot(bsdfSample.bsdfOverPdf, bsdfSample.bsdfOverPdf) != 0)
            {
                sampleSetIdx = rngGroup.UniformUintBounded_Faster(sc.numSampleSets);    // one set per thread group (:406-408)
                pos = p.pos; normal = p.normal; surface = p.surface;
                throughput = bsdfSample.bsdfOverPdf;
                prevHit.alpha_lobe = BSDF::LobeAlpha(p.surface, bsdfSample.lobe);
                prevHit.lobe = bsdfSample.lobe; prevHit.wi = bsdfSample.wi; prevHit.pdf = bsdfSample.pdf;
                eta_curr = dot(p.normal, bsdfSample.wi) < 0 ? p.eta_next : BSDF::ETA_AIR;
                inTranslucentMedium = eta_curr != BSDF::ETA_AIR;
                alive = true;
            }
        }
        ZR_PHASE();
        if (alive)
            nextHit = FindClosestEmissive(sc, pos, normal, bsdfSample.wi, surface.Transmissive());

        // lock-step bounce loop (ReSTIR_PT_PathTrace.hlsli:227-355) as block-synchronous phases (zr_rpt.cuh)
        while (__syncthreads_or(alive))
        {
            bool atRR = false;
            Hit hitInfo;
            float prevBsdfSamplePdf = 0; BSDF::LOBE prevBsdfSampleLobe = BSDF::DIFFUSE_R;
            const int pathVertex = bounce + 2;
            // phase: attributes + material of the vertex the previous sample hit
            if (alive && !nextHit.hit)
                alive = false;
            if (alive)
            {
                hitInfo = HitAttributes(sc, nextHit.geoIdx, nextHit.primIdx, nextHit.bary, nextHit.t);
                const float3 newPos = mad(hitInfo.t, bsdfSample.wi, pos);
                if (!GetMaterialData(sc, -bsdfSample.wi, eta_curr, hitInfo, surface, eta_next))
                    alive = false;
                else
                {
                    pos = newPos;
                    normal = hitInfo.normal;
                    prevBsdfSamplePdf = bsdfSample.pdf;
                    prevBsdfSampleLobe = bsdfSample.lobe;
                    tr = f3(1);
                    if (inTranslucentMedium && (surface.trDepth > 0))
                    {
                        const float3 c = surface.baseColor_Fr0_TrCol;
                        const float3 extCoeff = f3(-zr_logf(c.x), -zr_logf(c.y), -zr_logf(c.z)) / surface.trDepth;
                        tr = f3(zr_expf(-hitInfo.t * extCoeff.x), zr_expf(-hitInfo.t * extCoeff.y), zr_expf(-hitInfo.t * extCoeff.z));
                        throughput *= tr;
                    }
                }
            }
            ZR_PHASE();
            // EstimateDirectAndUpdateRC<Emissive>. phase: draw the next direction (NEE_Bsdf, ReSTIR_PT_NEE.hlsli:145-222)
            BSDF::BSDFSample nextBsdfSample = bsdfSample;
            const int nextBounce = pathVertex - 1;
            if (alive && nextBounce <= maxNumBounces)
                nextBsdfSample = BSDF::SampleBSDF(hitInfo.normal, surface, rngReplay);
            ZR_PHASE();
            // phase: closest hit along it
            RaySetup rs; rs.go = false;
            RayHit rh; rh.hit = false;
            if (alive)
            {
                rs = SetupClosestEmissive(pos, hitInfo.normal, nextBsdfSample.wi, surface.Transmissive());
                if (rs.go)
                    rh = TraceClosest(sc, rs.o, nextBsdfSample.wi, rs.tmin, FLT_MAX_);
            }
            ZR_PHASE();
            // phase: BSDF-sampled light hit, then light sample + BSDF value (NEE_Emissive, ReSTIR_PT_NEE.hlsli:224-302)
            NeeLightState nee;
            nee.facing = false; nee.ld = f3(0);
            BSDF::ShadingData surfNee;
            bool lightSample = false;
            uint32_t seed_nee = 0;
            RaySetup seg; seg.go = false;
            if (alive)
            {
                nextHit = FinishClosestEmissive(sc, rs, rh, nextBsdfSample.wi);
                const DirectLightingEstimate ls_b = NEE_Bsdf_Finish(sc, pos, surface, nextBounce, maxNumBounces, nextBsdfSample, nextHit);
                if (nextHit.HitWasEmissive())
                {
                    const float3 fOverPdf = throughput * ls_b.ld;
                    li += fOverPdf;
                    rc.L = Reconnection::half3(ls_b.ld * throughput_k);
                    MaybeSetCase2OrCase3(pathVertex, pos, hitInfo.normal, hitInfo.t, hitInfo.ID, hitInfo.meshIdx, surface,
                        prevHit, ls_b, 0, rc, prm.alpha_min);
                    r.Update(Math::Luminance(fOverPdf), fOverPdf, rc, rngThread);
                }
                lightSample = !IsSpecularSurface(surface);
                if (lightSample)
                {
                    seed_nee = rngThread.State;
                    surfNee = surface;
                    nee = NEE_Emissive_Begin(sc, pos, hitInfo.normal, surfNee, sampleSetIdx, rngThread);
                    if (nee.facing && dot(nee.ld, nee.ld) > 0)
                        seg = SetupSegment(pos, nee.ret.wi, nee.t, hitInfo.normal, nee.ret.ID, surfNee.Transmissive());
                }
            }
            ZR_PHASE();
            // phase: shadow segment
            if (lightSample && nee.facing && dot(nee.ld, nee.ld) > 0)
            {
                const bool visible = seg.go ? !TraceAnyExcept(sc, seg.o, nee.ret.wi, seg.tmin, seg.tmax, nee.ret.ID) : false;
                nee.ld *= visible ? 1.0f : 0.0f;
            }
            ZR_PHASE();
            // phase: sampler pdf of the light direction, MIS, reservoir update
            if (lightSample)
            {
                float bsdfPdf = 0;
                if (nee.facing && dot(nee.ld, nee.ld) > 0)
                {
                    bsdfPdf = BSDF::BSDFSamplerPdf(hitInfo.normal, surfNee, nee.ret.wi, rngThread);
                    bsdfPdf *= nee.dwdA;
                }
                const DirectLightingEstimate ls = NEE_Emissive_Finish(nee, bsdfPdf);
                const float3 fOverPdf = throughput * ls.ld;
                li += fOverPdf;
                if (rc.IsCase2() || rc.IsCase3())
                    rc.Clear();
                rc.L = Reconnection::half3(ls.ld * throughput_k);
                MaybeSetCase2OrCase3(pathVertex, pos, hitInfo.normal, hitInfo.t, hitInfo.ID, hitInfo.meshIdx, surface,
                    prevHit, ls, seed_nee, rc, prm.alpha_min);
                r.Update(Math::Luminance(fOverPdf), fOverPdf, rc, rngThread);
            }
            if (alive)
            {
                bsdfSample = nextBsdfSample;
                if (bounce >= (maxNumBounces - 1))
                    alive = false;
                else
                {
                    if (rc.IsCase2() || rc.IsCase3())
                        rc.Clear();
                    bounce++;
                    atRR = true;
                }
            }
            // Russian roulette against the wave's maximum throughput
            const uint32_t rrMask = __ballot_sync(0xffffffffu, atRR);
            if (rrMask == 0)
                continue;
            const int rrBounce = __shfl_sync(0xffffffffu, bounce, __ffs(rrMask) - 1);
            const bool doRR = prm.russianRoulette && (rrBounce >= 3);
            float waveThroughput = 0.0f;
            if (doRR)
                waveThroughput = WaveMax32(atRR ? Math::Luminance(throughput) : -FLT_MAX_);
            if (atRR)
            {
                do
                {
                    if (doRR && waveThroughput < 1)
                    {
                        const float p_terminate = fmaxf(0.05f, 1 - waveThroughput);
                        if (rngGroup.Uniform() < p_terminate) { alive = false; break; }
                        throughput /= (1 - p_terminate);
                        throughput_k /= ((int)rc.k <= bounce) ? (1 - p_terminate) : 1.0f;
                    }
                    if (dot(bsdfSample.bsdfOverPdf, bsdfSample.bsdfOverPdf) == 0) { alive = false; break; }
                    const float alpha_lobe = BSDF::LobeAlpha(surface, bsdfSample.lobe);
                    if (rc.Empty() && CanReconnect(prevHit.alpha_lobe, alpha_lobe, prevHit.lobe, bsdfSample.lobe, prm.alpha_min))
                    {
                        rc.SetCase1(pathVertex, pos, hitInfo.t, hitInfo.normal, hitInfo.ID, hitInfo.meshIdx, -surface.wo,
                            prevBsdfSampleLobe, prevBsdfSamplePdf, bsdfSample.wi, bsdfSample.lobe, bsdfSample.pdf);
                        throughput_k = f3(1);
                    }
                    if ((int)rc.k <= bounce)
                        throughput_k *= bsdfSample.bsdfOverPdf * tr;
                    const bool transmitted = dot(normal, bsdfSample.wi) < 0;
                    throughput *= bsdfSample.bsdfOverPdf;
                    eta_curr = transmitted ? (eta_curr == BSDF::ETA_AIR ? eta_next : BSDF::ETA_AIR) : eta_curr;
                    inTranslucentMedium = eta_curr != BSDF::ETA_AIR;
                    prevHit.alpha_lobe = alpha_lobe;
                    prevHit.lobe = bsdfSample.lobe;
                    prevHit.wi = bsdfSample.wi;
                    prevHit.pdf = bsdfSample.pdf;
                } while (false);
            }
        }

        AccountCost(prm.costMap, f.W, f.H, px.x, px.y, t0);
        if (!inBounds)
            return;
        r.rc.seed_replay = seedReplay0;
        const float targetLum = Math::Luminance(r.target);
        r.W = targetLum > 0 ? fmaxf(r.w_sum / targetLum, 1.0f) : 0;
        if (prm.temporalResample || prm.resetTemporal)
        {
            zr_rpt_reservoir rec;
            r.Write(rec, 0);
            StoreRecord(&res[idx], rec);
        }
        if (prm.temporalResample)
        {
            r.target = Math::Sanitize(r.target);
            target[idx] = f4(r.target.x, r.target.y, r.target.z, 0.0f);
        }
        else
        {
            li = isnan3(li) ? f3(0) : li;
            if (fc.Accumulate && fc.CameraStatic)
            {
                const float4 prev = finalImg[idx];
                finalImg[idx] = f4(prev.x + li.x, prev.y + li.y, prev.z + li.z, prev.w);
            }
            else
                finalImg[idx] = f4(li.x, li.y, li.z, 0.0f);
        }
    }

    // -------------------------------------------------------------------------------------------
    // Temporal reuse: Reconnect_CtT then Reconnect_TtC for the same pixel (replay inline).
    // A block is 32 x ZR_RPT_THREADS/32 pixels, one warp per 8x4 tile; block-synchronous phases throughout,
    // so no thread leaves before the last barrier.
    // -------------------------------------------------------------------------------------------
#ifndef ZR_RPT_THREADS
#define ZR_RPT_THREADS 1024
#endif
    __global__ void ZR_LB(ZR_RPT_THREADS) k_temporal(SceneDev sc, FrameView f, RptParams prm, zr_rpt_reservoir* __restrict__ resCurr,
        const zr_rpt_reservoir* __restrict__ resPrev, float4* __restrict__ target, float4* __restrict__ finalImg,
        uint32_t gridX, const uint32_t* __restrict__ order)
    {
        const zr_frame_constants& fc = f.fc;
        const long long t0 = clock64();
        const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const uint32_t bid = order[blockIdx.x];
        const int x = (int)((bid % gridX) * 32 + (warp & 3) * 8 + (lane & 7));
        const int y = (int)((bid / gridX) * (ZR_RPT_THREADS / 32) + (warp >> 2) * 4 + (lane >> 3));
        bool act = !(x >= (int)f.W || y >= (int)f.H || y < (int)prm.rowBegin || y >= (int)prm.rowEnd);
        const size_t idx = act ? (size_t)y * f.W + x : 0;
        if (act)
        {
            const GFlags flags = DecodeFlags(ld128(&f.core[idx]).w & 0xff);
            if (flags.invalid || flags.emissive) act = false;
        }

        zr_rpt_reservoir rec;
        Reservoir r_curr = Reservoir::Init();
        int ppx = 0, ppy = 0;
        bool ok = false, okReplay = false;
        Pixel cur, prev;
        if (act)
        {
            LoadRecord(&resCurr[idx], rec);
            r_curr = Reservoir::Load_NonReconnection(rec);
            const float4 tg = target[idx];
            r_curr.target = f3(tg.x, tg.y, tg.z);
            // temporal validity (identical tests in CtT, TtC and both replays; the replays use the tighter plane test)
            ok = PrevPixel(f, x, y, ppx, ppy);
            float prevViewDepth = FLT_MAX_;
            if (ok)
            {
                prevViewDepth = asfloat(__ldg(&f.pcore[(size_t)ppy * f.W + ppx].x));
                ok = prevViewDepth != FLT_MAX_;
            }
        }
        ZR_PHASE();
        if (ok)
        {
            cur = LoadPixel(f, sc, f.core, f.coat, x, y, false, x, y);
            prev = LoadPixel(f, sc, f.pcore, f.pcoat, ppx, ppy, true, x, y);
            ok = PlaneHeuristic(prev.pos, cur.normal, cur.pos, cur.z, 1.0f);
            okReplay = ok && PlaneHeuristic(prev.pos, cur.normal, cur.pos, cur.z, 0.01f);
            const bool matOk = !(prev.flags.emissive || (fabsf(prev.roughness - cur.roughness) > 0.3f) ||
                (prev.flags.transmissive != cur.flags.transmissive));
            ok = ok && matOk;
            okReplay = okReplay && matOk;
        }
        if (act && !ok)
        {
            if (!prm.spatialFlag)
                WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
            act = false;
        }
        const size_t pidx = ok ? (size_t)ppy * f.W + ppx : 0;
        zr_rpt_reservoir recPrev;
        Reservoir r_prev = Reservoir::Init();
        if (ok)
        {
            LoadRecord(&resPrev[pidx], recPrev);
            r_prev = Reservoir::Load_NonReconnection(recPrev);
        }

        // ---- Reconnect_CtT: scale w_sum by the MIS weight of the current sample in the temporal domain ----
        {
            const bool doCtT = ok && r_curr.w_sum != 0 && r_prev.M > 0 && !r_curr.rc.Empty();
            Reservoir rc_full = Reservoir::Init();
            Reconnection rcOrig = Reconnection::Init();
            if (doCtT)
            {
                rc_full = r_curr;
                rc_full.Load_Reconnection(rec);
                rcOrig = rc_full.rc;
                if (rc_full.rc.IsCase1() || rc_full.rc.IsCase2())
                    XkToPrev(sc, rc_full.rc);
            }
            const bool needCtx = doCtT && rc_full.rc.k > 2;
            ZR_PHASE();
            OffsetPathContext ctx = Replay_kGt2_Sync(needCtx && okReplay, sc, prev.pos, prev.normal, prev.eta_next, prev.surface, rcOrig, prm.alpha_min);
            if (needCtx && okReplay)
                ctx = ctx.Quantize();
            const OffsetPath shift = Shift2_Sync(doCtT, sc, prev.pos, prev.normal, prev.eta_next, prev.surface, rc_full.rc, &ctx, prm.alpha_min);
            if (doCtT)
            {
                const float target_prev = Math::Luminance(shift.target);
                if (target_prev > 0)
                {
                    const float targetLum_curr = r_curr.W > 0 ? r_curr.w_sum / r_curr.W : 0;
                    const float jacobian = rc_full.rc.partialJacobian > 0 ? shift.partialJacobian / rc_full.rc.partialJacobian : 0;
                    const float m_curr = targetLum_curr / (targetLum_curr + (float)r_prev.M * target_prev * jacobian);
                    r_curr.w_sum *= m_curr;
                    rec.w_sum = r_curr.w_sum;
                }
            }
        }

        // ---- Reconnect_TtC ----
        const uint32_t M_new = r_curr.M + r_prev.M;
        const uint32_t M_max = prm.M_max_temporal;
        if (ok && r_prev.rc.Empty())
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
            ok = false;
        }
        Reconnection rcReplay = Reconnection::Init();
        if (ok)
        {
            r_prev.Load_Reconnection(recPrev);
            rcReplay = r_prev.rc;
            if (r_prev.rc.IsCase1() || r_prev.rc.IsCase2())
                XkToCurr(sc, r_prev.rc);
        }
        const bool needCtx = ok && r_prev.rc.k > 2;
        ZR_PHASE();
        OffsetPathContext ctx = Replay_kGt2_Sync(needCtx && okReplay, sc, cur.pos, cur.normal, cur.eta_next, cur.surface, rcReplay, prm.alpha_min);
        if (needCtx && okReplay)
            ctx = ctx.Quantize();
        const OffsetPath shift = Shift2_Sync(ok, sc, cur.pos, cur.normal, cur.eta_next, cur.surface, r_prev.rc, &ctx, prm.alpha_min);
        AccountCost(prm.costMap, f.W, f.H, (uint32_t)x, (uint32_t)y, t0);
        if (!ok)
            return;         // past the last barrier
        const float targetLum_curr = Math::Luminance(shift.target);
        const float jacobian = r_prev.rc.partialJacobian > 0 ? shift.partialJacobian / r_prev.rc.partialJacobian : 0;
        bool changed = false;
        if (targetLum_curr > 1e-6f && jacobian > 1e-5f)
        {
            RNG rng = RNG::Init((uint32_t)y, (uint32_t)x, fc.FrameNum + 31);
            const float targetLum_prev = r_prev.W > 0 ? r_prev.w_sum / r_prev.W : 0;
            const float numerator = (float)r_prev.M * targetLum_prev;
            const float denom = numerator / jacobian + targetLum_curr;
            const float m_prev = denom > 0 ? numerator / denom : 0;
            const float w_prev = m_prev * r_prev.W * targetLum_curr;
            if (r_curr.Update(w_prev, shift.target, r_prev.rc, rng))
            {
                r_curr.rc.partialJacobian = shift.partialJacobian;
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

    // -------------------------------------------------------------------------------------------
    // Spatial search
    // -------------------------------------------------------------------------------------------
    __global__ void __launch_bounds__(256) k_spatial_search(FrameView f, RptParams prm, uint16_t* __restrict__ neighbor)
    {
        const zr_frame_constants& fc = f.fc;
        const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31);
        const uint32_t y = prm.rowBegin + blockIdx.y * 8 + (threadIdx.x >> 5);
        if (x >= f.W || y >= f.H || y >= prm.rowEnd) return;
        const size_t idx = (size_t)y * f.W + x;
        const uint4 c = ld128(&f.core[idx]);
        const GFlags flags = DecodeFlags(c.w & 0xff);
        if (flags.invalid || flags.emissive) return;
        const float roughness = (float)((c.w >> 8) & 0xff) / 255.0f;
        const float viewDepth = asfloat(c.x);
        const float2 renderDimF = f2((float)f.W, (float)f.H);
        const float2 jitter = f2(fc.CurrCameraJitter[0], fc.CurrCameraJitter[1]);
        const float3 pos = Math::WorldPosFromScreenSpace(f2((float)x, (float)y), renderDimF, viewDepth, fc.TanHalfFOV,
            fc.AspectRatio, fc.CurrViewInv, jitter);
        const float3 normal = Math::DecodeUnitVector(Math::DecodeUNorm2(c.y));
        const uint3 h = RNG::PCG3d(make_uint3(x, y, fc.FrameNum));
        RNG rng = RNG::Init(h.x, h.y, fc.FrameNum);
        const float u0 = rng.Uniform();
        const uint32_t offset = rng.UniformUint();
        const float theta = u0 * TWO_PI;
        float sinTheta, cosTheta;
        zr_sincosf(theta, &sinTheta, &cosTheta);
        int foundX = 0xffff, foundY = 0xffff;
        // The three candidates are tested in order and the first that passes wins (ReSTIR_PT_SpatialSearch.hlsl:95-141); their G-buffer
        // records are fetched together, so the kernel waits for one gather round trip instead of up to three dependent ones.
        int sxs[3], sys[3];
        bool inside[3];
        uint4 cand[3];
#pragma unroll
        for (uint32_t i = 0; i < 3; i++)
        {
            const uint32_t si = (offset + i) & 511;
            const float2 sampleUV = __ldg(reinterpret_cast<const float2*>(c_disk512) + si);
            float2 rotated = f2(dot(sampleUV, f2(cosTheta, -sinTheta)), dot(sampleUV, f2(sinTheta, cosTheta)));
            rotated = rotated * 15.0f;
            sxs[i] = (int)rintf((float)x + rotated.x); sys[i] = (int)rintf((float)y + rotated.y);
            inside[i] = !(sxs[i] < 0 || sys[i] < 0 || sxs[i] >= (int)f.W || sys[i] >= (int)f.H) && !(sxs[i] == (int)x && sys[i] == (int)y);
            cand[i] = inside[i] ? ld128(&f.core[(size_t)sys[i] * f.W + sxs[i]]) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (uint32_t i = 0; i < 3; i++)
        {
            if (foundX != 0xffff || !inside[i]) continue;
            const int sxp = sxs[i], syp = sys[i];
            const uint4 sc4 = cand[i];
            const GFlags sf = DecodeFlags(sc4.w & 0xff);
            if (sf.invalid || sf.emissive) continue;
            if (flags.metallic != sf.metallic) continue;
            if (flags.transmissive != sf.transmissive) continue;
            const float sampleRoughness = (float)((sc4.w >> 8) & 0xff) / 255.0f;
            if (fabsf(sampleRoughness - roughness) > 0.05f) continue;
            const float3 samplePos = Math::WorldPosFromScreenSpace(f2((float)sxp, (float)syp), renderDimF, asfloat(sc4.x),
                fc.TanHalfFOV, fc.AspectRatio, fc.CurrViewInv, jitter);
            const float3 sampleNormal = Math::DecodeUnitVector(Math::DecodeUNorm2(sc4.y));
            if (!(fabsf(dot(normal, samplePos - pos)) <= 0.01f * viewDepth)) continue;
            if (dot(sampleNormal, normal) < 0.9f) continue;
            foundX = sxp; foundY = syp;
        }
        uint32_t mx, my;
        if (foundX == 0xffff) { mx = 0xff; my = 0xff; }
        else { mx = (uint32_t)(foundX - (int)x + 32); my = (uint32_t)(foundY - (int)y + 32); }
        neighbor[idx] = (uint16_t)((mx & 0xff) | ((my & 0xff) << 8));
    }

    // -------------------------------------------------------------------------------------------
    // Sort (ReSTIR_PT_Sort.hlsl): counting sort of a 32x32 tile by reconnection k. One block per tile,
    // each thread owns a 2x2 quad. Ranks are class-major, then thread (wave, lane) order, then quad
    // order -- the reference takes wave offsets with InterlockedAdd in arrival order (a race); wave
    // order is the deterministic member of that family.
    // mode: 0 = CtT, 1 = TtC, 2 = CtS, 3 = StC
    // -------------------------------------------------------------------------------------------
    __global__ void __launch_bounds__(256) k_sort(FrameView f, int mode, uint32_t spatialFlag, const zr_rpt_reservoir* __restrict__ resCurr,
        const zr_rpt_reservoir* __restrict__ resPrev, const uint16_t* __restrict__ neighbor, uint16_t* __restrict__ threadMap,
        uint32_t dispX, uint32_t dispY, uint32_t tileRow0)
    {
        enum { SUCCESS = 0, INVALID_PIXEL = 1, NOT_FOUND = 2, EMPTY = 4 };
        __shared__ unsigned long long s_warp[8];
        const uint32_t Gx = blockIdx.x, Gy = blockIdx.y + tileRow0, Gidx = threadIdx.x;      // only the tile rows of the owned strip are launched
        const uint32_t GTx = Gidx & 15, GTy = Gidx >> 4;
        const bool againstEdge = (Gx == dispX - 1) || (Gy == dispY - 1);
        const bool lastGroup = (Gx == dispX - 1) && (Gy == dispY - 1);
        int dxs[4], dys[4], cls[4];
        uint32_t result[4];
#pragma unroll
        for (int i = 0; i < 4; i++)
        {
            const int gtx = (int)GTx * 2 + (i & 1), gty = (int)GTy * 2 + (i >> 1);
            const int dx = (int)(Gx * 32) + gtx, dy = (int)(Gy * 32) + gty;
            dxs[i] = dx; dys[i] = dy;
            int nx = 0, ny = 0;
            uint32_t err = SUCCESS;
            if ((uint32_t)dx >= f.W || (uint32_t)dy >= f.H)
                err = INVALID_PIXEL;
            else
            {
                const GFlags flags = FlagsAt(f.core, f.W, dx, dy);
                if (flags.invalid || flags.emissive)
                    err = INVALID_PIXEL;
                else if (mode == 1)
                {
                    if (!PrevPixel(f, dx, dy, nx, ny)) err = NOT_FOUND;
                }
                else if (mode == 3)
                {
                    if (!NeighborOf(f, neighbor, dx, dy, nx, ny)) err = NOT_FOUND;
                }
            }
            bool skip = err != SUCCESS;
            uint32_t k = Reconnection::EMPTY;
            if (err == SUCCESS)
            {
                const zr_rpt_reservoir* src = (mode == 1) ? resPrev : resCurr;
                const int sx = (mode == 1 || mode == 3) ? nx : dx, sy = (mode == 1 || mode == 3) ? ny : dy;
                const uint32_t kk = __ldg(&src[(size_t)sy * f.W + sx].meta) & 0xf;
                k = kk == Reconnection::EMPTY ? kk : kk + 2;
            }
            uint32_t res = err;
            if (k == Reconnection::EMPTY) { res |= EMPTY; skip = true; }
            bool edge = false;
            if (skip && againstEdge && ((uint32_t)dx < f.W) && ((uint32_t)dy < f.H))
            {
                res = SUCCESS; skip = false; edge = true;
            }
            int c = 4;
            if (!skip)
            {
                if (k == 2) c = 0;
                else if (k == 3) c = 1;
                else if (k == 4) c = 2;
                else c = 3;     // k >= 5 or edge case
                (void)edge;
            }
            cls[i] = c;
            result[i] = res;
        }
        auto writeOutput = [&](int dx, int dy, int mgx, int mgy, uint32_t res)
        {
            if ((Gx == dispX - 1) && (Gy != dispY - 1)) { const int t = mgx; mgx = mgy; mgy = t; }
            const int mx = (int)(Gx * 32) + mgx, my = (int)(Gy * 32) + mgy;
            uint32_t error;
            if (mode == 1) error = res & (spatialFlag ? (INVALID_PIXEL | NOT_FOUND) : INVALID_PIXEL);
            else if (mode == 3) error = res & INVALID_PIXEL;
            else error = res & (INVALID_PIXEL | EMPTY);
            if ((uint32_t)mx < f.W && (uint32_t)my < f.H)
            {
                const uint32_t ux = (uint32_t)(dx - mx + 31), uy = (uint32_t)(dy - my + 31);
                threadMap[(size_t)my * f.W + mx] = (uint16_t)(ux | (uy << 7) | ((error > 0 ? 1u : 0u) << 15));
            }
        };
        if (lastGroup)
        {
#pragma unroll
            for (int i = 0; i < 4; i++)
                writeOutput(dxs[i], dys[i], (int)GTx * 2 + (i & 1), (int)GTy * 2 + (i >> 1), result[i]);
            return;
        }
        // 5 counters of 11 bits packed into one 64-bit word, block-wide exclusive scan in thread order
        unsigned long long mine = 0;
#pragma unroll
        for (int i = 0; i < 4; i++) mine += 1ull << (11 * cls[i]);
        unsigned long long incl = mine;
        const uint32_t lane = Gidx & 31, warp = Gidx >> 5;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1)
        {
            const unsigned long long n = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= (uint32_t)off) incl += n;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        unsigned long long warpOff = 0, total = 0;
        for (uint32_t w = 0; w < 8; w++)
        {
            const unsigned long long v = s_warp[w];
            if (w < warp) warpOff += v;
            total += v;
        }
        const unsigned long long excl = warpOff + incl - mine;
        uint32_t base[5];
        uint32_t acc = 0;
#pragma unroll
        for (int c = 0; c < 5; c++) { base[c] = acc; acc += (uint32_t)((total >> (11 * c)) & 0x7ff); }
        uint32_t within[5] = { 0, 0, 0, 0, 0 };
#pragma unroll
        for (int i = 0; i < 4; i++)
        {
            const int c = cls[i];
            const uint32_t rank = base[c] + (uint32_t)((excl >> (11 * c)) & 0x7ff) + within[c];
            within[c]++;
            writeOutput(dxs[i], dys[i], (int)(rank & 31), (int)(rank >> 5), result[i]);
        }
    }

    // -------------------------------------------------------------------------------------------
    // Spatial reuse: Reconnect_CtS + Reconnect_StC for the same pixel, in the StC-sorted thread order
    // -------------------------------------------------------------------------------------------
    // A block is ZR_RPT_THREADS/64 consecutive 8x8 groups of the reference's swizzled dispatch (two waves each).
    __global__ void ZR_LB(ZR_RPT_THREADS) k_spatial(SceneDev sc, FrameView f, RptParams prm, const zr_rpt_reservoir* __restrict__ resIn,
        zr_rpt_reservoir* __restrict__ resOut, const float4* __restrict__ target, float4* __restrict__ finalImg,
        const uint16_t* __restrict__ neighbor, const uint16_t* __restrict__ threadMap, uint32_t dispX, uint32_t dispY,
        const uint32_t* __restrict__ order)
    {
        const zr_frame_constants& fc = f.fc;
        const long long t0 = clock64();
        uint2 sg = make_uint2(0, 0);
        const uint32_t groupFlat = order[blockIdx.x] * (ZR_RPT_THREADS / 64) + (threadIdx.x >> 6);
        const uint32_t tInGroup = threadIdx.x & 63;
        uint2 sp = make_uint2(0xffffffffu, 0xffffffffu);
        if (groupFlat < dispX * dispY)
            sp = SwizzleThreadGroup(groupFlat, 0, tInGroup & 7, tInGroup >> 3, 8, 8, dispX, 16, 4, 16 * dispY, sg);
        bool active = sp.x < f.W && sp.y < f.H;
        int x = (int)sp.x, y = (int)sp.y;
        if (active && prm.sortSpatial)
        {
            const uint16_t enc = __ldg(&threadMap[(size_t)sp.y * f.W + sp.x]);
            if (enc & (1u << 15)) active = false;
            x = (int)sp.x + (int)(enc & 0x3f) - 31;
            y = (int)sp.y + (int)((enc >> 7) & 0x3f) - 31;
        }
        if (active && (y < (int)prm.rowBegin || y >= (int)prm.rowEnd)) active = false;
        size_t idx = 0;
        zr_rpt_reservoir rec;
        Reservoir r_curr = Reservoir::Init();
        Pixel p;
        bool hasN = false;
        int nx = 0, ny = 0;
        if (active)
        {
            const GFlags flags = FlagsAt(f.core, f.W, x, y);
            if (flags.invalid || flags.emissive) active = false;
        }
        if (active)
        {
            idx = (size_t)y * f.W + x;
            p = LoadPixel(f, sc, f.core, f.coat, x, y, false, x, y);
            LoadRecord(&resIn[idx], rec);
            r_curr = Reservoir::Load_NonReconnection(rec);
            const float4 tg = __ldg(&target[idx]);
            r_curr.target = f3(tg.x, tg.y, tg.z);
            hasN = NeighborOf(f, neighbor, x, y, nx, ny);
        }
        const float wsum0 = active ? r_curr.w_sum : 0.0f;
        const float waveSum = WaveSum32(wsum0);
        const float avgEx0 = (waveSum - wsum0) / 32.0f;
        float waveAcc = WaveSum32(active && !hasN ? r_curr.w_sum : 0.0f);
        uint32_t M_max = prm.M_max_spatial;
        M_max = !r_curr.rc.Empty() && r_curr.rc.lobe_k_min_1 == BSDF::GLOSSY_T ? (M_max < 4 ? M_max : 4) : M_max;

        if (active && !hasN)
        {
            if (prm.boilingSuppression) SuppressOutlier(avgEx0, r_curr);
            WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
            CopyToNextFrame(rec, &resOut[idx], r_curr, M_max);
            active = false;
        }
        zr_rpt_reservoir recN;
        Reservoir r_spatial = Reservoir::Init();
        uint32_t M_new = 0;
        {
            // ---- Reconnect_CtS (its result only matters under the StC LoadWSum condition) ----
            bool doCtS = false;
            Reservoir rc_full = Reservoir::Init();
            Pixel pn, pr;
            if (active)
            {
                LoadRecord(&resIn[(size_t)ny * f.W + nx], recN);
                r_spatial = Reservoir::Load_NonReconnection(recN);
                doCtS = (r_curr.w_sum != 0) && !r_curr.rc.Empty() && (r_spatial.M > 0);
            }
            ZR_PHASE();
            if (doCtS)
            {
                rc_full = r_curr;
                rc_full.Load_Reconnection(rec);
                pn = LoadPixel(f, sc, f.core, f.coat, nx, ny, false, x, y);
            }
            const bool needCtx = doCtS && rc_full.rc.k > 2;
            if (needCtx)
                pr = LoadPixel(f, sc, f.core, f.coat, nx, ny, false, nx, ny);
            ZR_PHASE();
            OffsetPathContext ctx = Replay_kGt2_Sync(needCtx, sc, pr.pos, pr.normal, pr.eta_next, pr.surface, rc_full.rc, prm.alpha_min);
            if (needCtx)
                ctx = ctx.Quantize();
            const OffsetPath shift = Shift2_Sync(doCtS, sc, pn.pos, pn.normal, pn.eta_next, pn.surface, rc_full.rc, &ctx, prm.alpha_min);
            if (doCtS)
            {
                const float target_spatial = Math::Luminance(shift.target);
                if (target_spatial > 0)
                {
                    const float targetLum_curr = r_curr.W > 0 ? r_curr.w_sum / r_curr.W : 0;
                    const float jacobian = rc_full.rc.partialJacobian > 0 ? shift.partialJacobian / rc_full.rc.partialJacobian : 0;
                    const float numerator = (float)r_curr.M * targetLum_curr;
                    const float denom = numerator + (float)r_spatial.M * target_spatial * jacobian;
                    const float m_curr = denom > 0 ? numerator / denom : 0;
                    r_curr.w_sum *= m_curr;
                }
            }
            if (active)
                M_new = r_curr.M + r_spatial.M;
        }
        waveAcc += WaveSum32(active && r_spatial.rc.Empty() ? r_curr.w_sum : 0.0f);
        if (active && r_spatial.rc.Empty())
        {
            if (prm.boilingSuppression) SuppressOutlier(avgEx0, r_curr);
            const float targetLum = Math::Luminance(r_curr.target);
            r_curr.W = targetLum > 0 ? r_curr.w_sum / targetLum : 0;
            r_curr.M = M_new;
            CopyToNextFrame(rec, &resOut[idx], r_curr, M_max);
            WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
            active = false;
        }
        bool changed = false;
        if (active)
        {
            M_max = r_spatial.rc.x_k_in_motion ? (M_max < 4 ? M_max : 4) : M_max;
            r_spatial.rc.x_k_in_motion = false;
            r_spatial.Load_Reconnection(recN);
        }
        const bool needCtx = active && r_spatial.rc.k > 2;
        ZR_PHASE();
        OffsetPathContext ctx = Replay_kGt2_Sync(needCtx, sc, p.pos, p.normal, p.eta_next, p.surface, r_spatial.rc, prm.alpha_min);
        if (needCtx)
            ctx = ctx.Quantize();
        const OffsetPath shift = Shift2_Sync(active, sc, p.pos, p.normal, p.eta_next, p.surface, r_spatial.rc, &ctx, prm.alpha_min);
        if (active)
        {
            const float targetLum_curr = Math::Luminance(shift.target);
            const float targetLum_spatial = r_spatial.W > 0 ? r_spatial.w_sum / r_spatial.W : 0;
            const float jacobian = r_spatial.rc.partialJacobian > 0 ? shift.partialJacobian / r_spatial.rc.partialJacobian : 0;
            if (targetLum_curr > 1e-6f && jacobian > 1e-5f && jacobian < 100)
            {
                const uint3 h = RNG::PCG3d(make_uint3((uint32_t)x, (uint32_t)y, (uint32_t)y));
                RNG rng = RNG::Init(h.x, h.z, fc.FrameNum + 511);
                const float numerator = (float)r_spatial.M * targetLum_spatial;
                const float denom = numerator / jacobian + (float)r_curr.M * targetLum_curr;
                const float m_spatial = denom > 0 ? numerator / denom : 0;
                const float w_spatial = m_spatial * r_spatial.W * targetLum_curr;
                if (r_curr.Update(w_spatial, shift.target, r_spatial.rc, rng))
                {
                    r_curr.rc.partialJacobian = shift.partialJacobian;
                    changed = true;
                }
            }
            const float targetLum = Math::Luminance(r_curr.target);
            r_curr.W = targetLum > 0 ? r_curr.w_sum / targetLum : 0;
            r_curr.M = M_new;
        }
        if (prm.boilingSuppression)
        {
            const float total = waveAcc + WaveSum32(active ? r_curr.w_sum : 0.0f);
            if (active)
                SuppressOutlier((total - r_curr.w_sum) / 32.0f, r_curr);
        }
        AccountCost(prm.costMap, f.W, f.H, sp.x, sp.y, t0);
        if (!active)
            return;
        if (changed)
        {
            const uint32_t mmax = shift.surfKMin1Tramsmissive ? (M_max < 4 ? M_max : 4) : M_max;
            zr_rpt_reservoir out;
            r_curr.Write(out, mmax);
            StoreRecord(&resOut[idx], out);
        }
        else
            CopyToNextFrame(rec, &resOut[idx], r_curr, M_max);
        WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
    }

    std::string asset_path2(const char* name)
    {
        Dl_info info;
        std::string dir = ".";
        if (dladdr((void*)&asset_path2, &info) && info.dli_fname)
        {
            std::string p = info.dli_fname;
            size_t s = p.find_last_of('/');
            if (s != std::string::npos) dir = p.substr(0, s);
        }
        return dir + "/assets/" + name;
    }
}
} // namespace zr

// ------------------------------------------------------------------------------------------------
// IndirectLighting pass object (IndirectLighting/IndirectLighting.h:72-108)
// ------------------------------------------------------------------------------------------------
struct zr_indirect_pass
{
    uint32_t width = 0, height = 0;
    zr_rpt_reservoir* d_res[2] = { nullptr, nullptr };
    float4* d_target = nullptr;
    float4* d_final = nullptr;
    uint16_t* d_neighbor = nullptr;
    uint16_t* d_threadMap[2] = { nullptr, nullptr };   // CtN, NtC
    int currTemporalIdx = 0;
    bool isTemporalReservoirValid = false;
    bool resetTemporalTextures = true;
    bool patternLoaded = false;
    // strip-sharded frames (SURVEY 8e): owned rows, halo-exchange hook, optional cost map
    uint32_t rowBegin = 0, rowEnd = 0xffffffffu;
    zr_halo_exchange_fn exchange = nullptr;
    void* exchangeUser = nullptr;
    unsigned long long* d_costMap = nullptr;
    // block schedules (zr_schedule.h), rebuilt when the rows or the tile costs change
    zr::TileCosts tileCosts;
    zr::BlockSchedule schedPathTrace, schedTemporal, schedSpatial;
    // spatial reuse: per-case shift queues + TMA-staged streaming merge (rpt_spatial.cu) by default, the fused kernel on request
    zr::SpatialQueued spatialQueued;
    zr::TemporalQueued temporalQueued;
    zr::WavefrontPT wavefront;
    int execution = ZR_RPT_EXEC_QUEUED;
    zr_status UpdateSchedules()
    {
        const uint32_t y0 = rowBegin, y1 = rowEnd < height ? rowEnd : height, v = tileCosts.version;
        if (!schedPathTrace.UpToDate(y0, y1, v))
            ZR_CUDA(schedPathTrace.Upload(zr::ScheduleSwizzled((width + 15) / 16, (height + 7) / 8, 16, 8, ZR_PT_THREADS / 128, y0, y1, tileCosts), y0, y1, v));
        if (!schedTemporal.UpToDate(y0, y1, v))
            ZR_CUDA(schedTemporal.Upload(zr::ScheduleTiles((width + 31) / 32, (height + ZR_RPT_THREADS / 32 - 1) / (ZR_RPT_THREADS / 32), 32,
                ZR_RPT_THREADS / 32, y0, y1, tileCosts), y0, y1, v));
        if (!schedSpatial.UpToDate(y0, y1, v))
            ZR_CUDA(schedSpatial.Upload(zr::ScheduleSwizzled((width + 7) / 8, (height + 7) / 8, 8, 8, ZR_RPT_THREADS / 64, y0, y1, tileCosts), y0, y1, v));
        return ZR_OK;
    }
    zr_indirect_params params{};

    static void Defaults(zr_indirect_params* p)
    {
        // IndirectLighting.h:231-244, IndirectLighting.cpp:146-165
        p->max_non_tr_bounces = 3; p->max_glossy_tr_bounces = 4; p->russian_roulette = 1; p->temporal_resample = 1;
        p->num_spatial_passes = 1; p->M_max_temporal = 10; p->M_max_spatial = 8; p->boiling_suppression = 1;
        p->sort_temporal = 1; p->sort_spatial = 1; p->alpha_min = 0.175f * 0.175f;
    }

    void Release()
    {
        for (int i = 0; i < 2; i++) { if (d_res[i]) cudaFree(d_res[i]); d_res[i] = nullptr; if (d_threadMap[i]) cudaFree(d_threadMap[i]); d_threadMap[i] = nullptr; }
        schedPathTrace.Release(); schedTemporal.Release(); schedSpatial.Release();
        spatialQueued.Release();
        temporalQueued.Release();
        wavefront.Release();
        if (d_target) cudaFree(d_target); if (d_final) cudaFree(d_final); if (d_neighbor) cudaFree(d_neighbor);
        d_target = d_final = nullptr; d_neighbor = nullptr;
    }

    zr_status OnWindowResized(uint32_t w, uint32_t h)
    {
        Release();
        width = w; height = h;
        const size_t n = (size_t)w * h;
        for (int i = 0; i < 2; i++)
        {
            ZR_CUDA(cudaMalloc(&d_res[i], n * sizeof(zr_rpt_reservoir)));
            ZR_CUDA(cudaMalloc(&d_threadMap[i], n * 2));
        }
        ZR_CUDA(cudaMalloc(&d_target, n * 16));
        ZR_CUDA(cudaMalloc(&d_final, n * 16));
        ZR_CUDA(cudaMalloc(&d_neighbor, n * 2));
        zr_status st = spatialQueued.Resize(w, h, d_res[0], d_res[1]);
        if (st != ZR_OK) return st;
        st = temporalQueued.Resize(w, h);
        if (st != ZR_OK) return st;
        st = wavefront.Resize(w, h);
        if (st != ZR_OK) return st;
        // k_pathtrace's parked state needs more than the 48 KB of static shared memory. The carveout asks for just the shared
        // memory its resident blocks use (plus the 1 KB the system reserves per block); the rest of the 256 KB stays L1 for
        // what still spills.
        ZR_CUDA(cudaFuncSetAttribute(zr::k_pathtrace, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)zr::PT_SMEM_BYTES));
        int ptBlocks = 0;
        ZR_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ptBlocks, zr::k_pathtrace, ZR_PT_THREADS, zr::PT_SMEM_BYTES));
        if (ptBlocks < 1)
        {
            zr::set_error("zr_indirect_pass: k_pathtrace (%d threads, %zu B shared) cannot be resident", ZR_PT_THREADS, zr::PT_SMEM_BYTES);
            return ZR_ERR_UNSUPPORTED;
        }
        const size_t ptSmem = (size_t)ptBlocks * (zr::PT_SMEM_BYTES + 1024);
        ZR_CUDA(cudaFuncSetAttribute(zr::k_pathtrace, cudaFuncAttributePreferredSharedMemoryCarveout,
            (int)((ptSmem * 100 + 228 * 1024 - 1) / (228 * 1024))));
        return ResetTemporal();
    }

    zr_status ResetTemporal()
    {
        const size_t n = (size_t)width * height;
        ZR_CLEAR_BEGIN();
        for (int i = 0; i < 2; i++)
        {
            ZR_CUDA(cudaMemset(d_res[i], 0, n * sizeof(zr_rpt_reservoir)));
            ZR_CUDA(cudaMemset(d_threadMap[i], 0, n * 2));
        }
        ZR_CUDA(cudaMemset(d_target, 0, n * 16));
        ZR_CUDA(cudaMemset(d_final, 0, n * 16));
        ZR_CUDA(cudaMemset(d_neighbor, 0, n * 2));
        ZR_CLEAR_END();
        currTemporalIdx = 0;
        isTemporalReservoirValid = false;
        resetTemporalTextures = true;
        return ZR_OK;
    }

    zr_status LoadPattern()
    {
        if (patternLoaded) return ZR_OK;
        std::vector<float> pat(1024);
        const std::string path = zr::asset_path2("disk512.bin");
        FILE* fp = fopen(path.c_str(), "rb");
        if (!fp || fread(pat.data(), 4, 1024, fp) != 1024)
        {
            if (fp) fclose(fp);
            zr::set_error("zr_indirect_pass: cannot read %s (tools/extract_reference_tables.py writes it)", path.c_str());
            return ZR_ERR_NOT_INITIALIZED;
        }
        fclose(fp);
        ZR_CUDA(cudaMemcpyToSymbol(zr::c_disk512, pat.data(), 4096));
        patternLoaded = true;
        return ZR_OK;
    }

    zr_status Render(const zr_frame_inputs* in, int lastStage, cudaStream_t stream)
    {
        using namespace zr;
        if (!in || !in->scene || !in->curr.d_core || !in->curr.d_motion_emissive || !in->curr.d_coat)
        {
            set_error("zr_indirect_pass_render: missing scene or G-buffer");
            return ZR_ERR_INVALID_ARG;
        }
        if (in->frame.RenderWidth != width || in->frame.RenderHeight != height)
        {
            set_error("zr_indirect_pass_render: frame is %ux%u but the pass was sized %ux%u", in->frame.RenderWidth,
                in->frame.RenderHeight, width, height);
            return ZR_ERR_INVALID_ARG;
        }
        if (in->scene->dev.numEmissives == 0 || !in->scene->aliasBuilt)
        {
            set_error("zr_indirect_pass_render: emissive integrator needs emissive triangles and zr_prelighting_render first "
                "(the sun/sky variant is not part of this build)");
            return ZR_ERR_UNSUPPORTED;
        }
        if (in->scene->dev.sampleSetSize && !in->scene->samplesValid)
        {
            set_error("zr_indirect_pass_render: presampling is enabled but zr_presample_emissives has not run");
            return ZR_ERR_NOT_INITIALIZED;
        }
        zr_status st = LoadPattern();
        if (st != ZR_OK) return st;

        const bool doTemporal = params.temporal_resample && isTemporalReservoirValid;
        const bool doSpatial = (params.num_spatial_passes > 0) && doTemporal;
        if (doTemporal && (!in->prev.d_core || !in->prev.d_coat))
        {
            set_error("zr_indirect_pass_render: temporal reuse needs the previous G-buffer");
            return ZR_ERR_INVALID_ARG;
        }
        FrameView f;
        f.fc = in->frame;
        f.core = (const uint4*)in->curr.d_core; f.depth = (const float*)in->curr.d_depth;
        f.me = (const uint2*)in->curr.d_motion_emissive; f.coat = (const uint2*)in->curr.d_coat;
        f.pcore = (const uint4*)in->prev.d_core; f.pcoat = (const uint2*)in->prev.d_coat;
        f.W = width; f.H = height;
        RptParams prm;
        prm.maxNonTrBounces = params.max_non_tr_bounces; prm.maxGlossyTrBounces = params.max_glossy_tr_bounces;
        prm.russianRoulette = params.russian_roulette; prm.M_max_temporal = params.M_max_temporal; prm.M_max_spatial = params.M_max_spatial;
        prm.boilingSuppression = params.boiling_suppression; prm.sortSpatial = params.sort_spatial; prm.alpha_min = params.alpha_min;
        prm.temporalResample = doTemporal; prm.resetTemporal = resetTemporalTextures; prm.spatialFlag = doSpatial;
        prm.rowBegin = rowBegin; prm.rowEnd = rowEnd < height ? rowEnd : height;
        prm.costMap = d_costMap;
        st = UpdateSchedules();
        if (st != ZR_OK) return st;
        const uint32_t rows = prm.rowEnd - prm.rowBegin;

        int cur = currTemporalIdx;
        if (execution == ZR_RPT_EXEC_WAVEFRONT && !d_costMap)
        {
            st = wavefront.Run(in->scene->dev, f, prm, d_res[cur], d_target, d_final, stream);
            if (st != ZR_OK) return st;
        }
        else
        {
            // the lock-step kernel (also while a cost map is being measured: it accounts the cycles of its blocks per tile)
            const uint32_t dispX = (width + 15) / 16, dispY = (height + 7) / 8;
            ZR_PROF("k_pathtrace", stream);
            k_pathtrace<<<schedPathTrace.count, ZR_PT_THREADS, PT_SMEM_BYTES, stream>>>(in->scene->dev, f, prm, d_res[cur], d_target, d_final, dispX, dispY,
                schedPathTrace.d_order);
            ZR_LAUNCH_CHECK();
        }
        if (doTemporal && lastStage != ZR_RPT_STAGE_PATHTRACE)
        {
            if (execution != ZR_RPT_EXEC_FUSED)
            {
                st = temporalQueued.Run(spatialQueued, in->scene->dev, f, prm, d_res[cur], d_res[1 - cur], d_target, d_final, stream);
                if (st != ZR_OK) return st;
            }
            else
            {
                ZR_PROF("k_temporal", stream);
                k_temporal<<<schedTemporal.count, ZR_RPT_THREADS, 0, stream>>>(in->scene->dev, f, prm, d_res[cur], d_res[1 - cur],
                    d_target, d_final, (width + 31) / 32, schedTemporal.d_order);
                ZR_LAUNCH_CHECK();
            }
        }
        // reservoirs written so far are read by neighbours (spatial pass) and by the next frame's temporal pass
        if (exchange)
        {
            const zr_image2d plane{ d_res[cur], width, height, width * 64u, 64u };
            exchange(exchangeUser, &plane, 1, stream);
        }
        if (doSpatial && lastStage != ZR_RPT_STAGE_PATHTRACE && lastStage != ZR_RPT_STAGE_TEMPORAL)
        {
            for (uint32_t pass = 0; pass < params.num_spatial_passes; pass++)
            {
                ZR_PROF("k_spatial_search", stream);
                k_spatial_search<<<dim3((width + 31) / 32, (rows + 7) / 8), 256, 0, stream>>>(f, prm, d_neighbor);
                ZR_LAUNCH_CHECK();
                zr_rpt_reservoir* rin = d_res[cur];
                zr_rpt_reservoir* rout = d_res[1 - cur];
                cur = 1 - cur;
                if (params.sort_spatial)
                {
                    const uint32_t sx = (width + 31) / 32, sy = (height + 31) / 32;
                    ZR_PROF("k_sort", stream);
                    const uint32_t ty0 = prm.rowBegin / 32, ty1 = (prm.rowEnd + 31) / 32;
                    k_sort<<<dim3(sx, ty1 - ty0), 256, 0, stream>>>(f, 3, 1u, rin, nullptr, d_neighbor, d_threadMap[1], sx, sy, ty0);
                    ZR_LAUNCH_CHECK();
                }
                if (execution != ZR_RPT_EXEC_FUSED)
                {
                    st = spatialQueued.Run(in->scene->dev, f, prm, rin, rout, d_target, d_final, d_neighbor, d_threadMap[1], stream);
                    if (st != ZR_OK) return st;
                }
                else
                {
                    const uint32_t dispX = (width + 7) / 8, dispY = (height + 7) / 8;
                    ZR_PROF("k_spatial", stream);
                    k_spatial<<<schedSpatial.count, ZR_RPT_THREADS, 0, stream>>>(in->scene->dev, f, prm, rin, rout, d_target, d_final, d_neighbor,
                        d_threadMap[1], dispX, dispY, schedSpatial.d_order);
                    ZR_LAUNCH_CHECK();
                }
                if (exchange)
                {
                    const zr_image2d plane{ rout, width, height, width * 64u, 64u };
                    exchange(exchangeUser, &plane, 1, stream);
                }
            }
        }
        isTemporalReservoirValid = true;
        currTemporalIdx = 1 - cur;
        resetTemporalTextures = false;
        return ZR_OK;
    }
};

extern "C"
{
    zr_status zr_indirect_pass_create(uint32_t width, uint32_t height, zr_indirect_pass** out)
    {
        if (!out || !width || !height) { zr::set_error("zr_indirect_pass_create: bad args"); return ZR_ERR_INVALID_ARG; }
        zr_indirect_pass* p = new zr_indirect_pass();
        zr_indirect_pass::Defaults(&p->params);
        if (const char* e = getenv("ZETARAY_B200_SPATIAL"))      // A/B switch for measurements: "fused" | "queued"
            p->execution = std::string(e) == "fused" ? ZR_RPT_EXEC_FUSED : (std::string(e) == "wavefront" ? ZR_RPT_EXEC_WAVEFRONT : ZR_RPT_EXEC_QUEUED);
        zr_status s = p->OnWindowResized(width, height);
        if (s != ZR_OK) { p->Release(); delete p; return s; }
        *out = p;
        return ZR_OK;
    }
    zr_status zr_indirect_pass_resize(zr_indirect_pass* p, uint32_t width, uint32_t height)
    {
        if (!p || !width || !height) return ZR_ERR_INVALID_ARG;
        return p->OnWindowResized(width, height);
    }
    zr_status zr_indirect_pass_reset_temporal(zr_indirect_pass* p) { return p ? p->ResetTemporal() : ZR_ERR_INVALID_ARG; }
    zr_status zr_indirect_pass_default_params(zr_indirect_params* out)
    {
        if (!out) return ZR_ERR_INVALID_ARG;
        zr_indirect_pass::Defaults(out);
        return ZR_OK;
    }
    zr_status zr_indirect_pass_set_params(zr_indirect_pass* p, const zr_indirect_params* params)
    {
        if (!p || !params) return ZR_ERR_INVALID_ARG;
        if (params->max_non_tr_bounces < 1 || params->max_non_tr_bounces > 8 || params->max_glossy_tr_bounces < 1 ||
            params->max_glossy_tr_bounces > 8 || params->M_max_temporal > 15 || params->M_max_spatial > 15 || params->num_spatial_passes > 2)
        {
            zr::set_error("zr_indirect_pass_set_params: value out of range (bounces 1..8, M_max <= 15, spatial passes <= 2)");
            return ZR_ERR_INVALID_ARG;
        }
        p->params = *params;
        return ZR_OK;
    }
    zr_status zr_indirect_pass_render(zr_indirect_pass* p, const zr_frame_inputs* in, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, ZR_RPT_STAGE_ALL, (cudaStream_t)stream);
    }
    zr_status zr_indirect_pass_render_until(zr_indirect_pass* p, const zr_frame_inputs* in, zr_indirect_stage last_stage, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, (int)last_stage, (cudaStream_t)stream);
    }
    zr_status zr_indirect_pass_get_output(zr_indirect_pass* p, zr_indirect_output id, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        const uint32_t w = p->width, h = p->height;
        switch (id)
        {
        case ZR_INDIRECT_FINAL: *out = zr_image2d{ p->d_final, w, h, w * 16u, 16u }; break;
        // after Render() the frame's output reservoirs are the ones the NEXT frame will call "previous"
        case ZR_INDIRECT_RESERVOIR_CURR: *out = zr_image2d{ p->d_res[1 - p->currTemporalIdx], w, h, w * 64u, 64u }; break;
        case ZR_INDIRECT_RESERVOIR_PREV: *out = zr_image2d{ p->d_res[p->currTemporalIdx], w, h, w * 64u, 64u }; break;
        case ZR_INDIRECT_TARGET: *out = zr_image2d{ p->d_target, w, h, w * 16u, 16u }; break;
        case ZR_INDIRECT_NEIGHBOR: *out = zr_image2d{ p->d_neighbor, w, h, w * 2u, 2u }; break;
        case ZR_INDIRECT_THREADMAP_CTN: *out = zr_image2d{ p->d_threadMap[0], w, h, w * 2u, 2u }; break;
        case ZR_INDIRECT_THREADMAP_NTC: *out = zr_image2d{ p->d_threadMap[1], w, h, w * 2u, 2u }; break;
        default: zr::set_error("zr_indirect_pass_get_output: unknown output id"); return ZR_ERR_INVALID_ARG;
        }
        return ZR_OK;
    }
    zr_status zr_indirect_pass_describe_io(zr_indirect_pass* p, zr_resource_use* uses, int* n)
    {
        if (!p || !uses || !n) return ZR_ERR_INVALID_ARG;
        // IndirectLighting reads curr + prev G-buffers, BVH and alias table (PathTracer.cpp:469-547)
        uses[0] = zr_resource_use{ ZR_RES_GBUFFER_CURR, 0 };
        uses[1] = zr_resource_use{ ZR_RES_GBUFFER_PREV, 0 };
        uses[2] = zr_resource_use{ ZR_RES_SCENE_BVH, 0 };
        uses[3] = zr_resource_use{ ZR_RES_ALIAS_TABLE, 0 };
        uses[4] = zr_resource_use{ ZR_RES_INDIRECT_FINAL, 1 };
        *n = 5;
        return ZR_OK;
    }
    zr_status zr_indirect_pass_set_halo_exchange(zr_indirect_pass* p, zr_halo_exchange_fn fn, void* user)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        p->exchange = fn; p->exchangeUser = user;
        return ZR_OK;
    }
    zr_status zr_indirect_pass_set_schedule_costs(zr_indirect_pass* p, const double* h_tile_cost, uint32_t tiles_x, uint32_t tiles_y)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        if (h_tile_cost && (tiles_x != (p->width + 31) / 32 || tiles_y != (p->height + 31) / 32))
        {
            zr::set_error("zr_indirect_pass_set_schedule_costs: expected %u x %u tiles", (p->width + 31) / 32, (p->height + 31) / 32);
            return ZR_ERR_INVALID_ARG;
        }
        p->tileCosts.cost.assign(h_tile_cost ? h_tile_cost : nullptr, h_tile_cost ? h_tile_cost + (size_t)tiles_x * tiles_y : nullptr);
        p->tileCosts.tilesX = h_tile_cost ? tiles_x : 0;
        p->tileCosts.version++;
        return ZR_OK;
    }
    zr_status zr_indirect_pass_set_cost_map(zr_indirect_pass* p, void* d_cycles)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        p->d_costMap = (unsigned long long*)d_cycles;
        return ZR_OK;
    }
    zr_status zr_indirect_pass_set_execution(zr_indirect_pass* p, zr_indirect_execution mode)
    {
        if (!p || (mode != ZR_RPT_EXEC_FUSED && mode != ZR_RPT_EXEC_QUEUED && mode != ZR_RPT_EXEC_WAVEFRONT)) { zr::set_error("zr_indirect_pass_set_execution: bad args"); return ZR_ERR_INVALID_ARG; }
        p->execution = (int)mode;
        return ZR_OK;
    }
    zr_status zr_indirect_pass_set_rows(zr_indirect_pass* p, uint32_t y0, uint32_t y1)
    {
        if (!p || y0 >= y1 || y0 >= p->height) { zr::set_error("zr_indirect_pass_set_rows: empty row range"); return ZR_ERR_INVALID_ARG; }
        p->rowBegin = y0; p->rowEnd = y1;
        return ZR_OK;
    }
    void zr_indirect_pass_destroy(zr_indirect_pass* p) { if (p) { p->Release(); delete p; } }
}
