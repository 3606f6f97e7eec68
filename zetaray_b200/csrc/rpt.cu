// rpt.cu -- ReSTIR PT: path generation, temporal and spatial path reuse, and the IndirectLighting pass.
//
// Replaces IndirectLighting/ReSTIR_PT/*.hlsl (24 compiled variants, IndirectLighting.h:257-289) and the
// host sequencing of IndirectLighting.cpp:370-1025 for the emissive-light integrator.
//
// Dispatch structure (the reference records 1 + 6 + 7 dispatches per frame):
//   k_pathtrace        == ReSTIR_PT_PathTrace           one warp == one reference wave (16x2 pixels of a 16x8
//                                                        group), bounce loop in lock-step so the Russian-roulette
//                                                        wave-max is a warp max
//   temporal reuse     == Sort x2 + Replay x2 + Reconnect_CtT + Reconnect_TtC: classify -> per-case shift queues -> merge
//                         (rpt_temporal.cu). None of them has a wave-scope op, so the sorted thread maps cannot change results.
//   k_spatial_search   == ReSTIR_PT_SpatialSearch
//   k_sort             == ReSTIR_PT_Sort (only the StC map is needed: it defines which 32 pixels share the
//                         boiling-suppression wave sums)
//   spatial reuse      == Replay x2 + Reconnect_CtS + Reconnect_StC: classify -> per-case shift queues -> merge in the
//                         StC-sorted order (rpt_spatial.cu)
// Per-pixel state moves as 128-bit accesses: 64-byte reservoir records, float4 target/final, uint4 G-buffer.
#include "zr_rpt_io.cuh"
#include "zr_rpt_spatial.h"
#include "zr_schedule.h"

namespace zr
{
namespace
{
    using namespace RPT;

    // 512 x float2, indexed per pixel by a random offset: a __constant__ table would serialise the 32 different addresses of a warp
    __device__ __align__(8) float c_disk512[1024];

    // -------------------------------------------------------------------------------------------
    // PathTrace
    // -------------------------------------------------------------------------------------------
// 768 threads at 80 registers with the parked state below (157 KB of shared memory per block). Measured on an H100 SXM (700 W):
// 2.61 ms per bench frame, against 2.60 ms at 640 x 96 registers and 2.68 ms at 512 x 128; 640 threads spill far less but are no
// faster. An earlier sweep, before the traversal rewrite: 3.33 ms, against 3.65 ms at 1024 x 64, 3.52 ms at 512 x 128 and 4.40 ms
// at 512 x 2 blocks x 64 (DESIGN 4.1). Swept before the plain material build existed; both builds use this shape.
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
    // Dynamic shared memory: PT_SMEM_BYTES (PtParked per thread). MF: the material features the kernel is compiled for
    // (BSDF::ShadingDataT); the scene's materials must use no others.
    template<uint32_t MF>
    __global__ void ZR_LB(ZR_PT_THREADS) k_pathtrace(SceneDev sc, FrameView f, RptParams prm, zr_rpt_reservoir* __restrict__ res,
        float4* __restrict__ target, float4* __restrict__ finalImg, uint32_t dispX, uint32_t dispY, const uint32_t* __restrict__ order)
    {
        using SD = BSDF::ShadingDataT<MF>;
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
        SD surface;
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
            const PixelT<SD> p = LoadPixel<SD>(f, sc, f.core, f.coat, px.x, px.y, false, px.x, px.y);
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
                    if (inTranslucentMedium && surface.TrDepthGt0())
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
            bool lightSample = false;
            uint32_t seed_nee = 0;
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
                    SD surfNee = surface;
                    nee = NEE_Emissive_Begin(sc, pos, hitInfo.normal, surfNee, sampleSetIdx, rngThread);
                }
            }
            ZR_PHASE();
            // phase: shadow segment. The segment is set up here rather than carried across the barrier; SetWi leaves
            // Transmissive() as it was, so `surface` answers for the copy NEE_Emissive_Begin shaded with.
            if (lightSample && nee.facing && dot(nee.ld, nee.ld) > 0)
            {
                const RaySetup seg = SetupSegment(pos, nee.ret.wi, nee.t, hitInfo.normal, nee.ret.ID, surface.Transmissive());
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
                    // the shading copy NEE_Emissive_Begin evaluated the light sample with, rebuilt by the same SetWi instead of
                    // carried through the shadow-segment traversal
                    SD surfNee = surface;
                    surfNee.SetWi(nee.ret.wi, hitInfo.normal);
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
    // Debug views (RPT_DEBUG_VIEW, IndirectLighting_Common.h:58-67)
    // -------------------------------------------------------------------------------------------
    // RPT_Util::DebugColor (ReSTIR_PT/Util.hlsli:69-139) of the reconnection packed in a record's meta word, constants as the
    // reference has them (GLOSSY_R is 0.4284 in one lobe view and 0.284 in the other). A record's k is 2..16 or EMPTY and every
    // non-empty reconnection is one of the three cases, so the colour never falls through to the radiance.
    ZR_D float3 DebugColor(uint32_t view, uint32_t meta)
    {
        Reservoir r;
        r.UnpackMetadata(meta);
        const Reconnection& rc = r.rc;
        if (rc.Empty())
            return f3(0);
        if (view == ZR_RPT_DEBUG_VIEW_K)
            return rc.k == 2 ? f3(0.1f, 0.25f, 0.88f) : rc.k == 3 ? f3(0.13f, 0.55f, 0.14f) : rc.k == 4 ? f3(0.69f, 0.45f, 0.1f) :
                f3(0.88f, 0.08f, 0.1f);
        if (view == ZR_RPT_DEBUG_VIEW_CASE)
            return rc.IsCase1() ? f3(0.85f, 0.096f, 0.1f) : rc.IsCase2() ? f3(0.13f, 0.6f, 0.14f) : f3(0.1f, 0.27f, 0.888f);
        if (view == ZR_RPT_DEBUG_VIEW_FOUND_CONNECTION)
            return f3(0.234f, 0.12f, 0.2134f);
        if (view == ZR_RPT_DEBUG_VIEW_CONNECTION_LOBE_K_MIN_1)
        {
            const BSDF::LOBE l = rc.lobe_k_min_1;
            return l == BSDF::DIFFUSE_R ? f3(0.384f, 0.12f, 0.2134f) : l == BSDF::GLOSSY_R ? f3(0.12f, 0.4284f, 0.2134f) :
                l == BSDF::GLOSSY_T ? f3(0.1134f, 0.12f, 0.634f) : l == BSDF::DIFFUSE_T ? f3(0.25f, 0.25f, 0.25f) : f3(0.55f, 0.55f, 0.0f);
        }
        if (rc.IsCase3())
            return f3(0);
        const BSDF::LOBE l = rc.lobe_k;
        return l == BSDF::DIFFUSE_R ? f3(0.384f, 0.12f, 0.2134f) : l == BSDF::GLOSSY_R ? f3(0.12f, 0.284f, 0.2134f) :
            l == BSDF::GLOSSY_T ? f3(0.1134f, 0.12f, 0.634f) : l == BSDF::DIFFUSE_T ? f3(0.25f, 0.25f, 0.0f) : f3(0.25f, 0.25f, 0.25f);
    }

    // The frame's writes of the indirect output, in the reference's order; each is followed by k_rpt_debug_view in a debug frame.
    enum DebugStage : uint32_t { DV_PATHTRACE, DV_TEMPORAL, DV_SPATIAL };

    // Overwrites what one stage (k_pathtrace, k_temporal_merge or one k_spatial_merge) just wrote to FINAL with the debug view, for
    // the pixels that stage wrote. Where the reference colours the output (ReSTIR_PT_PathTrace.hlsl:548, Reconnect_TtC.hlsl:386,
    // Reconnect_StC.hlsl:349) the colour is DebugColor of the reservoir the stage left in resOut; every other write of the stage is
    // WriteOutputColor with the filter on (Util.hlsli:141-160), so black. The branch is recovered from planes the stage leaves:
    //   DV_TEMPORAL  black unless the temporal flag is set and the previous frame's reservoir (resGate) at the reprojected pixel holds
    //                a reconnection
    //   DV_SPATIAL   black unless the pixel has a neighbour and the neighbour's input reservoir (resGate) holds a reconnection; the
    //                pixels are the ones k_spatial_merge visits, thread position (x, y) -> pixel through the StC thread map
    // prevFinal is FINAL as it was before the stage; it is read only where the stage accumulates. The alpha channel is left as the
    // stage wrote it. One thread per pixel of rows [y0, ...): for DV_SPATIAL y0 is the first row of the strip's first 32x32 tile.
    __global__ void __launch_bounds__(256) k_rpt_debug_view(FrameView f, RptParams prm, uint32_t view, uint32_t stage, uint32_t y0,
        const zr_rpt_reservoir* __restrict__ resOut, const zr_rpt_reservoir* __restrict__ resGate, const uint8_t* __restrict__ tflags,
        const uint16_t* __restrict__ neighbor, const uint16_t* __restrict__ threadMap, const float4* __restrict__ prevFinal,
        float4* __restrict__ finalImg)
    {
        const zr_frame_constants& fc = f.fc;
        int x = (int)(blockIdx.x * 32 + (threadIdx.x & 31));
        int y = (int)(y0 + blockIdx.y * 8 + (threadIdx.x >> 5));
        if (x >= (int)f.W || y >= (int)f.H) return;
        if (stage == DV_SPATIAL && prm.sortSpatial)
        {
            const uint32_t enc = __ldg(&threadMap[(size_t)y * f.W + x]);
            if (enc & (1u << 15)) return;
            const int lx = (x & 31) + (int)(enc & 0x3f) - 31, ly = (y & 31) + (int)((enc >> 7) & 0x3f) - 31;
            if ((uint32_t)lx >= 32u || (uint32_t)ly >= 32u) return;
            x = (x & ~31) + lx; y = (y & ~31) + ly;
            if (x >= (int)f.W || y >= (int)f.H) return;
        }
        if (y < (int)prm.rowBegin || y >= (int)prm.rowEnd) return;
        const size_t idx = (size_t)y * f.W + x;
        const GFlags flags = FlagsAt(f.core, f.W, x, y);
        if (flags.invalid || flags.emissive) return;

        bool colour = true;
        if (stage == DV_TEMPORAL)
        {
            int ppx = 0, ppy = 0;
            colour = (__ldg(&tflags[idx]) & TF_OK) != 0;
            if (colour)
            {
                PrevPixel(f, x, y, ppx, ppy);
                colour = (__ldg(&resGate[(size_t)ppy * f.W + ppx].meta) & 0xf) != Reconnection::EMPTY;
            }
        }
        else if (stage == DV_SPATIAL)
        {
            int nx = 0, ny = 0;
            colour = NeighborOf(f, neighbor, x, y, nx, ny) && (__ldg(&resGate[(size_t)ny * f.W + nx].meta) & 0xf) != Reconnection::EMPTY;
        }
        const float3 c = colour ? DebugColor(view, __ldg(&resOut[idx].meta)) : f3(0);
        // the path-trace write accumulates whenever the camera is static, WriteOutputColor from the second static frame on
        const bool accumulate = fc.Accumulate && fc.CameraStatic && (stage == DV_PATHTRACE || fc.NumFramesCameraStatic > 1);
        float4 o = finalImg[idx];
        if (accumulate)
        {
            const float4 prev = prevFinal[idx];
            o.x = prev.x + c.x; o.y = prev.y + c.y; o.z = prev.z + c.z;
        }
        else
        {
            o.x = c.x; o.y = c.y; o.z = c.z;
        }
        finalImg[idx] = o;
    }
}
} // namespace zr

// ------------------------------------------------------------------------------------------------
// IndirectLighting pass object (IndirectLighting/IndirectLighting.h:72-108)
// ------------------------------------------------------------------------------------------------
struct zr_indirect_pass
{
    uint32_t width = 0, height = 0;
    struct Sized
    {
        zr::Planes planes{ "zr_indirect_pass" };
        zr_rpt_reservoir* d_res[2] = { nullptr, nullptr };
        float4* d_target = nullptr;
        float4* d_final = nullptr;
        uint16_t* d_neighbor = nullptr;
        uint16_t* d_threadMap = nullptr;    // NtC
        // temporal and spatial reuse: per-case shift queues + streaming merge (rpt_temporal.cu, rpt_spatial.cu)
        zr::SpatialQueued queued;
    } sz;
    zr::ShiftStreams shiftStreams;
    // Debug view (zr_rpt_debug_view) and what its frames need besides the pass's planes, allocated by the first frame with a view at
    // a size: the reservoirs k_pathtrace writes when temporal reuse is off (it keeps none then), and FINAL before the stage that
    // writes it, where that stage accumulates.
    uint32_t debugView = ZR_RPT_DEBUG_VIEW_NONE;
    struct DebugPlanes
    {
        zr::Planes planes{ "zr_indirect_pass" };
        size_t n = 0;
        zr_rpt_reservoir* d_res = nullptr;
        float4* d_prevFinal = nullptr;
    } dbg;
    int currTemporalIdx = 0;
    bool isTemporalReservoirValid = false;
    bool resetTemporalTextures = true;
    bool patternLoaded = false;
    zr::LightingStrip strip{ "zr_indirect_pass" };  // the block schedule is k_pathtrace's
    zr_indirect_params params = Defaults();

    static zr_indirect_params Defaults()
    {
        // IndirectLighting.h:231-244, IndirectLighting.cpp:146-165
        zr_indirect_params p{};
        p.max_non_tr_bounces = 3; p.max_glossy_tr_bounces = 4; p.russian_roulette = 1; p.temporal_resample = 1;
        p.num_spatial_passes = 1; p.M_max_temporal = 10; p.M_max_spatial = 8; p.boiling_suppression = 1;
        p.sort_temporal = 1; p.sort_spatial = 1; p.alpha_min = 0.175f * 0.175f;
        return p;
    }

    zr_status Setup()
    {
        // k_pathtrace's parked state needs more than the 48 KB of static shared memory. Both material-feature builds are set up,
        // whichever scenes the pass will render.
        decltype(&zr::k_pathtrace<zr::BSDF::MF_ALL>) const kernels[2] = { zr::k_pathtrace<zr::BSDF::MF_NONE>, zr::k_pathtrace<zr::BSDF::MF_ALL> };
        for (const auto kernel : kernels)
            ZR_TRY(zr::ReserveParkedSmem(kernel, ZR_PT_THREADS, zr::PT_SMEM_BYTES, "zr_indirect_pass: k_pathtrace"));
        return shiftStreams.Init();
    }

    zr_status OnWindowResized(uint32_t w, uint32_t h)
    {
        const size_t n = (size_t)w * h;
        Sized next;
        for (int i = 0; i < 2; i++) ZR_TRY(next.planes.Alloc(next.d_res[i], n));
        ZR_TRY(next.planes.Alloc(next.d_threadMap, n));
        ZR_TRY(next.planes.Alloc(next.d_target, n));
        ZR_TRY(next.planes.Alloc(next.d_final, n));
        ZR_TRY(next.planes.Alloc(next.d_neighbor, n));
        ZR_TRY(next.queued.Build(w, h, next.d_res[0], next.d_res[1]));
        ZR_TRY(next.planes.Clear());
        sz = std::move(next);
        width = w; height = h;
        strip.ForgetSize();
        ResetFlags();
        return ZR_OK;
    }

    void ResetFlags() { currTemporalIdx = 0; isTemporalReservoirValid = false; resetTemporalTextures = true; }
    zr_status ResetTemporal()
    {
        ZR_TRY(sz.planes.Clear());
        ResetFlags();
        return ZR_OK;
    }

    zr_status FitDebugPlanes()
    {
        const size_t n = (size_t)width * height;
        if (dbg.n == n) return ZR_OK;
        DebugPlanes next;
        ZR_TRY(next.planes.Alloc(next.d_res, n, false));
        ZR_TRY(next.planes.Alloc(next.d_prevFinal, n, false));
        next.n = n;
        dbg = std::move(next);
        return ZR_OK;
    }

    zr_status LoadPattern()
    {
        if (patternLoaded) return ZR_OK;
        float pat[1024];
        zr_status st = zr::read_asset("zr_indirect_pass", "disk512.bin", pat, sizeof(pat));
        if (st != ZR_OK) return st;
        ZR_CUDA(cudaMemcpyToSymbol(zr::c_disk512, pat, 4096));
        patternLoaded = true;
        return ZR_OK;
    }

    zr_status Render(const zr_frame_inputs* in, cudaStream_t stream)
    {
        using namespace zr;
        FrameView f;
        zr_status st = LightingFrame("zr_indirect_pass", in, width, height, f);
        if (st != ZR_OK) return st;
        st = LoadPattern();
        if (st != ZR_OK) return st;

        const bool doTemporal = params.temporal_resample && isTemporalReservoirValid;
        const bool doSpatial = (params.num_spatial_passes > 0) && doTemporal;
        if (doTemporal && (!in->prev.d_core || !in->prev.d_coat))
        {
            set_error("zr_indirect_pass_render: temporal reuse needs the previous G-buffer");
            return ZR_ERR_INVALID_ARG;
        }
        RptParams prm;
        prm.maxNonTrBounces = params.max_non_tr_bounces; prm.maxGlossyTrBounces = params.max_glossy_tr_bounces;
        prm.russianRoulette = params.russian_roulette; prm.M_max_temporal = params.M_max_temporal; prm.M_max_spatial = params.M_max_spatial;
        prm.boilingSuppression = params.boiling_suppression; prm.sortSpatial = params.sort_spatial; prm.alpha_min = params.alpha_min;
        prm.temporalResample = doTemporal; prm.resetTemporal = resetTemporalTextures; prm.spatialFlag = doSpatial;
        prm.rowBegin = strip.rowBegin; prm.rowEnd = strip.ClampedRowEnd(height);
        prm.costMap = strip.d_costMap;
        st = strip.Schedule(width, height, 16, 8, ZR_PT_THREADS / 128);
        if (st != ZR_OK) return st;
        const uint32_t rows = prm.rowEnd - prm.rowBegin;

        int cur = currTemporalIdx;
        const uint32_t dispX = (width + 15) / 16, dispY = (height + 7) / 8;
        const bool plain = (in->scene->materialFeatures & BSDF::MF_ALL) == 0;

        // Debug frames: each stage that writes FINAL is followed by k_rpt_debug_view over the pixels it wrote. Nothing else changes:
        // a frame without a view launches exactly the kernels above and below.
        const bool view = debugView != ZR_RPT_DEBUG_VIEW_NONE;
        if (view)
        {
            st = FitDebugPlanes();
            if (st != ZR_OK) return st;
        }
        const zr_frame_constants& fc = f.fc;
        const bool accumPathTrace = fc.Accumulate && fc.CameraStatic, accumReuse = accumPathTrace && fc.NumFramesCameraStatic > 1;
        auto snapshot = [&](bool accumulate) -> zr_status
        {
            if (accumulate)
            {
                const size_t first = (size_t)prm.rowBegin * width;
                ZR_CUDA(cudaMemcpyAsync(dbg.d_prevFinal + first, sz.d_final + first, (size_t)rows * width * sizeof(float4),
                    cudaMemcpyDeviceToDevice, stream));
            }
            return ZR_OK;
        };
        auto debugPass = [&](DebugStage stage, const zr_rpt_reservoir* resOut, const zr_rpt_reservoir* resGate) -> zr_status
        {
            const uint32_t y0 = stage == DV_SPATIAL ? prm.rowBegin / 32 * 32 : prm.rowBegin;
            const uint32_t y1 = stage == DV_SPATIAL ? std::min(height, (prm.rowEnd + 31) / 32 * 32) : prm.rowEnd;
            ZR_PROF("k_rpt_debug_view", stream);
            k_rpt_debug_view<<<dim3((width + 31) / 32, (y1 - y0 + 7) / 8), 256, 0, stream>>>(f, prm, debugView, stage, y0, resOut, resGate,
                sz.queued.d_flags, sz.d_neighbor, sz.d_threadMap, dbg.d_prevFinal, sz.d_final);
            ZR_LAUNCH_CHECK();
            return ZR_OK;
        };

        // With temporal reuse off k_pathtrace writes no reservoir after the first frame; a debug frame has it write them to a plane of
        // its own, so the pass's reservoirs stay as they would be without the view.
        zr_rpt_reservoir* ptRes = sz.d_res[cur];
        RptParams ptPrm = prm;
        if (view && !doTemporal)
        {
            if (!prm.resetTemporal)
            {
                ptRes = dbg.d_res;
                ptPrm.resetTemporal = 1;
            }
            ZR_TRY(snapshot(accumPathTrace));
        }
        ZR_PROF("k_pathtrace", stream);
        (plain ? k_pathtrace<BSDF::MF_NONE> : k_pathtrace<BSDF::MF_ALL>)<<<strip.sched[0].count, ZR_PT_THREADS, PT_SMEM_BYTES, stream>>>(in->scene->dev, f, ptPrm, ptRes, sz.d_target, sz.d_final, dispX, dispY,
            strip.sched[0].d_order);
        ZR_LAUNCH_CHECK();
        if (view && !doTemporal)
            ZR_TRY(debugPass(DV_PATHTRACE, ptRes, nullptr));
        if (doTemporal)
        {
            const bool temporalWrites = view && !doSpatial;
            if (temporalWrites)
                ZR_TRY(snapshot(accumReuse));
            st = sz.queued.RunTemporal(shiftStreams, in->scene->dev, f, prm, sz.d_res[cur], sz.d_res[1 - cur], sz.d_target, sz.d_final, plain, stream);
            if (st != ZR_OK) return st;
            if (temporalWrites)
                ZR_TRY(debugPass(DV_TEMPORAL, sz.d_res[cur], sz.d_res[1 - cur]));
        }
        // reservoirs written so far are read by neighbours (spatial pass) and by the next frame's temporal pass
        strip.Exchange(sz.d_res[cur], width, height, 64u, stream);
        if (doSpatial)
        {
            for (uint32_t pass = 0; pass < params.num_spatial_passes; pass++)
            {
                ZR_PROF("k_spatial_search", stream);
                k_spatial_search<<<dim3((width + 31) / 32, (rows + 7) / 8), 256, 0, stream>>>(f, prm, sz.d_neighbor);
                ZR_LAUNCH_CHECK();
                zr_rpt_reservoir* rin = sz.d_res[cur];
                zr_rpt_reservoir* rout = sz.d_res[1 - cur];
                cur = 1 - cur;
                if (params.sort_spatial)
                {
                    const uint32_t sx = (width + 31) / 32, sy = (height + 31) / 32;
                    ZR_PROF("k_sort", stream);
                    const uint32_t ty0 = prm.rowBegin / 32, ty1 = (prm.rowEnd + 31) / 32;
                    k_sort<<<dim3(sx, ty1 - ty0), 256, 0, stream>>>(f, 3, 1u, rin, nullptr, sz.d_neighbor, sz.d_threadMap, sx, sy, ty0);
                    ZR_LAUNCH_CHECK();
                }
                if (view)
                    ZR_TRY(snapshot(accumReuse));
                st = sz.queued.Run(shiftStreams, in->scene->dev, f, prm, rin, rout, sz.d_target, sz.d_final, sz.d_neighbor, sz.d_threadMap, plain, stream);
                if (st != ZR_OK) return st;
                if (view)
                    ZR_TRY(debugPass(DV_SPATIAL, rout, rin));
                strip.Exchange(rout, width, height, 64u, stream);
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
    zr_status zr_indirect_pass_create(uint32_t width, uint32_t height, zr_indirect_pass** out) { return zr::CreatePass("zr_indirect_pass", width, height, out); }
    zr_status zr_indirect_pass_resize(zr_indirect_pass* p, uint32_t width, uint32_t height) { return zr::ResizePass("zr_indirect_pass", p, width, height); }
    zr_status zr_indirect_pass_reset_temporal(zr_indirect_pass* p) { return zr::ResetPass(p); }
    zr_status zr_indirect_pass_default_params(zr_indirect_params* out) { return zr::DefaultParams<zr_indirect_pass>(out); }
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
    zr_status zr_indirect_pass_set_debug_view(zr_indirect_pass* p, uint32_t view)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        if (view > ZR_RPT_DEBUG_VIEW_CONNECTION_LOBE_K)
        {
            zr::set_error("zr_indirect_pass_set_debug_view: view %u out of range (0..%u)", view, (uint32_t)ZR_RPT_DEBUG_VIEW_CONNECTION_LOBE_K);
            return ZR_ERR_INVALID_ARG;
        }
        p->debugView = view;
        if (view == ZR_RPT_DEBUG_VIEW_NONE)
            p->dbg = zr_indirect_pass::DebugPlanes();       // frees them
        return ZR_OK;
    }
    zr_status zr_indirect_pass_render(zr_indirect_pass* p, const zr_frame_inputs* in, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, (cudaStream_t)stream);
    }
    zr_status zr_indirect_pass_get_output(zr_indirect_pass* p, zr_indirect_output id, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        const uint32_t w = p->width, h = p->height;
        switch (id)
        {
        case ZR_INDIRECT_FINAL: *out = zr_image2d{ p->sz.d_final, w, h, w * 16u, 16u }; break;
        // after Render() the frame's output reservoirs are the ones the NEXT frame will call "previous"
        case ZR_INDIRECT_RESERVOIR_CURR: *out = zr_image2d{ p->sz.d_res[1 - p->currTemporalIdx], w, h, w * 64u, 64u }; break;
        case ZR_INDIRECT_RESERVOIR_PREV: *out = zr_image2d{ p->sz.d_res[p->currTemporalIdx], w, h, w * 64u, 64u }; break;
        case ZR_INDIRECT_TARGET: *out = zr_image2d{ p->sz.d_target, w, h, w * 16u, 16u }; break;
        case ZR_INDIRECT_NEIGHBOR: *out = zr_image2d{ p->sz.d_neighbor, w, h, w * 2u, 2u }; break;
        case ZR_INDIRECT_THREADMAP_NTC: *out = zr_image2d{ p->sz.d_threadMap, w, h, w * 2u, 2u }; break;
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
    zr_status zr_indirect_pass_set_halo_exchange(zr_indirect_pass* p, zr_halo_exchange_fn fn, void* user) { return p ? p->strip.SetHaloExchange(fn, user) : ZR_ERR_INVALID_ARG; }
    zr_status zr_indirect_pass_set_schedule_costs(zr_indirect_pass* p, const double* h_tile_cost, uint32_t tiles_x, uint32_t tiles_y)
    {
        return p ? p->strip.SetScheduleCosts(h_tile_cost, tiles_x, tiles_y, p->width, p->height) : ZR_ERR_INVALID_ARG;
    }
    zr_status zr_indirect_pass_set_cost_map(zr_indirect_pass* p, void* d_cycles) { return p ? p->strip.SetCostMap(d_cycles) : ZR_ERR_INVALID_ARG; }
    zr_status zr_indirect_pass_set_rows(zr_indirect_pass* p, uint32_t y0, uint32_t y1) { return p ? p->strip.SetRows(y0, y1, p->height) : ZR_ERR_INVALID_ARG; }
    void zr_indirect_pass_destroy(zr_indirect_pass* p) { delete p; }
}
