// rpt_wavefront.cu -- ReSTIR PT path generation (ReSTIR_PT_PathTrace.hlsl:227-355, 360-540) as a WAVEFRONT: one kernel launch per
// bounce over a compacted queue of the paths that are still alive, instead of k_pathtrace's lock-step bounce loop (rpt.cu) in which
// a path that has left the scene keeps its lane until the last path of its 1024-pixel block ends (ncu: 11 of 32 lanes active on the
// Cornell frame, 9 on the tunnel). Same bytes as k_pathtrace and the oracle.
//
//   k_pt_begin      per pixel: G-buffer -> first vertex, first BSDF sample, its closest-hit query; pixels whose path cannot start
//                   are finished on the spot, the others go to queue 0
//   k_pt_bounce     persistent blocks (512 threads x 2 per SM) claim 512 paths at a time: [end-of-bounce step of the previous bounce]
//                   -> hit attributes + material | next BSDF sample | closest hit | light sample + BSDF value | shadow segment |
//                   sampler pdf, MIS, reservoir update -- the block-synchronous phases of zr_rpt.cuh, every lane on a live path.
//                   Survivors are appended to the other queue, finished paths write reservoir / target / colour.
// Path state (PtState, 448 bytes) stays at its pixel's slot between launches; only the 4-byte queue entries are compacted.
//
// The one wave-scope operation of the reference shader, Russian roulette against the WAVE's maximum throughput
// (ReSTIR_PT_PathTrace.hlsl:295-308, bounces >= 3), falls on a launch boundary: a path that reaches the roulette publishes its
// throughput with an atomic max into the slot of its reference wave (16 x 2 pixels), and the next launch starts with the roulette
// step, reading the slot. A maximum does not depend on the order of its operands, so the result is the lock-step one.
#include "zr_rpt_spatial.h"
#include "zr_rpt_shift.cuh"

namespace zr
{
namespace
{
    using namespace RPT;

    struct PtState
    {
        float3 pos, normal, li, throughput, throughput_k, tr;
        // the BSDF sample leaving `pos` and what it hit
        float3 wi, bsdfOverPdf; float pdf; uint32_t lobe;
        float hit_t; uint32_t hit_geo, hit_prim; float2 hit_bary; uint32_t hit_flag;
        PrevHit prevHit;
        float eta_curr, eta_next;
        int bounce, maxNumBounces;
        uint32_t rngReplay, rngThread, rngGroup, sampleSetIdx, seedReplay0;
        uint32_t inMedium, pendingStep;
        // inputs of the end-of-bounce step (roulette, SetCase1, throughput update) that belong to the vertex just shaded
        float alpha_lobe; float3 wo; float cur_t; uint32_t curID, curMesh; uint32_t prevSampleLobe; float prevSamplePdf;
        Reconnection rc;
        Reservoir r;
    };
    constexpr int PT_STATE_BYTES = 448;
    // block size of the path-generation kernels: like k_pathtrace, 1024 threads x 1 block per SM
    constexpr int WF_THREADS = 1024, WF_MINBLOCKS = 1;
    static_assert(sizeof(PtState) <= PT_STATE_BYTES, "PtState outgrew its slot");

    // order-preserving key of a float for atomicMax on unsigned; 0 = "no operand yet" (below every float)
    ZR_D uint32_t MaxKey(float f) { const uint32_t u = asuint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
    ZR_D float MaxKeyDecode(uint32_t k) { return k == 0 ? -FLT_MAX_ : asfloat((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

    struct PtOut { zr_rpt_reservoir* res; float4* target; float4* finalImg; };

    // what k_pathtrace does after its loop (ReSTIR_PT_PathTrace.hlsl:527-540)
    ZR_D void FinishPath(const zr_frame_constants& fc, const RptParams& prm, const PtOut& o, size_t idx, Reservoir& r, float3 li, uint32_t seedReplay0)
    {
        r.rc.seed_replay = seedReplay0;
        const float targetLum = Math::Luminance(r.target);
        r.W = targetLum > 0 ? fmaxf(r.w_sum / targetLum, 1.0f) : 0;
        if (prm.temporalResample || prm.resetTemporal)
        {
            zr_rpt_reservoir rec;
            r.Write(rec, 0);
            StoreRecord(&o.res[idx], rec);
        }
        if (prm.temporalResample)
        {
            r.target = Math::Sanitize(r.target);
            o.target[idx] = f4(r.target.x, r.target.y, r.target.z, 0.0f);
        }
        else
        {
            li = isnan3(li) ? f3(0) : li;
            if (fc.Accumulate && fc.CameraStatic)
            {
                const float4 prev = o.finalImg[idx];
                o.finalImg[idx] = f4(prev.x + li.x, prev.y + li.y, prev.z + li.z, prev.w);
            }
            else
                o.finalImg[idx] = f4(li.x, li.y, li.z, 0.0f);
        }
    }

    // block-aggregated append of at most one entry per thread to a single queue (all threads of the block call it)
    ZR_D void AppendOne(bool have, uint32_t item, uint32_t* __restrict__ queue, uint32_t* __restrict__ counter, uint32_t* s_count, uint32_t* s_base)
    {
        const uint32_t lane = threadIdx.x & 31;
        if (threadIdx.x == 0) *s_count = 0;
        __syncthreads();
        const uint32_t m = __ballot_sync(0xffffffffu, have);
        uint32_t base = 0;
        if (m && lane == 0) base = atomicAdd(s_count, __popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        const uint32_t off = base + __popc(m & ((1u << lane) - 1));
        __syncthreads();
        if (threadIdx.x == 0) *s_base = *s_count ? atomicAdd(counter, *s_count) : 0;
        __syncthreads();
        if (have) queue[*s_base + off] = item;
    }

    // -----------------------------------------------------------------------------------------------------------------
    // first vertex (everything k_pathtrace does before its loop)
    // -----------------------------------------------------------------------------------------------------------------
    __global__ void __launch_bounds__(WF_THREADS, WF_MINBLOCKS) k_pt_begin(SceneDev sc, FrameView f, RptParams prm, PtOut out,
        unsigned char* __restrict__ states, uint32_t* __restrict__ queue, uint32_t* __restrict__ counter)
    {
        __shared__ uint32_t s_count, s_base;
        const zr_frame_constants& fc = f.fc;
        const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31);
        const uint32_t y = prm.rowBegin + blockIdx.y * (WF_THREADS / 32) + (threadIdx.x >> 5);
        bool inBounds = x < f.W && y < f.H && y < prm.rowEnd;
        const size_t idx = inBounds ? (size_t)y * f.W + x : 0;
        if (inBounds)
        {
            const GFlags flags = FlagsAt(f.core, f.W, (int)x, (int)y);
            if (flags.invalid || flags.emissive)
            {
                if (!fc.Accumulate || !fc.CameraStatic)
                    out.finalImg[idx] = f4(0, 0, 0, 0);
                inBounds = false;
            }
        }
        PtState st;
        bool alive = false;
        BSDF::BSDFSample bsdfSample = BSDF::BSDFSample::Init();
        BSDF::ShadingData surface;
        if (inBounds)
        {
            st.pos = f3(0); st.normal = f3(0); st.li = f3(0); st.throughput = f3(0); st.throughput_k = f3(1); st.tr = f3(1);
            st.rc = Reconnection::Init();
            st.r = Reservoir::Init();
            st.prevHit.alpha_lobe = 0; st.prevHit.wi = f3(0); st.prevHit.pdf = 0; st.prevHit.lobe = BSDF::DIFFUSE_R;
            st.eta_curr = BSDF::ETA_AIR; st.eta_next = BSDF::DEFAULT_ETA_MAT;
            st.inMedium = 0; st.bounce = 0; st.pendingStep = 0;
            st.hit_flag = 0; st.hit_t = 0; st.hit_geo = 0; st.hit_prim = 0; st.hit_bary = f2(0, 0);
            st.alpha_lobe = 0; st.wo = f3(0); st.cur_t = 0; st.curID = 0; st.curMesh = 0; st.prevSampleLobe = 0; st.prevSamplePdf = 0;
            st.sampleSetIdx = 0;
            const Pixel p = LoadPixel(f, sc, f.core, f.coat, (int)x, (int)y, false, (int)x, (int)y);
            // the reference's group / wave of this pixel: 16 x 8 thread groups, swizzled group id == the group's tile coordinates
            RNG rngGroup = RNG::Init4(x / 16, y / 8, fc.FrameNum, 1);
            const uint3 state = RNG::PCG3d(make_uint3(x, y, fc.FrameNum));
            RNG rngReplay = RNG::InitSeed(state.x);
            st.rngThread = state.y;             // RNG::InitSeed(state.y).State
            st.seedReplay0 = state.x;
            st.maxNumBounces = (int)(p.surface.specTr ? prm.maxGlossyTrBounces : prm.maxNonTrBounces);
            bsdfSample = BSDF::SampleBSDF(p.normal, p.surface, rngReplay);
            if (dot(bsdfSample.bsdfOverPdf, bsdfSample.bsdfOverPdf) != 0)
            {
                st.sampleSetIdx = rngGroup.UniformUintBounded_Faster(sc.numSampleSets);
                st.pos = p.pos; st.normal = p.normal; surface = p.surface;
                st.throughput = bsdfSample.bsdfOverPdf;
                st.prevHit.alpha_lobe = BSDF::LobeAlpha(p.surface, bsdfSample.lobe);
                st.prevHit.lobe = bsdfSample.lobe; st.prevHit.wi = bsdfSample.wi; st.prevHit.pdf = bsdfSample.pdf;
                st.eta_curr = dot(p.normal, bsdfSample.wi) < 0 ? p.eta_next : BSDF::ETA_AIR;
                st.inMedium = st.eta_curr != BSDF::ETA_AIR ? 1u : 0u;
                alive = true;
            }
            st.rngReplay = rngReplay.State;
            st.rngGroup = rngGroup.State;
        }
        ZR_PHASE();
        if (alive)
        {
            const HitEmissive nextHit = FindClosestEmissive(sc, st.pos, st.normal, bsdfSample.wi, surface.Transmissive());
            st.hit_flag = nextHit.hit ? 1u : 0u; st.hit_t = nextHit.t; st.hit_geo = nextHit.geoIdx; st.hit_prim = nextHit.primIdx; st.hit_bary = nextHit.bary;
            st.wi = bsdfSample.wi; st.bsdfOverPdf = bsdfSample.bsdfOverPdf; st.pdf = bsdfSample.pdf; st.lobe = (uint32_t)bsdfSample.lobe;
            *reinterpret_cast<PtState*>(states + idx * PT_STATE_BYTES) = st;
        }
        else if (inBounds)
            FinishPath(fc, prm, out, idx, st.r, st.li, st.seedReplay0);
        AppendOne(alive, x | (y << 16), queue, counter, &s_count, &s_base);
    }

    // -----------------------------------------------------------------------------------------------------------------
    // one bounce
    // -----------------------------------------------------------------------------------------------------------------
    __global__ void __launch_bounds__(WF_THREADS, WF_MINBLOCKS) k_pt_bounce(SceneDev sc, FrameView f, RptParams prm, PtOut out,
        unsigned char* __restrict__ states, const uint32_t* __restrict__ queueIn, uint32_t* __restrict__ queueOut, uint32_t* __restrict__ counters,
        uint32_t slotIn, uint32_t slotOut, const uint32_t* __restrict__ waveMaxIn, uint32_t* __restrict__ waveMaxOut, uint32_t wavesX)
    {
        __shared__ uint32_t s_claim, s_count, s_base;
        const zr_frame_constants& fc = f.fc;
        const uint32_t total = counters[slotIn];
        for (;;)
        {
            __syncthreads();
            if (threadIdx.x == 0) s_claim = atomicAdd(&counters[8 + slotIn], (uint32_t)WF_THREADS);
            __syncthreads();
            const uint32_t base = s_claim;
            if (base >= total) break;
            bool alive = base + threadIdx.x < total;
            uint32_t item = 0, x = 0, y = 0;
            size_t idx = 0;
            const bool wasQueued = alive;
            // loop-carried state of k_pathtrace, read field by field from the path's slot (no staging copy of the 448-byte record)
            float3 pos = f3(0), li = f3(0), throughput = f3(0), throughput_k = f3(1), tr = f3(1);
            BSDF::BSDFSample bsdfSample = BSDF::BSDFSample::Init();
            HitEmissive nextHit; nextHit.hit = false; nextHit.t = 0; nextHit.geoIdx = 0; nextHit.primIdx = 0; nextHit.bary = f2(0, 0);
            nextHit.emissiveTriIdx = UINT32_MAX_; nextHit.lightPos = f3(0);
            Reconnection rc = Reconnection::Init();
            Reservoir r = Reservoir::Init();
            PrevHit prevHit; prevHit.alpha_lobe = 0; prevHit.wi = f3(0); prevHit.pdf = 0; prevHit.lobe = BSDF::DIFFUSE_R;
            float eta_curr = BSDF::ETA_AIR, eta_next = BSDF::DEFAULT_ETA_MAT;
            bool inTranslucentMedium = false;
            int bounce = 0, maxNumBounces = 0;
            uint32_t sampleSetIdx = 0, seedReplay0 = 0;
            RNG rngReplay, rngThread, rngGroup;
            rngReplay.State = 0; rngThread.State = 0; rngGroup.State = 0;
            PtState* gp = nullptr;
            if (alive)
            {
                item = __ldg(&queueIn[base + threadIdx.x]);
                x = item & 0xffff; y = item >> 16;
                idx = (size_t)y * f.W + x;
                gp = reinterpret_cast<PtState*>(states + idx * PT_STATE_BYTES);
                pos = gp->pos; li = gp->li; throughput = gp->throughput; throughput_k = gp->throughput_k; tr = gp->tr;
                bsdfSample.wi = gp->wi; bsdfSample.bsdfOverPdf = gp->bsdfOverPdf; bsdfSample.pdf = gp->pdf; bsdfSample.lobe = (BSDF::LOBE)gp->lobe;
                nextHit.hit = gp->hit_flag != 0; nextHit.t = gp->hit_t; nextHit.geoIdx = gp->hit_geo; nextHit.primIdx = gp->hit_prim; nextHit.bary = gp->hit_bary;
                rc = gp->rc; r = gp->r; prevHit = gp->prevHit;
                eta_curr = gp->eta_curr; eta_next = gp->eta_next; inTranslucentMedium = gp->inMedium != 0;
                bounce = gp->bounce; maxNumBounces = gp->maxNumBounces; sampleSetIdx = gp->sampleSetIdx; seedReplay0 = gp->seedReplay0;
                rngReplay.State = gp->rngReplay; rngThread.State = gp->rngThread; rngGroup.State = gp->rngGroup;
            }
            // ---- end-of-bounce step of the previous bounce (ReSTIR_PT_PathTrace.hlsl:295-355): roulette against the wave maximum,
            //      SetCase1, throughput / medium / previous-hit update ----
            if (alive && gp->pendingStep)
            {
                const bool doRR = prm.russianRoulette && (bounce >= 3);
                do
                {
                    if (doRR)
                    {
                        const float waveThroughput = MaxKeyDecode(__ldg(&waveMaxIn[(y >> 1) * wavesX + (x >> 4)]));
                        if (waveThroughput < 1)
                        {
                            const float p_terminate = fmaxf(0.05f, 1 - waveThroughput);
                            if (rngGroup.Uniform() < p_terminate) { alive = false; break; }
                            throughput /= (1 - p_terminate);
                            throughput_k /= ((int)rc.k <= bounce) ? (1 - p_terminate) : 1.0f;
                        }
                    }
                    if (dot(bsdfSample.bsdfOverPdf, bsdfSample.bsdfOverPdf) == 0) { alive = false; break; }
                    const float alpha_lobe = gp->alpha_lobe;
                    const float3 normalPrev = gp->normal;
                    if (rc.Empty() && CanReconnect(prevHit.alpha_lobe, alpha_lobe, prevHit.lobe, bsdfSample.lobe, prm.alpha_min))
                    {
                        rc.SetCase1(bounce + 1, pos, gp->cur_t, normalPrev, gp->curID, gp->curMesh, -gp->wo,
                            (BSDF::LOBE)gp->prevSampleLobe, gp->prevSamplePdf, bsdfSample.wi, bsdfSample.lobe, bsdfSample.pdf);
                        throughput_k = f3(1);
                    }
                    if ((int)rc.k <= bounce)
                        throughput_k *= bsdfSample.bsdfOverPdf * tr;
                    const bool transmitted = dot(normalPrev, bsdfSample.wi) < 0;
                    throughput *= bsdfSample.bsdfOverPdf;
                    eta_curr = transmitted ? (eta_curr == BSDF::ETA_AIR ? eta_next : BSDF::ETA_AIR) : eta_curr;
                    inTranslucentMedium = eta_curr != BSDF::ETA_AIR;
                    prevHit.alpha_lobe = alpha_lobe;
                    prevHit.lobe = bsdfSample.lobe;
                    prevHit.wi = bsdfSample.wi;
                    prevHit.pdf = bsdfSample.pdf;
                } while (false);
            }
            BSDF::ShadingData surface;
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
            // phase: draw the next direction (NEE_Bsdf, ReSTIR_PT_NEE.hlsli:145-222)
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
            bool atRR = false;
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
            // the wave-wide maximum of the roulette is taken over the paths that reach it at this bounce
            if (atRR && prm.russianRoulette && bounce >= 3)
            {
                const float lum = Math::Luminance(throughput);
                if (lum == lum)         // fmaxf ignores NaN operands
                    atomicMax(&waveMaxOut[(y >> 1) * wavesX + (x >> 4)], MaxKey(lum));
            }
            if (alive)
            {
                gp->pos = pos; gp->normal = hitInfo.normal; gp->li = li; gp->throughput = throughput; gp->throughput_k = throughput_k; gp->tr = tr;
                gp->wi = bsdfSample.wi; gp->bsdfOverPdf = bsdfSample.bsdfOverPdf; gp->pdf = bsdfSample.pdf; gp->lobe = (uint32_t)bsdfSample.lobe;
                gp->hit_flag = nextHit.hit ? 1u : 0u; gp->hit_t = nextHit.t; gp->hit_geo = nextHit.geoIdx; gp->hit_prim = nextHit.primIdx; gp->hit_bary = nextHit.bary;
                gp->prevHit = prevHit; gp->eta_curr = eta_curr; gp->eta_next = eta_next; gp->inMedium = inTranslucentMedium ? 1u : 0u;
                gp->bounce = bounce; gp->rngReplay = rngReplay.State; gp->rngThread = rngThread.State; gp->rngGroup = rngGroup.State;
                gp->pendingStep = 1;
                gp->alpha_lobe = BSDF::LobeAlpha(surface, bsdfSample.lobe);
                gp->wo = surface.wo; gp->cur_t = hitInfo.t; gp->curID = hitInfo.ID; gp->curMesh = hitInfo.meshIdx;
                gp->prevSampleLobe = (uint32_t)prevBsdfSampleLobe; gp->prevSamplePdf = prevBsdfSamplePdf;
                gp->rc = rc; gp->r = r;
            }
            else if (wasQueued)
                FinishPath(fc, prm, out, idx, r, li, seedReplay0);
            AppendOne(alive, item, queueOut, &counters[slotOut], &s_count, &s_base);
        }
    }
}

// -------------------------------------------------------------------------------------------------------------------
void WavefrontPT::Release()
{
    if (d_states) cudaFree(d_states);
    if (d_queue[0]) cudaFree(d_queue[0]);
    if (d_queue[1]) cudaFree(d_queue[1]);
    if (d_counters) cudaFree(d_counters);
    if (d_waveMax[0]) cudaFree(d_waveMax[0]);
    if (d_waveMax[1]) cudaFree(d_waveMax[1]);
    d_states = nullptr; d_queue[0] = d_queue[1] = nullptr; d_counters = nullptr; d_waveMax[0] = d_waveMax[1] = nullptr;
}

zr_status WavefrontPT::Resize(uint32_t w, uint32_t h)
{
    Release();
    width = w; height = h;
    wavesX = (w + 15) / 16;
    numWaves = (size_t)wavesX * ((h + 1) / 2);
    return ZR_OK;       // 448 bytes of state per pixel: allocated when the mode is first used
}

zr_status WavefrontPT::Allocate()
{
    const size_t n = (size_t)width * height;
    ZR_CUDA(cudaMalloc(&d_states, n * PT_STATE_BYTES));
    ZR_CUDA(cudaMalloc(&d_queue[0], n * 4));
    ZR_CUDA(cudaMalloc(&d_queue[1], n * 4));
    ZR_CUDA(cudaMalloc(&d_counters, 16 * sizeof(uint32_t)));
    ZR_CUDA(cudaMalloc(&d_waveMax[0], numWaves * 4));
    ZR_CUDA(cudaMalloc(&d_waveMax[1], numWaves * 4));
    int dev = 0;
    ZR_CUDA(cudaGetDevice(&dev));
    ZR_CUDA(cudaDeviceGetAttribute(&numSMs, cudaDevAttrMultiProcessorCount, dev));
    return ZR_OK;
}

zr_status WavefrontPT::Run(const SceneDev& sc, const FrameView& f, const RptParams& prm, zr_rpt_reservoir* res, float4* target, float4* finalImg,
    cudaStream_t stream)
{
    if (!width) { set_error("zr_indirect_pass: wavefront path generation is not initialised"); return ZR_ERR_NOT_INITIALIZED; }
    if (!d_states)
    {
        const zr_status st = Allocate();
        if (st != ZR_OK) return st;
    }
    const PtOut out{ res, target, finalImg };
    const uint32_t rows = prm.rowEnd - prm.rowBegin;
    // counters: [0], [1] = entries in queue 0 / 1; [8], [9] = claim cursors
    ZR_CUDA(cudaMemsetAsync(d_counters, 0, 16 * sizeof(uint32_t), stream));
    {
        ZR_PROF("k_pt_begin", stream);
        k_pt_begin<<<dim3((width + 31) / 32, (rows + WF_THREADS / 32 - 1) / (WF_THREADS / 32)), WF_THREADS, 0, stream>>>(sc, f, prm, out, d_states,
            d_queue[0], d_counters + 0);
        ZR_LAUNCH_CHECK();
    }
    const uint32_t maxBounces = prm.maxNonTrBounces > prm.maxGlossyTrBounces ? prm.maxNonTrBounces : prm.maxGlossyTrBounces;
    const uint32_t grid = (uint32_t)numSMs * WF_MINBLOCKS;
    ZR_PROF("k_pt_bounce", stream);
    for (uint32_t i = 0; i < maxBounces; i++)
    {
        const uint32_t in = i & 1, outSlot = (i + 1) & 1;
        // the queue this launch fills and its cursor start empty; the wave-maximum slots it publishes to as well
        ZR_CUDA(cudaMemsetAsync(d_counters + outSlot, 0, 4, stream));
        ZR_CUDA(cudaMemsetAsync(d_counters + 8 + outSlot, 0, 4, stream));
        const bool rrPossible = prm.russianRoulette && (i + 1 >= 3);        // paths that continue leave launch i with bounce == i + 1
        if (rrPossible)
            ZR_CUDA(cudaMemsetAsync(d_waveMax[in], 0, numWaves * 4, stream));
        k_pt_bounce<<<grid, WF_THREADS, 0, stream>>>(sc, f, prm, out, d_states, d_queue[in], d_queue[outSlot], d_counters, in, outSlot,
            d_waveMax[outSlot], d_waveMax[in], wavesX);
        zr::count_launch();
    }
    zr::prof_after();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return zr::cuda_fail(e, "k_pt_bounce launch");
    return ZR_OK;
}
} // namespace zr
