// rgi.cu -- IndirectLighting with INTEGRATOR::ReSTIR_GI (emissive NEE): one kernel per frame.
//
// Replaces IndirectLighting/ReSTIR_GI/ReSTIR_GI.hlsl (+ Resampling.hlsli, PathTracing.hlsli, ReSTIR_GI_NEE.hlsli,
// Reservoir.hlsli, ../NEE.hlsli) and the host sequencing of IndirectLighting.cpp:277-368 for the ReSTIR_GI_WoPS / _WPS
// variants: a path-traced initial candidate (second path vertex + its outgoing radiance), temporal reuse with one or two
// reprojected candidates weighted by the reconnection Jacobian, wave-level outlier suppression; NEE after the first indirect
// vertex optionally from the light voxel grid (ReSTIR_GI_LVG). Not built: sun/sky NEE, ray differentials (they only feed texture LOD; no textures in this build), the spatial
// pass (commented out upstream, Resampling.hlsli:603-608).
// A block is 16 consecutive 8x8 groups of the reference's swizzled dispatch, one warp per reference wave, so the
// Russian-roulette WaveActiveMax (PathTracing.hlsli:64-67, evaluated over the lanes at the same loop iteration) is a warp max
// and SuppressOutlierReservoirs (Resampling.hlsli:533-539) a warp sum. Block barriers keep the warps of a block at the
// same stage (zr_rpt.cuh "block-synchronous phases"); this first version synchronises per stage, not inside NEE or the
// temporal resampling.
// D3D semantics kept: FindTemporalCandidate does not reject negative tap coordinates and out-of-bounds texture reads
// return 0, so LoadPrev / the reservoir readers return zeros there.
// With the degenerate-ray cut of zr_scene.cuh::Traverse compiled into THIS translation unit -- in either formulation, empty stack or
// early return -- ptxas has been seen to lay k_rgi out so that warps run the traversal with about half the active lanes, although
// the atrium's ReSTIR GI frame contains no degenerate ray at all. The other kernels are unaffected and the path tracer needs the
// cut (a zero-direction ray otherwise sweeps the whole tree), so only this unit opts out. Cost: a zero-direction ray (2-3 per 14 400 pixels on scenes with glass) sweeps the tree here.
#define ZR_NO_DEGENERATE_RAY_EARLY_OUT
#include "zr_pixel.cuh"
#include "zr_rpt.cuh"       // ZR_PHASE
#include "zr_planes.h"
#include "zr_schedule.h"

#include "zr_rgi.cuh"

namespace zr
{
namespace
{
#ifndef ZR_RGI_THREADS
#define ZR_RGI_THREADS 1024
#endif
    // PlainPT = true: IndirectLighting/PathTracer/PathTracer.hlsl (INTEGRATOR::PATH_TRACING) -- the same dispatch shape, RNG
    // seeds and PathTrace loop without reservoirs or reuse (main :98-212, EstimateIndirectLighting :58-104).
    template<bool PlainPT>
    __global__ void ZR_LB(ZR_RGI_THREADS) k_rgi(SceneDev sc, FrameView f, GIParams prm, zr_rgi_reservoir* __restrict__ resCurr,
        const zr_rgi_reservoir* __restrict__ resPrev, float4* __restrict__ finalImg, uint32_t dispX, uint32_t dispY,
        const uint32_t* __restrict__ order)
    {
        const zr_frame_constants& fc = f.fc;
        uint2 sg = make_uint2(0, 0);
        const uint32_t groupFlat = order[blockIdx.x] * (ZR_RGI_THREADS / 64) + (threadIdx.x >> 6);
        const uint32_t tInGroup = threadIdx.x & 63;
        uint2 px = make_uint2(0xffffffffu, 0xffffffffu);
        if (groupFlat < dispX * dispY)
            px = SwizzleThreadGroup(groupFlat, 0, tInGroup & 7, tInGroup >> 3, 8, 8, dispX, 16, 4, 16 * dispY, sg);
        bool active = px.x < f.W && px.y < f.H && px.y >= prm.rowBegin && px.y < prm.rowEnd;
        const size_t idx = active ? (size_t)px.y * f.W + px.x : 0;
        GFlags flags = DecodeFlags(0);
        float roughness = 0;
        float3 baseColor = f3(0);
        if (active)
        {
            const uint4 g = ld128(&f.core[idx]);
            flags = DecodeFlags(g.w & 0xff);
            roughness = (float)((g.w >> 8) & 0xff) / 255.0f;
            baseColor = f3((float)(g.z & 0xff) / 255.0f, (float)((g.z >> 8) & 0xff) / 255.0f, (float)((g.z >> 16) & 0xff) / 255.0f);
            if (flags.invalid || flags.emissive)
            {
                if (!fc.Accumulate || !fc.CameraStatic)
                {
                    const float4 prev = finalImg[idx];
                    finalImg[idx] = f4(0, 0, 0, prev.w);
                }
                active = false;
            }
        }
        // ---- main :96-150 + EstimateIndirectLighting :547-556 ----
        Pixel p;
        BSDF::ShadingData surface0 = BSDF::ShadingData::InitEmpty();
        RNG rngThread, rngGroup;
        rngThread.State = rngGroup.State = 0;
        int maxNumBounces = 0;
        uint32_t sampleSetIdx = 0;
        GIReservoir r = GIReservoir::Init();
        BSDF::BSDFSample bsdfSample0 = BSDF::BSDFSample::Init();
        if (active)
        {
            p = LoadPixel(f, sc, f.core, f.coat, (int)px.x, (int)px.y, false, (int)px.x, (int)px.y);
            const float3 wo = normalize(p.origin - p.pos);
            // PathTracer.hlsl:184-185 also passes flags.trDepthGt0 as the transmission depth
            surface0 = BSDF::ShadingData::Init(p.normal, wo, flags.metallic, roughness, baseColor, BSDF::ETA_AIR, p.eta_next, flags.transmissive,
                (PlainPT && flags.trDepthGt0) ? 1.0f : 0.0f, 0.0f, 0.0f, f3(0.0f), 0.0f, BSDF::DEFAULT_ETA_COAT, sc.rho);
            rngGroup = RNG::Init(sg.x ^ 61u, sg.y ^ 61u, fc.FrameNum);
            rngThread = RNG::Init(px.x ^ 511u, px.y ^ 31u, fc.FrameNum);
            maxNumBounces = (int)(flags.transmissive ? prm.maxGlossyTrBounces : prm.maxNonTrBounces);
            if (!PlainPT && prm.stochasticMultiBounce && (roughness >= 0.1f || fc.CameraStatic))
                maxNumBounces = rngGroup.Uniform() < 0.5f ? 1 : maxNumBounces;
            sampleSetIdx = rngGroup.UniformUintBounded_Faster(sc.numSampleSets);
        }
        ZR_PHASE();
        // ---- RIS_InitialCandidates :39-81 ----
        if (active)
            bsdfSample0 = BSDF::SampleBSDF(p.normal, surface0, rngThread);
        bool traced = active && (bsdfSample0.pdf != 0);
        ZR_PHASE();
        Hit hit0 = RPT::MissHit();
        if (traced)
        {
            hit0 = FindClosest(sc, p.pos, p.normal, bsdfSample0.wi, surface0.Transmissive());
            traced = hit0.hit;
        }
        float3 hitPos0 = f3(0);
        // ---- PathTrace (PathTracing.hlsli:10-98), lock-step ----
        float3 pos = f3(0), normal = f3(0), li = f3(0), throughput = f3(1.0f);
        float eta_curr = BSDF::ETA_AIR, eta_next = BSDF::DEFAULT_ETA_MAT;
        bool inTranslucentMedium = false;
        int bounce = 0;
        BSDF::BSDFSample bsdfSample = bsdfSample0;
        Hit hitInfo = hit0;
        BSDF::ShadingData surface = BSDF::ShadingData::InitEmpty();
        bool tracing = traced;
        if (traced)
        {
            hitPos0 = p.pos + hit0.t * bsdfSample0.wi;
            pos = p.pos; normal = p.normal;
            eta_curr = dot(normal, bsdfSample0.wi) < 0 ? p.eta_next : BSDF::ETA_AIR;
            inTranslucentMedium = dot(normal, bsdfSample0.wi) < 0;
        }
        while (__syncthreads_or(tracing))
        {
            bool atRR = false;
            if (tracing)
            {
                const float3 hitPos = mad(hitInfo.t, bsdfSample.wi, pos);
                if (!GetMaterialData(sc, -bsdfSample.wi, eta_curr, hitInfo, surface, eta_next))
                    tracing = false;
                else
                {
                    li += throughput * NEE<PlainPT>(sc, fc, hitPos, hitInfo.normal, surface, sampleSetIdx, bounce, rngThread);
                    // ACCOUNT_FOR_TRANSMITTANCE == 1 (PathTracing.hlsli:41-48): Beer's law inside a translucent medium
                    if (PlainPT && inTranslucentMedium && (surface.trDepth > 0))
                    {
                        const float3 c = surface.baseColor_Fr0_TrCol;
                        const float3 extCoeff = f3(-zr_logf(c.x), -zr_logf(c.y), -zr_logf(c.z)) / surface.trDepth;
                        throughput *= f3(zr_expf(-hitInfo.t * extCoeff.x), zr_expf(-hitInfo.t * extCoeff.y), zr_expf(-hitInfo.t * extCoeff.z));
                    }
                    if (bounce >= (maxNumBounces - 1))
                        tracing = false;
                    else
                    {
                        pos = hitPos;
                        normal = hitInfo.normal;
                        bounce++;
                        atRR = true;
                    }
                }
            }
            // Russian roulette against the wave's maximum throughput
            const uint32_t rrMask = __ballot_sync(0xffffffffu, atRR);
            bool doRR = false;
            float waveThroughput = 0.0f;
            if (rrMask)
            {
                const int rrBounce = __shfl_sync(0xffffffffu, bounce, __ffs(rrMask) - 1);
                doRR = prm.russianRoulette && (rrBounce >= 3);
                if (doRR)
                    waveThroughput = WaveMax32(atRR ? Math::Luminance(throughput) : -FLT_MAX_);
            }
            ZR_PHASE();
            if (atRR)
            {
                bool go = true;
                if (doRR)
                {
                    const float p_terminate = fmaxf(0.05f, 1 - waveThroughput);
                    if (rngGroup.Uniform() < p_terminate)
                        go = false;
                    else
                        throughput /= (1 - p_terminate);
                }
                if (go)
                {
                    bsdfSample = BSDF::BSDFSample::Init();
                    if (bounce < maxNumBounces)
                        bsdfSample = BSDF::SampleBSDF(normal, surface, rngThread);
                    if (Math::Luminance(bsdfSample.bsdfOverPdf) == 0)
                        go = false;
                }
                if (go)
                {
                    hitInfo = FindClosest(sc, pos, normal, bsdfSample.wi, surface.Transmissive());
                    if (!hitInfo.hit)
                        go = false;
                }
                if (go)
                {
                    throughput *= bsdfSample.bsdfOverPdf;
                    const bool transmitted = dot(normal, bsdfSample.wi) < 0;
                    eta_curr = transmitted ? (eta_curr == BSDF::ETA_AIR ? eta_next : BSDF::ETA_AIR) : eta_curr;
                    inTranslucentMedium = transmitted ? !inTranslucentMedium : inTranslucentMedium;
                }
                tracing = go;
            }
        }
        if (PlainPT)
        {
            // EstimateIndirectLighting :97-103, main :199-211
            if (!active)
                return;
            float3 liOut = f3(0);
            if (traced)
            {
                liOut = li;
                if (dot(liOut, liOut) > 0)
                    liOut *= bsdfSample0.bsdfOverPdf;
            }
            liOut = isnan3(liOut) ? f3(0) : liOut;
            const float4 prev = finalImg[idx];
            if (fc.Accumulate && fc.CameraStatic)
                finalImg[idx] = f4(prev.x + liOut.x, prev.y + liOut.y, prev.z + liOut.z, prev.w);
            else
                finalImg[idx] = f4(liOut.x, liOut.y, liOut.z, prev.w);
            return;
        }
        // ---- rest of RIS_InitialCandidates :83-113 ----
        if (traced)
        {
            const float3 lo = li;
            float3 target = lo;
            if (dot(lo, lo) > 0)
            {
                surface0.SetWi(bsdfSample0.wi, p.normal);
                target *= BSDF::Unified(surface0).f;
            }
            const float targetLum = Math::Luminance(target);
            const float w = targetLum / fmaxf(bsdfSample0.pdf, 1e-6f);
            r.Update(w, hitPos0, hit0.normal, hit0.ID, lo, target, rngThread);
            r.W = targetLum > 0 ? 1.0f / bsdfSample0.pdf : 0.0f;
        }
        ZR_PHASE();
        // ---- temporal reuse (EstimateIndirectLighting :564-596) ----
        if (prm.temporalResample)
        {
            if (active)
            {
                const float2 renderDim = f2((float)f.W, (float)f.H);
                const float2 motionVec = unpack_snorm16x2(__ldg(&f.me[idx].x));
                const float2 currUV = f2((float)px.x + 0.5f, (float)px.y + 0.5f) / renderDim;
                const float2 prevUV = currUV - motionVec;
                TemporalSampleData data[2]; bool valid[2];
                FindTemporalCandidate(f, sc, (int)px.x, (int)px.y, p.pos, p.normal, p.z, roughness, surface0.specTr, prevUV, rngThread, data, valid);
                if (valid[1] && roughness > 0.05f)
                    TemporalResample2(f, sc, resPrev, p.pos, p.normal, surface0, data, r, rngThread);
                else if (valid[0])
                    TemporalResample1(f, sc, resPrev, p.pos, p.normal, surface0, data[0], r, rngThread);
            }
            if (prm.boilingSuppression)
            {
                const float waveSum = WaveSum32(active ? r.w_sum : 0.0f);
                if (active)
                {
                    const float waveAvg = (waveSum - r.w_sum) / 31.0f;
                    if (r.w_sum > 25 * waveAvg)
                        r.M = 1;
                }
            }
        }
        if (!active)
            return;
        if (prm.temporalResample || prm.resetTemporal)
        {
            zr_rgi_reservoir rec;
            WriteReservoir(rec, r, (float)prm.M_max);
            uint4 v[3];
            memcpy(v, &rec, 48);
            uint4* q = reinterpret_cast<uint4*>(&resCurr[idx]);
            q[0] = v[0]; q[1] = v[1]; q[2] = v[2];
        }
        float3 liOut = r.target_z * r.W;
        liOut = isnan3(liOut) ? f3(0) : liOut;
        const float4 prev = finalImg[idx];
        if (fc.Accumulate && fc.CameraStatic)
            finalImg[idx] = f4(prev.x + liOut.x, prev.y + liOut.y, prev.z + liOut.z, prev.w);
        else
            finalImg[idx] = f4(liOut.x, liOut.y, liOut.z, prev.w);
    }
}
} // namespace zr

// ------------------------------------------------------------------------------------------------
// IndirectLighting pass object for INTEGRATOR::ReSTIR_GI (IndirectLighting.cpp:277-368, :1016-1024)
// ------------------------------------------------------------------------------------------------
struct zr_gi_pass
{
    uint32_t width = 0, height = 0;
    struct Sized
    {
        zr::Planes planes{ "zr_gi_pass" };
        zr_rgi_reservoir* d_res[2] = { nullptr, nullptr };
        float4* d_final = nullptr;
    } sz;
    int currTemporalIdx = 0;
    bool isTemporalReservoirValid = false;
    bool resetTemporalTextures = true;
    zr_gi_params params = Defaults();
    bool plainPathTracer = false;       // INTEGRATOR::PATH_TRACING instead of ReSTIR_GI (both read cb_ReSTIR_GI in the reference)
    // the hook makes the reservoirs just written coherent across strips (they are next frame's temporal candidates, searched up to
    // 16 px around the reprojected pixel: ReSTIR_GI/Params.hlsli:45); no tile costs are ever set, so blocks run in plain order
    zr::LightingStrip strip{ "zr_gi_pass" };

    static zr_gi_params Defaults()
    {
        // IndirectLighting.h:231-244, IndirectLighting.cpp:143-160
        zr_gi_params p{};
        p.max_non_tr_bounces = 3; p.max_glossy_tr_bounces = 4; p.russian_roulette = 1; p.stochastic_multi_bounce = 1;
        p.boiling_suppression = 1; p.M_max = 10; p.temporal_resample = 1;
        return p;
    }
    zr_status Setup() { return ZR_OK; }
    zr_status OnWindowResized(uint32_t w, uint32_t h)
    {
        const size_t n = (size_t)w * h;
        Sized next;
        for (int i = 0; i < 2; i++) ZR_TRY(next.planes.Alloc(next.d_res[i], n));
        ZR_TRY(next.planes.Alloc(next.d_final, n));
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
    zr_status Render(const zr_frame_inputs* in, cudaStream_t stream)
    {
        using namespace zr;
        FrameView f;
        zr_status st = LightingFrame("zr_gi_pass", in, width, height, f);
        if (st != ZR_OK) return st;
        if (in->scene->dev.lvg && in->scene->dev.sampleSetSize && !in->scene->lvgValid)
        {
            set_error("zr_gi_pass_render: the light voxel grid is enabled but zr_build_light_voxel_grid has not run");
            return ZR_ERR_NOT_INITIALIZED;
        }
        const bool doTemporal = !plainPathTracer && params.temporal_resample && isTemporalReservoirValid;
        if (doTemporal && !in->prev.d_core)
        {
            set_error("zr_gi_pass_render: temporal reuse needs the previous G-buffer");
            return ZR_ERR_INVALID_ARG;
        }
        GIParams prm{ params.max_non_tr_bounces, params.max_glossy_tr_bounces, params.russian_roulette, params.stochastic_multi_bounce,
            params.boiling_suppression, params.M_max, doTemporal ? 1u : 0u, resetTemporalTextures ? 1u : 0u, strip.rowBegin, strip.ClampedRowEnd(height) };
        const uint32_t dispX = (width + 7) / 8, dispY = (height + 7) / 8;
        st = strip.Schedule(width, height, 8, 8, ZR_RGI_THREADS / 64);
        if (st != ZR_OK) return st;
        const BlockSchedule& sched = strip.sched[0];
        const int cur = currTemporalIdx;
        if (plainPathTracer)
        {
            ZR_PROF("k_pathtracer", stream);
            k_rgi<true><<<sched.count, ZR_RGI_THREADS, 0, stream>>>(in->scene->dev, f, prm, sz.d_res[cur], sz.d_res[1 - cur], sz.d_final, dispX, dispY, sched.d_order);
            ZR_LAUNCH_CHECK();
            return ZR_OK;       // no reservoirs: the ReSTIR GI history is left as it is (and is dropped by SetMethod)
        }
        ZR_PROF("k_rgi", stream);
        k_rgi<false><<<sched.count, ZR_RGI_THREADS, 0, stream>>>(in->scene->dev, f, prm, sz.d_res[cur], sz.d_res[1 - cur], sz.d_final, dispX, dispY, sched.d_order);
        ZR_LAUNCH_CHECK();
        strip.Exchange(sz.d_res[cur], width, height, (uint32_t)sizeof(zr_rgi_reservoir), stream);
        isTemporalReservoirValid = true;
        currTemporalIdx = 1 - cur;
        resetTemporalTextures = false;
        return ZR_OK;
    }
};

extern "C"
{
    zr_status zr_gi_pass_create(uint32_t width, uint32_t height, zr_gi_pass** out) { return zr::CreatePass("zr_gi_pass", width, height, out); }
    zr_status zr_gi_pass_resize(zr_gi_pass* p, uint32_t width, uint32_t height) { return zr::ResizePass("zr_gi_pass", p, width, height); }
    zr_status zr_gi_pass_reset_temporal(zr_gi_pass* p) { return zr::ResetPass(p); }
    zr_status zr_gi_pass_default_params(zr_gi_params* out) { return zr::DefaultParams<zr_gi_pass>(out); }
    zr_status zr_gi_pass_set_params(zr_gi_pass* p, const zr_gi_params* params)
    {
        if (!p || !params) return ZR_ERR_INVALID_ARG;
        if (params->max_non_tr_bounces < 1 || params->max_non_tr_bounces > 8 || params->max_glossy_tr_bounces < 1 ||
            params->max_glossy_tr_bounces > 8 || params->M_max == 0 || params->M_max > 2047)
        {
            zr::set_error("zr_gi_pass_set_params: value out of range (bounces 1..8, M_max 1..2047)");
            return ZR_ERR_INVALID_ARG;
        }
        p->params = *params;
        return ZR_OK;
    }
    // IndirectLighting::SetMethod for the two integrators that share this pass object (IndirectLighting.cpp:203-235):
    // ZR_INTEGRATOR_PATH_TRACING or ZR_INTEGRATOR_RESTIR_GI; a change drops the temporal history.
    zr_status zr_gi_pass_set_method(zr_gi_pass* p, zr_integrator method)
    {
        if (!p || (method != ZR_INTEGRATOR_PATH_TRACING && method != ZR_INTEGRATOR_RESTIR_GI))
        {
            zr::set_error("zr_gi_pass_set_method: PATH_TRACING (0) or RESTIR_GI (1); ReSTIR PT is zr_indirect_pass");
            return ZR_ERR_INVALID_ARG;
        }
        const bool plain = method == ZR_INTEGRATOR_PATH_TRACING;
        if (plain == p->plainPathTracer) return ZR_OK;
        p->plainPathTracer = plain;
        return p->ResetTemporal();
    }
    zr_status zr_gi_pass_set_rows(zr_gi_pass* p, uint32_t y0, uint32_t y1) { return p ? p->strip.SetRows(y0, y1, p->height) : ZR_ERR_INVALID_ARG; }
    zr_status zr_gi_pass_set_halo_exchange(zr_gi_pass* p, zr_halo_exchange_fn fn, void* user) { return p ? p->strip.SetHaloExchange(fn, user) : ZR_ERR_INVALID_ARG; }
    zr_status zr_gi_pass_render(zr_gi_pass* p, const zr_frame_inputs* in, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, (cudaStream_t)stream);
    }
    zr_status zr_gi_pass_get_output(zr_gi_pass* p, zr_gi_output id, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        const uint32_t w = p->width, h = p->height;
        switch (id)
        {
        case ZR_GI_FINAL: *out = zr_image2d{ p->sz.d_final, w, h, w * 16u, 16u }; break;
        case ZR_GI_RESERVOIR_CURR: *out = zr_image2d{ p->sz.d_res[1 - p->currTemporalIdx], w, h, w * 48u, 48u }; break;
        case ZR_GI_RESERVOIR_PREV: *out = zr_image2d{ p->sz.d_res[p->currTemporalIdx], w, h, w * 48u, 48u }; break;
        default: zr::set_error("zr_gi_pass_get_output: unknown output id"); return ZR_ERR_INVALID_ARG;
        }
        return ZR_OK;
    }
    void zr_gi_pass_destroy(zr_gi_pass* p) { delete p; }
}
