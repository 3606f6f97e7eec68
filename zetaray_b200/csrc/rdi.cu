// rdi.cu -- ReSTIR DI for emissive triangles and the DirectLighting pass.
//
// Replaces DirectLighting/Emissive/ReSTIR_DI_Temporal.hlsl:29-390, ReSTIR_DI_Spatial.hlsl:27-192,
// Resampling.hlsli:36-519, PairwiseMIS.hlsli:10-232, Reservoir.hlsli:10-213, Util.hlsli:9-120 and the host
// sequencing of DirectLighting.cpp:166-284 (compiled configuration: USE_HALF_VECTOR_COPY_SHIFT 0, alias-table
// candidates, no presampled sets).
//
// Layout: the reservoir's two textures (RGBA32UI + RG32F, 24 B/px) are one 32-byte record = 2 x 128-bit;
// the RGBA16F target plane is a uint2 (8 B/px). k_di_spatial keeps the reference's 8x8 group / swizzle so one
// warp is one reference wave (the disocclusion vote is a wave op) and the group RNG is seeded by the block id.
#include "zr_pixel.cuh"
#include "zr_planes.h"
#include "zr_schedule.h"

#include "zr_rdi.cuh"
#include "zr_sky.cuh"

namespace zr
{
namespace
{
// Block sizes and register bounds: k_di_temporal 384 threads at 80 registers with its reservoir parked in shared memory (below),
// k_di_spatial 256 at 128; two blocks per SM each. Measured on an H100 SXM (700 W, 1980 MHz), ms per bench frame, at one block per SM:
// k_di_temporal 1.013 at 768 x 80 parked, 1.078 at 512 x 128 parked, 1.099 at 512 x 128 unparked; k_di_spatial 0.632 at 512 x 128,
// 0.644 with its reservoirs and neighbour list parked, 0.763 parked at 768 x 80, so it is not parked (DESIGN 4.1, item 2).
// In the renderer's frame DirectLighting runs at the least stream priority in the SM time that IndirectLighting leaves idle
// (renderer.cu). A DI block that takes an SM there holds it to its end while the chain's next kernel waits, so smaller blocks were
// measured at the same register bounds and the same threads per SM: bench.py's ms per frame, and the kernels' ms from its single-stream
// pass, medians of three runs in each of three sessions (A, B, C), builds alternating within a session:
//
//   temporal x spatial threads   frame   k_di_temporal   k_di_spatial   session
//   768 x 512 (previous)         6.394   1.020           0.636          A
//   384 x 512                    6.350   0.973           0.636          A
//   256 x 512                    6.345   1.072           0.634          A
//   768 x 256                    6.329   1.015           0.594          A
//   768 x 512 (previous)         6.367   1.015           0.634          B
//   384 x 256                    6.291   0.979           0.595          B
//   384 x 256                    6.286   0.971           0.596          C
//   384 x 128                    6.375   0.976           0.650          C
//   192 x 256                    6.348   1.134           0.597          C
//   128 x 256                    6.394   1.283           0.597          C
//
// 384 x 256 is the fastest frame, and each kernel is also faster on its own at its new size. Both material builds use these shapes. A
// block is always whole 8x8 groups (threads / 64 of them), the unit of the group RNG and the disocclusion vote.
#ifndef ZR_RDI_TEMPORAL_THREADS
#define ZR_RDI_TEMPORAL_THREADS 384
#endif
#ifndef ZR_RDI_SPATIAL_THREADS
#define ZR_RDI_SPATIAL_THREADS 256
#endif
    static_assert(ZR_RDI_TEMPORAL_THREADS % 64 == 0 && ZR_RDI_SPATIAL_THREADS % 64 == 0, "a DI block is whole 8x8 groups");
    // the register bound through __launch_bounds__'s blocks-per-SM argument, whatever the block size
    constexpr int DI_TEMPORAL_REGS = 80, DI_SPATIAL_REGS = 128;
    static_assert(ZR_RDI_TEMPORAL_THREADS * DI_TEMPORAL_REGS <= 65536 && ZR_RDI_SPATIAL_THREADS * DI_SPATIAL_REGS <= 65536,
        "a DI block must fit the register file at its bound");
    // k_di_temporal's RIS reservoir: only reservoir updates and the MIS tails touch it, yet it crosses the roughly 20 barriers of
    // RIS_InitialCandidates_Sync and TemporalResample1_Sync. It lives in dynamic shared memory, one record per thread, as
    // k_pathtrace's PtParked does. Reservoir's float2 makes the record a multiple of 8 bytes, so its stride cannot be an odd number
    // of words; 2 mod 4 words is the next best: the 32 lanes of a warp fall in 16 different banks, two per bank.
    struct DiTemporalParked
    {
        Reservoir r;
        uint32_t pad[2];
    };
    static_assert(sizeof(DiTemporalParked) % 16 == 8, "DiTemporalParked must be 2 mod 4 words");
    constexpr size_t DI_TEMPORAL_SMEM_BYTES = (size_t)ZR_RDI_TEMPORAL_THREADS * sizeof(DiTemporalParked);

    // ReSTIR_DI_Temporal.hlsl main + EstimateDirectLighting. A block is ZR_RDI_TEMPORAL_THREADS/64 consecutive 8x8 groups of the
    // reference's swizzled dispatch, walking the resampling phases together (no thread leaves before the last barrier).
    // MF: the material features the kernel is compiled for (BSDF::ShadingDataT); the scene's materials must use no others.
    // Dynamic shared memory: DI_TEMPORAL_SMEM_BYTES.
    template<uint32_t MF>
    __global__ void __launch_bounds__(ZR_RDI_TEMPORAL_THREADS, 65536 / (ZR_RDI_TEMPORAL_THREADS * DI_TEMPORAL_REGS)) k_di_temporal(SceneDev sc, FrameView f, DIParams prm, zr_rdi_reservoir* __restrict__ resCurr,
        const zr_rdi_reservoir* __restrict__ resPrev, uint2* __restrict__ target, float4* __restrict__ finalImg, uint32_t dispX, uint32_t dispY,
        const uint32_t* __restrict__ order)
    {
        using SD = BSDF::ShadingDataT<MF>;
        extern __shared__ DiTemporalParked s_diTemporalParked[];
        const zr_frame_constants& fc = f.fc;
        uint2 sg = make_uint2(0, 0);
        const uint32_t groupFlat = order[blockIdx.x] * (ZR_RDI_TEMPORAL_THREADS / 64) + (threadIdx.x >> 6);
        const uint32_t tInGroup = threadIdx.x & 63;
        uint2 px = make_uint2(0xffffffffu, 0xffffffffu);
        if (groupFlat < dispX * dispY)
            px = SwizzleThreadGroup(groupFlat, 0, tInGroup & 7, tInGroup >> 3, 8, 8, dispX, 16, 4, 16 * dispY, sg);
        const long long t0 = clock64();
        bool act = !(px.x >= f.W || px.y >= f.H || px.y < prm.rowBegin || px.y >= prm.rowEnd);
        const uint32_t x = px.x, y = px.y;
        const size_t idx = act ? (size_t)y * f.W + x : 0;
        if (act)
        {
            const GFlags flags = FlagsAt(f.core, f.W, x, y);
            if (flags.invalid)
            {
                // the sky / sun-disk background belongs to the sun-sky path (not in this build)
                finalImg[idx] = f4(0, 0, 0, 0);
                act = false;
            }
            else if (flags.emissive && !prm.spatial)
            {
                WriteEmissive(fc, f, finalImg, idx);
                act = false;
            }
        }
        PixelT<SD> p;
        p.surface = SD::InitEmpty();
        p.pos = f3(0); p.normal = f3(0); p.roughness = 0;
        RNG rng_thread; rng_thread.State = 0;
        int numBsdfSamples = 0;
        if (act)
        {
            p = LoadPixel<SD>(f, sc, f.core, f.coat, x, y, false, x, y);
            rng_thread = RNG::Init(x, y, fc.FrameNum);
            numBsdfSamples = (!p.surface.GlossSpecular() && p.roughness < 0.3f) ? 2 : 1;
        }
        // group-uniform index so that every thread of an 8x8 group uses the same presampled set (ReSTIR_DI_Temporal.hlsl:368-370)
        RNG rng_group = RNG::Init(groupFlat % dispX, groupFlat / dispX, fc.FrameNum);
        const uint32_t sampleSetIdx = rng_group.UniformUintBounded_Faster(sc.numSampleSets);
        Reservoir& r = s_diTemporalParked[threadIdx.x].r;
        RIS_InitialCandidates_Sync(r, act, sc, p.pos, p.normal, p.roughness, p.surface, sampleSetIdx, numBsdfSamples, rng_thread);
        if (prm.temporal)
        {
            float2 motionVec = f2(0, 0);
            TemporalCandidateT<SD> tc; tc.valid = false; tc.px = tc.py = 0; tc.pos = tc.normal = f3(0);
            tc.surface = SD::InitEmpty();
            ZR_PHASE();
            if (act)
            {
                motionVec = unpack_snorm16x2(__ldg(&f.me[idx].x));
                const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / f2((float)f.W, (float)f.H);
                const float2 prevUV = currUV - motionVec;
                tc = FindTemporalCandidate(f, sc, p.pos, p.normal, p.roughness, p.surface, prevUV);
            }
            TemporalResample1_Sync(act && tc.valid, sc, p.pos, p.normal, p.surface, tc, resPrev, f.W, r, rng_thread);
            if (act && prm.spatial)
            {
                const bool disoccluded = !tc.valid && (dot(motionVec, motionVec) > 0);
                r.target = disoccluded ? -r.target : r.target;
                WriteTarget(target, idx, r.target);
                r.target = Math::Sanitize(r.target);
            }
        }
        AccountCost(prm.costMap, f.W, f.H, px.x, px.y, t0);
        if (!act)
            return;
        if (prm.temporal || prm.reset)
        {
            zr_rdi_reservoir rec;
            r.Write(rec, prm.M_max);
            StoreRdi(&resCurr[idx], rec);
        }
        if (!prm.spatial || !prm.temporal)
            WriteFinal(fc, finalImg, idx, r.target * r.W);
    }

    // ReSTIR_DI_Spatial.hlsl main + SpatialResample
    template<uint32_t MF>
    __global__ void __launch_bounds__(ZR_RDI_SPATIAL_THREADS, 65536 / (ZR_RDI_SPATIAL_THREADS * DI_SPATIAL_REGS)) k_di_spatial(SceneDev sc, FrameView f, DIParams prm, const zr_rdi_reservoir* __restrict__ resCurr,
        const uint2* __restrict__ target, float4* __restrict__ finalImg, uint32_t dispX, uint32_t dispY,
        const uint32_t* __restrict__ order)
    {
        using SD = BSDF::ShadingDataT<MF>;
        const zr_frame_constants& fc = f.fc;
        uint2 sg = make_uint2(0, 0);
        const uint32_t groupFlat = order[blockIdx.x] * (ZR_RDI_SPATIAL_THREADS / 64) + (threadIdx.x >> 6);
        const uint32_t tInGroup = threadIdx.x & 63;
        uint2 px = make_uint2(0xffffffffu, 0xffffffffu);
        if (groupFlat < dispX * dispY)
            px = SwizzleThreadGroup(groupFlat, 0, tInGroup & 7, tInGroup >> 3, 8, 8, dispX, 16, 4, 16 * dispY, sg);
        const long long t0 = clock64();
        bool active = px.x < f.W && px.y < f.H && px.y >= prm.rowBegin && px.y < prm.rowEnd;
        const int x = (int)px.x, y = (int)px.y;
        const size_t idx = active ? (size_t)y * f.W + x : 0;
        if (active)
        {
            const GFlags flags = FlagsAt(f.core, f.W, x, y);
            if (flags.invalid) active = false;
            else if (flags.emissive)
            {
                WriteEmissive(fc, f, finalImg, idx);
                active = false;
            }
        }
        PixelT<SD> p;
        p.surface = SD::InitEmpty();
        p.pos = f3(0); p.normal = f3(0); p.roughness = 0; p.z = 0;
        Reservoir r = Reservoir::Init();
        bool disoccluded = false;
        if (active)
        {
            p = LoadPixel<SD>(f, sc, f.core, f.coat, x, y, false, x, y);
            zr_rdi_reservoir rec;
            LoadRdi(&resCurr[idx], rec);
            r = Reservoir::Load(rec);
            if (r.lightIdx != UINT32_MAX_)
            {
                const zr_emissive_tri& tri = sc.emissives[r.lightIdx];
                r.lightID = tri.ID;
                const float3 vtx0 = Light::Vtx0(tri);
                const float3 vtx1 = Light::DecodeEmissiveTriV1(tri);
                const float3 vtx2 = Light::DecodeEmissiveTriV2(tri);
                r.lightPos = (1.0f - r.bary.x - r.bary.y) * vtx0 + r.bary.x * vtx1 + r.bary.y * vtx2;
                r.lightNormal = cross(vtx1 - vtx0, vtx2 - vtx0);
                r.lightNormal = dot(r.lightNormal, r.lightNormal) == 0 ? r.lightNormal : normalize(r.lightNormal);
                r.doubleSided = Light::IsDoubleSided(tri);
                r.target = LoadTarget(target, idx);
                disoccluded = r.target.x < 0 || r.target.y < 0 || r.target.z < 0;
                r.target = abs3(r.target);
            }
        }
        const uint32_t waveDisoccluded = __popc(__ballot_sync(0xffffffffu, active && disoccluded));
        RNG rng_group = RNG::Init(groupFlat % dispX, groupFlat / dispX, fc.FrameNum);
        rng_group.UniformUintBounded_Faster(sc.numSampleSets);    // sample-set index: drawn, not used by the spatial pass (:137)
        const bool extra = !prm.stochasticSpatial || (rng_group.Uniform() < 0.6f);
        if (prm.extraDisocclusion)
            disoccluded = disoccluded && (waveDisoccluded > 3);
        int numSamples = extra ? 2 : 1;
        numSamples = !disoccluded ? numSamples : 4;
        RNG rng = RNG::Init((uint32_t)x, (uint32_t)y, fc.FrameNum);
        const float u0 = rng.Uniform();
        const int offset = (int)rng.UniformUintBounded_Faster(8);
        const float theta = u0 * TWO_PI;
        float sinTheta, cosTheta;
        zr_sincosf(theta, &sinTheta, &cosTheta);
        PairwiseMIS pairwiseMIS = PairwiseMIS::Init((uint32_t)numSamples, r);
        float3 samplePos[4]; int spx[4], spy[4]; uint32_t k = 0;
        ZR_PHASE();
        for (int i = 0; i < 4; i++)
        {
            if (!(active && i < numSamples)) continue;
            const float2 sampleUV = f2(c_disk32[((offset + i) & 31) * 2], c_disk32[((offset + i) & 31) * 2 + 1]);
            float2 rotated;
            rotated.x = dot(sampleUV, f2(cosTheta, -sinTheta));
            rotated.y = dot(sampleUV, f2(sinTheta, cosTheta));
            rotated = rotated * 16.0f;
            const float fx = fmaxf(rintf((float)x + rotated.x), 0.0f), fy = fmaxf(rintf((float)y + rotated.y), 0.0f);
            if (fx >= (float)f.W || fy >= (float)f.H) continue;
            const int qx = (int)fx, qy = (int)fy;
            float rough_i;
            const GFlags flags_i = FlagsAt(f.core, f.W, qx, qy, &rough_i);
            if (flags_i.invalid || flags_i.emissive) continue;
            const PixelT<SD> pi = LoadPixel<SD>(f, sc, f.core, f.coat, qx, qy, false, qx, qy);
            bool valid = PlaneHeuristicDI(pi.pos, p.normal, p.pos, p.z);
            valid = valid && (fabsf(rough_i - p.roughness) < 0.15f);
            if (!valid) continue;
            samplePos[k] = pi.pos; spx[k] = qx; spy[k] = qy;
            k++;
        }
        pairwiseMIS.k = k;
        for (uint32_t i = 0; i < 4; i++)
        {
            const bool go = active && (i < k);
            if (!__syncthreads_or(go))
                break;
            PixelT<SD> pi;
            pi.normal = f3(0);
            SD surface_i = SD::InitEmpty();
            Reservoir r_spatial = Reservoir::Init();
            float3 pos_i = f3(0);
            if (go)
            {
                pi = LoadPixel<SD>(f, sc, f.core, f.coat, spx[i], spy[i], false, spx[i], spy[i]);
                // the neighbour surface is rebuilt with transmission depth = 0 (Resampling.hlsli:507-510)
                const uint4 c = ld128(&f.core[(size_t)spy[i] * f.W + spx[i]]);
                const float3 bc = f3((float)(c.z & 0xff) / 255.0f, (float)((c.z >> 8) & 0xff) / 255.0f, (float)((c.z >> 16) & 0xff) / 255.0f);
                const float bw = pi.flags.subsurface ? (float)(c.z >> 24) / 255.0f : 0.0f;
                pos_i = samplePos[i];
                const float3 wo_i = normalize(pi.origin - pos_i);
                surface_i = SD::Init(pi.normal, wo_i, pi.flags.metallic, pi.roughness, bc, BSDF::ETA_AIR,
                    pi.eta_next, pi.flags.transmissive, 0.0f, to_half(bw), pi.surface.coat_weight, pi.surface.coat_color,
                    pi.coatRoughness, pi.coatIor, sc.rho);
                zr_rdi_reservoir recN;
                LoadRdi(&resCurr[(size_t)spy[i] * f.W + spx[i]], recN);
                r_spatial = Reservoir::Load(recN);
            }
            pairwiseMIS.Stream_Sync(go, sc, r, p.pos, p.normal, p.surface, r_spatial, pos_i, pi.normal, surface_i, rng);
        }
        AccountCost(prm.costMap, f.W, f.H, px.x, px.y, t0);
        if (!active)
            return;
        pairwiseMIS.End(r, rng);
        const Reservoir rs = pairwiseMIS.r_s;
        WriteFinal(fc, finalImg, idx, rs.target * rs.W);
    }

    // The sky behind geometry in accumulating frames (ReSTIR_DI_Temporal.hlsl:274-281), after k_di_temporal / k_di_spatial, which leave
    // invalid pixels at 0: each invalid pixel of rows [rowBegin, rowEnd) becomes its value before the frame, kept only past the first
    // accumulated frame, plus Le_SkyWithSunDisk. `before` is FINAL as it was before k_di_temporal.
    __global__ void __launch_bounds__(256) k_di_sky(zr_frame_constants fc, const uint4* __restrict__ core, Sky::LutView lut,
        const float4* __restrict__ before, float4* __restrict__ finalImg, uint32_t rowBegin, uint32_t rowEnd)
    {
        const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31);
        const uint32_t y = rowBegin + blockIdx.y * 8 + (threadIdx.x >> 5);
        const uint32_t W = fc.RenderWidth;
        if (x >= W || y >= rowEnd) return;
        const size_t i = (size_t)y * W + x;
        if (!(__ldg(&core[i].w) & ZR_GBUFFER_FLAG_INVALID)) return;
        const float4 b = before[i];
        const float3 prev = f3(b.x, b.y, b.z);
        const float3 c = prev * (float)(fc.NumFramesCameraStatic > 1) + Sky::Le_SkyWithSunDisk(fc, lut, x, y);
        finalImg[i] = f4(c.x, c.y, c.z, b.w);
    }
}
} // namespace zr

// ------------------------------------------------------------------------------------------------
// DirectLighting pass object (DirectLighting/Emissive/DirectLighting.h:36-57)
// ------------------------------------------------------------------------------------------------
struct zr_direct_pass
{
    uint32_t width = 0, height = 0;
    struct Sized
    {
        zr::Planes planes{ "zr_direct_pass" };
        zr_rdi_reservoir* d_res[2] = { nullptr, nullptr };
        uint2* d_target = nullptr;      // RGBA16F
        float4* d_final = nullptr;
    } sz;
    int currTemporalIdx = 0;
    bool isTemporalReservoirValid = false;
    bool resetTemporalTextures = true;
    bool patternLoaded = false;
    zr_direct_params params = Defaults();
    zr::LightingStrip strip{ "zr_direct_pass" };     // sched[0]: k_di_temporal, sched[1]: k_di_spatial (8x8-group blocks)
    // zr_direct_pass_set_sky: the LUT (not owned) and, only while it is set, FINAL's copy from before the accumulating frame
    zr::Sky::LutView sky{ nullptr, 0, 0 };
    struct SkyCopy
    {
        zr::Planes planes{ "zr_direct_pass" };
        float4* d_before = nullptr;
    } skyCopy;

    static zr_direct_params Defaults()
    {
        // DirectLighting.cpp:99-107, DirectLighting.h:93-98
        zr_direct_params p{};
        p.temporal_resample = 1; p.spatial_resample = 1; p.stochastic_spatial = 1; p.extra_disocclusion_sampling = 1;
        p.M_max = 20; p.alpha_min = 0.05f * 0.05f;
        return p;
    }
    zr_status Setup()
    {
        // both material-feature builds, whichever scenes the pass will render
        using zr::BSDF::MF_NONE; using zr::BSDF::MF_ALL;
        ZR_TRY(zr::ReserveParkedSmem(zr::k_di_temporal<MF_NONE>, ZR_RDI_TEMPORAL_THREADS, zr::DI_TEMPORAL_SMEM_BYTES, "zr_direct_pass: k_di_temporal"));
        ZR_TRY(zr::ReserveParkedSmem(zr::k_di_temporal<MF_ALL>, ZR_RDI_TEMPORAL_THREADS, zr::DI_TEMPORAL_SMEM_BYTES, "zr_direct_pass: k_di_temporal"));
        return ZR_OK;
    }
    zr_status OnWindowResized(uint32_t w, uint32_t h)
    {
        const size_t n = (size_t)w * h;
        Sized next;
        for (int i = 0; i < 2; i++) ZR_TRY(next.planes.Alloc(next.d_res[i], n));
        ZR_TRY(next.planes.Alloc(next.d_target, n));
        ZR_TRY(next.planes.Alloc(next.d_final, n));
        ZR_TRY(next.planes.Clear());
        SkyCopy nextSky;
        if (sky.texels) ZR_TRY(nextSky.planes.Alloc(nextSky.d_before, n, false));
        sz = std::move(next);
        skyCopy = std::move(nextSky);
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
    zr_status SetSky(const zr_image2d* lut)
    {
        zr::Sky::LutView view;
        ZR_TRY(zr::Sky::ViewOf("zr_direct_pass_set_sky", lut, view));
        SkyCopy next;
        if (view.texels && !skyCopy.d_before) ZR_TRY(next.planes.Alloc(next.d_before, (size_t)width * height, false));
        if (!view.texels || !skyCopy.d_before) skyCopy = std::move(next);
        sky = view;
        return ZR_OK;
    }
    zr_status LoadPattern()
    {
        if (patternLoaded) return ZR_OK;
        float pat[64];
        zr_status st = zr::read_asset("zr_direct_pass", "disk32.bin", pat, sizeof(pat));
        if (st != ZR_OK) return st;
        ZR_CUDA(cudaMemcpyToSymbol(zr::c_disk32, pat, 256));
        patternLoaded = true;
        return ZR_OK;
    }
    zr_status Render(const zr_frame_inputs* in, cudaStream_t stream)
    {
        using namespace zr;
        FrameView f;
        zr_status st = LightingFrame("zr_direct_pass", in, width, height, f);
        if (st != ZR_OK) return st;
        st = LoadPattern();
        if (st != ZR_OK) return st;
        const bool doTemporal = isTemporalReservoirValid && params.temporal_resample;
        const bool doSpatial = doTemporal && params.spatial_resample;
        if (doTemporal && (!in->prev.d_core || !in->prev.d_coat))
        {
            set_error("zr_direct_pass_render: temporal reuse needs the previous G-buffer");
            return ZR_ERR_INVALID_ARG;
        }
        DIParams prm{ doTemporal, doSpatial, params.stochastic_spatial, params.extra_disocclusion_sampling, params.M_max,
            params.alpha_min, resetTemporalTextures, strip.rowBegin, strip.ClampedRowEnd(height), strip.d_costMap };
        const uint32_t dispX = (width + 7) / 8, dispY = (height + 7) / 8;
        const int cur = currTemporalIdx;
        // the two kernels have different block sizes, so each has its own block table
        st = strip.Schedule(width, height, 8, 8, ZR_RDI_TEMPORAL_THREADS / 64, 0);
        if (st != ZR_OK) return st;
        st = strip.Schedule(width, height, 8, 8, ZR_RDI_SPATIAL_THREADS / 64, 1);
        if (st != ZR_OK) return st;
        const BlockSchedule& schedT = strip.sched[0];
        const BlockSchedule& schedS = strip.sched[1];
        const bool plain = (in->scene->materialFeatures & BSDF::MF_ALL) == 0;
        const bool skyAccumulates = sky.texels && in->frame.Accumulate && in->frame.CameraStatic;
        if (skyAccumulates)
        {
            const size_t rowBytes = (size_t)width * sizeof(float4), first = (size_t)prm.rowBegin * width;
            ZR_CUDA(cudaMemcpyAsync(skyCopy.d_before + first, sz.d_final + first, (prm.rowEnd - prm.rowBegin) * rowBytes,
                cudaMemcpyDeviceToDevice, stream));
        }
        ZR_PROF("k_di_temporal", stream);
        (plain ? k_di_temporal<BSDF::MF_NONE> : k_di_temporal<BSDF::MF_ALL>)<<<schedT.count, ZR_RDI_TEMPORAL_THREADS, DI_TEMPORAL_SMEM_BYTES, stream>>>(in->scene->dev, f, prm, sz.d_res[cur], sz.d_res[1 - cur], sz.d_target, sz.d_final, dispX, dispY, schedT.d_order);
        ZR_LAUNCH_CHECK();
        // the temporal output is what neighbours read in the spatial pass and what the next frame reprojects into
        strip.Exchange(sz.d_res[cur], width, height, 32u, stream);
        if (doSpatial)
        {
            ZR_PROF("k_di_spatial", stream);
            (plain ? k_di_spatial<BSDF::MF_NONE> : k_di_spatial<BSDF::MF_ALL>)<<<schedS.count, ZR_RDI_SPATIAL_THREADS, 0, stream>>>(in->scene->dev, f, prm, sz.d_res[cur], sz.d_target, sz.d_final, dispX, dispY, schedS.d_order);
            ZR_LAUNCH_CHECK();
        }
        if (skyAccumulates)
        {
            const dim3 grid((width + 31) / 32, (prm.rowEnd - prm.rowBegin + 7) / 8);
            ZR_PROF("k_di_sky", stream);
            k_di_sky<<<grid, 256, 0, stream>>>(in->frame, f.core, sky, skyCopy.d_before, sz.d_final, prm.rowBegin, prm.rowEnd);
            ZR_LAUNCH_CHECK();
        }
        isTemporalReservoirValid = true;
        currTemporalIdx = 1 - cur;
        resetTemporalTextures = false;
        return ZR_OK;
    }
};

extern "C"
{
    zr_status zr_direct_pass_create(uint32_t width, uint32_t height, zr_direct_pass** out) { return zr::CreatePass("zr_direct_pass", width, height, out); }
    zr_status zr_direct_pass_resize(zr_direct_pass* p, uint32_t width, uint32_t height) { return zr::ResizePass("zr_direct_pass", p, width, height); }
    zr_status zr_direct_pass_reset_temporal(zr_direct_pass* p) { return zr::ResetPass(p); }
    zr_status zr_direct_pass_default_params(zr_direct_params* out) { return zr::DefaultParams<zr_direct_pass>(out); }
    zr_status zr_direct_pass_set_params(zr_direct_pass* p, const zr_direct_params* params)
    {
        if (!p || !params) return ZR_ERR_INVALID_ARG;
        if (params->M_max == 0 || params->M_max > 31) { zr::set_error("zr_direct_pass_set_params: M_max must be in 1..31 (5-bit field)"); return ZR_ERR_INVALID_ARG; }
        p->params = *params;
        return ZR_OK;
    }
    zr_status zr_direct_pass_set_sky(zr_direct_pass* p, const zr_image2d* lut) { return p ? p->SetSky(lut) : ZR_ERR_INVALID_ARG; }
    zr_status zr_direct_pass_render(zr_direct_pass* p, const zr_frame_inputs* in, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, (cudaStream_t)stream);
    }
    zr_status zr_direct_pass_set_rows(zr_direct_pass* p, uint32_t y0, uint32_t y1) { return p ? p->strip.SetRows(y0, y1, p->height) : ZR_ERR_INVALID_ARG; }
    zr_status zr_direct_pass_set_halo_exchange(zr_direct_pass* p, zr_halo_exchange_fn fn, void* user) { return p ? p->strip.SetHaloExchange(fn, user) : ZR_ERR_INVALID_ARG; }
    zr_status zr_direct_pass_set_schedule_costs(zr_direct_pass* p, const double* h_tile_cost, uint32_t tiles_x, uint32_t tiles_y)
    {
        return p ? p->strip.SetScheduleCosts(h_tile_cost, tiles_x, tiles_y, p->width, p->height) : ZR_ERR_INVALID_ARG;
    }
    zr_status zr_direct_pass_set_cost_map(zr_direct_pass* p, void* d_cycles) { return p ? p->strip.SetCostMap(d_cycles) : ZR_ERR_INVALID_ARG; }
    zr_status zr_direct_pass_get_output(zr_direct_pass* p, zr_direct_output id, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        const uint32_t w = p->width, h = p->height;
        switch (id)
        {
        case ZR_DIRECT_FINAL: *out = zr_image2d{ p->sz.d_final, w, h, w * 16u, 16u }; break;
        case ZR_DIRECT_RESERVOIR_CURR: *out = zr_image2d{ p->sz.d_res[1 - p->currTemporalIdx], w, h, w * 32u, 32u }; break;
        case ZR_DIRECT_TARGET: *out = zr_image2d{ p->sz.d_target, w, h, w * 8u, 8u }; break;
        default: zr::set_error("zr_direct_pass_get_output: unknown output id"); return ZR_ERR_INVALID_ARG;
        }
        return ZR_OK;
    }
    zr_status zr_direct_pass_describe_io(zr_direct_pass* p, zr_resource_use* uses, int* n)
    {
        if (!p || !uses || !n) return ZR_ERR_INVALID_ARG;
        uses[0] = zr_resource_use{ ZR_RES_GBUFFER_CURR, 0 };
        uses[1] = zr_resource_use{ ZR_RES_GBUFFER_PREV, 0 };
        uses[2] = zr_resource_use{ ZR_RES_SCENE_BVH, 0 };
        uses[3] = zr_resource_use{ ZR_RES_ALIAS_TABLE, 0 };
        uses[4] = zr_resource_use{ ZR_RES_DI_FINAL, 1 };
        *n = 5;
        return ZR_OK;
    }
    void zr_direct_pass_destroy(zr_direct_pass* p) { delete p; }
}
