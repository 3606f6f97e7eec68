// ORACLE -- test infrastructure, not product code (see orc_math.h header).
//
// CPU restatement of the ReSTIR PT frame (SURVEY 8a-14, a-16), dispatch by dispatch:
//   ReSTIR_PT_PathTrace.hlsl      PathTrace :195-358, RIS_InitialCandidates :360-417, main :423-559
//   ReSTIR_PT_Sort.hlsl           counting sort of 32x32 tiles by reconnection k :114-368
//   ReSTIR_PT_SpatialSearch.hlsl  :21-146
//   ReSTIR_PT_Replay.hlsl         (folded into the reconnect steps, see OffsetPathContext::Quantize)
//   ReSTIR_PT_Reconnect_CtT/TtC/CtS/StC.hlsl
//   IndirectLighting.cpp:370-1025 host sequencing, flags, ping-pong
// Wave-scope operations (RR wave max, boiling-suppression wave sums, sort prefix sums) are replayed
// with the reference's lane -> pixel maps (16x8 / 8x8 / 16x16 groups, row-major lanes, group swizzle).
// Deterministic choices where the reference is racy or unspecified (DESIGN.md): waves of a sort
// group take their offsets in wave order; wave sums use the xor-butterfly order.
#include "orc_api.h"
#include "orc_rpt.h"
#include "orc_pixel.h"
#include <functional>
#include <thread>

using namespace orc;
using namespace orc::RPT;

namespace
{
    struct Params
    {
        uint32_t maxNonTrBounces, maxGlossyTrBounces, russianRoulette, M_max_temporal, M_max_spatial;
        uint32_t boilingSuppression, sortTemporal, sortSpatial;
        float alpha_min;
    };

    // Util.hlsli:9-42
    uint16_t EncodeSorted(int dx, int dy, int mx, int my, uint32_t error)
    {
        int ddx = dx - mx, ddy = dy - my;
        uint32_t ux = (uint32_t)(ddx + 31), uy = (uint32_t)(ddy + 31);
        return (uint16_t)(ux | (uy << 7) | ((error > 0 ? 1u : 0u) << 15));
    }
    void DecodeSorted(int x, int y, uint16_t encoded, int& ox, int& oy, bool& error)
    {
        error = (encoded & (1 << 15)) != 0;
        int dx = (int)(encoded & 0x3f) - 31, dy = (int)((encoded >> 7) & 0x3f) - 31;
        ox = x + dx; oy = y + dy;
    }

    void WriteOutputColor(const zr_frame_constants& fc, float4* finalImg, size_t idx, float3 li)
    {
        li = isnan3(li) ? f3(0) : li;
        if (fc.Accumulate && fc.CameraStatic && fc.NumFramesCameraStatic > 1)
        {
            float4 prev = finalImg[idx];
            finalImg[idx] = f4(prev.x + li.x, prev.y + li.y, prev.z + li.z, prev.w);
        }
        else
            finalImg[idx] = f4(li.x, li.y, li.z, finalImg[idx].w);
    }

    // -------------------------------------------------------------------------------------------
    // PathTrace (K8)
    // -------------------------------------------------------------------------------------------
    struct PrevHit { float alpha_lobe; float3 wi; float pdf; LOBE lobe; };

    struct PTLane
    {
        bool inBounds = false, alive = false;
        int px = 0, py = 0;
        float3 pos, normal; ShadingData surface; BSDF::BSDFSample bsdfSample; HitEmissive nextHit;
        Reconnection rc; Reservoir r; float3 li, throughput, throughput_k; PrevHit prevHit;
        float eta_curr; bool inTranslucentMedium; int bounce; int maxNumBounces;
        RNG rngReplay, rngThread, rngGroup; uint32_t seedReplay0; uint32_t sampleSetIdx = 0;
        // carried over the wave op
        Hit hitInfo; float eta_next; float3 tr; float prevBsdfSamplePdf; LOBE prevBsdfSampleLobe; int pathVertex;
    };

    void MaybeSetCase2OrCase3(int pathVertex, float3 pos, float3 normal, float t, uint32_t ID, uint32_t meshIdx,
        const ShadingData& surface, const PrevHit& prevHit, const DirectLightingEstimate& ls, uint32_t seed_nee, Reconnection& rc, float alpha_min)
    {
        const float alpha_lobe_direct = BSDF::LobeAlpha(surface, ls.lobe);
        if (rc.Empty() && CanReconnect(prevHit.alpha_lobe, alpha_lobe_direct, prevHit.lobe, ls.lobe, alpha_min))
        {
            rc.SetCase2(pathVertex, pos, t, normal, ID, meshIdx, prevHit.wi, prevHit.lobe, prevHit.pdf, ls.wi, ls.lobe,
                ls.pdf_solidAngle, ls.lt, ls.pdf_light, ls.le, seed_nee, ls.dwdA);
        }
        if (rc.Empty() && (alpha_lobe_direct >= alpha_min))
        {
            rc.SetCase3(pathVertex + 1, ls.pos, ls.lt, ls.lobe, ls.ID, ls.le, ls.normal, ls.pdf_solidAngle, ls.pdf_light,
                ls.dwdA, ls.wi, ls.twoSided, seed_nee);
        }
    }

    // loop top .. Russian-roulette point. returns 0 = left the loop, 1 = reached the RR point
    int PT_PhaseA(const Scene& sc, PTLane& s, const Params& prm)
    {
        s.pathVertex = s.bounce + 2;
        s.hitInfo.hit = s.nextHit.hit;
        s.hitInfo.t = s.nextHit.t;
        if (!s.nextHit.hit)
            return 0;
        s.hitInfo = HitAttributes(sc, s.nextHit.geoIdx, s.nextHit.primIdx, s.nextHit.bary, s.nextHit.t);
        float3 newPos = mad(s.hitInfo.t, s.bsdfSample.wi, s.pos);
        if (!GetMaterialData(sc, -s.bsdfSample.wi, s.eta_curr, s.hitInfo, s.surface, s.eta_next))
            return 0;
        s.pos = newPos;
        s.normal = s.hitInfo.normal;
        s.prevBsdfSamplePdf = s.bsdfSample.pdf;
        s.prevBsdfSampleLobe = s.bsdfSample.lobe;
        s.tr = f3(1);
        if (s.inTranslucentMedium && (s.surface.trDepth > 0))
        {
            float3 c = s.surface.baseColor_Fr0_TrCol;
            float3 extCoeff = f3(-zr_logf(c.x), -zr_logf(c.y), -zr_logf(c.z)) / s.surface.trDepth;
            s.tr = f3(zr_expf(-s.hitInfo.t * extCoeff.x), zr_expf(-s.hitInfo.t * extCoeff.y), zr_expf(-s.hitInfo.t * extCoeff.z));
            s.throughput *= s.tr;
        }
        // EstimateDirectAndUpdateRC<Emissive = true>
        {
            BSDF::BSDFSample nextBsdfSample = s.bsdfSample;     // HLSL leaves it uninitialised when not sampled; see NEE_Bsdf
            int nextBounce = s.pathVertex - 1;
            DirectLightingEstimate ls_b = NEE_Bsdf(sc, s.pos, s.hitInfo.normal, s.surface, nextBounce, s.maxNumBounces,
                nextBsdfSample, s.nextHit, s.rngReplay);
            if (s.nextHit.HitWasEmissive())
            {
                const float3 fOverPdf = s.throughput * ls_b.ld;
                s.li += fOverPdf;
                s.rc.L = Reconnection::half3(ls_b.ld * s.throughput_k);
                MaybeSetCase2OrCase3(s.pathVertex, s.pos, s.hitInfo.normal, s.hitInfo.t, s.hitInfo.ID, s.hitInfo.meshIdx, s.surface,
                    s.prevHit, ls_b, 0, s.rc, prm.alpha_min);
                float risWeight = Math::Luminance(fOverPdf);
                s.r.Update(risWeight, fOverPdf, s.rc, s.rngThread);
            }
            const bool specular = IsSpecularSurface(s.surface);
            if (!specular)
            {
                const uint32_t seed_nee = s.rngThread.State;
                DirectLightingEstimate ls = NEE_Emissive(sc, s.pos, s.hitInfo.normal, s.surface, s.sampleSetIdx, s.rngThread);
                const float3 fOverPdf = s.throughput * ls.ld;
                s.li += fOverPdf;
                if (s.rc.IsCase2() || s.rc.IsCase3())
                    s.rc.Clear();
                s.rc.L = Reconnection::half3(ls.ld * s.throughput_k);
                MaybeSetCase2OrCase3(s.pathVertex, s.pos, s.hitInfo.normal, s.hitInfo.t, s.hitInfo.ID, s.hitInfo.meshIdx, s.surface,
                    s.prevHit, ls, seed_nee, s.rc, prm.alpha_min);
                float risWeight = Math::Luminance(fOverPdf);
                s.r.Update(risWeight, fOverPdf, s.rc, s.rngThread);
            }
            s.bsdfSample = nextBsdfSample;
        }
        if (s.bounce >= (s.maxNumBounces - 1))
            return 0;
        if (s.rc.IsCase2() || s.rc.IsCase3())
            s.rc.Clear();
        s.bounce++;
        return 1;
    }

    // after the (optional) wave op. returns false if the lane leaves the loop
    bool PT_PhaseB(PTLane& s, const Params& prm, bool doRR, float waveThroughput)
    {
        if (doRR)
        {
            if (waveThroughput < 1)
            {
                float p_terminate = fmaxf(0.05f, 1 - waveThroughput);
                if (s.rngGroup.Uniform() < p_terminate)
                    return false;
                s.throughput /= (1 - p_terminate);
                s.throughput_k /= ((int)s.rc.k <= s.bounce) ? (1 - p_terminate) : 1.0f;
            }
        }
        if (dot(s.bsdfSample.bsdfOverPdf, s.bsdfSample.bsdfOverPdf) == 0)
            return false;
        const float alpha_lobe = BSDF::LobeAlpha(s.surface, s.bsdfSample.lobe);
        if (s.rc.Empty() && CanReconnect(s.prevHit.alpha_lobe, alpha_lobe, s.prevHit.lobe, s.bsdfSample.lobe, prm.alpha_min))
        {
            s.rc.SetCase1(s.pathVertex, s.pos, s.hitInfo.t, s.hitInfo.normal, s.hitInfo.ID, s.hitInfo.meshIdx, -s.surface.wo,
                s.prevBsdfSampleLobe, s.prevBsdfSamplePdf, s.bsdfSample.wi, s.bsdfSample.lobe, s.bsdfSample.pdf);
            s.throughput_k = f3(1);
        }
        if ((int)s.rc.k <= s.bounce)
            s.throughput_k *= s.bsdfSample.bsdfOverPdf * s.tr;
        bool transmitted = dot(s.normal, s.bsdfSample.wi) < 0;
        s.throughput *= s.bsdfSample.bsdfOverPdf;
        s.eta_curr = transmitted ? (s.eta_curr == BSDF::ETA_AIR ? s.eta_next : BSDF::ETA_AIR) : s.eta_curr;
        s.inTranslucentMedium = s.eta_curr != BSDF::ETA_AIR;
        s.prevHit.alpha_lobe = alpha_lobe;
        s.prevHit.lobe = s.bsdfSample.lobe;
        s.prevHit.wi = s.bsdfSample.wi;
        s.prevHit.pdf = s.bsdfSample.pdf;
        return true;
    }

    void PathTracePass(const Frame& f, const Params& prm, bool temporalResample, bool resetTemporal, zr_rpt_reservoir* res,
        float4* target, float4* finalImg, int nthreads)
    {
        const zr_frame_constants& fc = *f.fc;
        const uint32_t dispX = (f.W + 15) / 16, dispY = (f.H + 7) / 8;
        const uint32_t numGroupsInTile = 16 * dispY;
        const uint32_t numWaves = dispX * dispY * 4;
        parallel_for(numWaves, nthreads, [&](uint32_t w0, uint32_t w1)
        {
            std::vector<PTLane> lanes(32);
            for (uint32_t wv = w0; wv < w1; wv++)
            {
                const uint32_t group = wv / 4, wave = wv % 4;
                const uint32_t Gx = group % dispX, Gy = group / dispX;
                for (int l = 0; l < 32; l++)
                {
                    PTLane& s = lanes[l];
                    s = PTLane();
                    uint32_t GTx = l % 16, GTy = wave * 2 + l / 16;
                    uint32_t sx, sy, sgx, sgy;
                    SwizzleThreadGroup(Gx, Gy, GTx, GTy, 16, 8, dispX, 16, 4, numGroupsInTile, sx, sy, sgx, sgy);
                    if (sx >= f.W || sy >= f.H)
                        continue;
                    s.inBounds = true; s.px = (int)sx; s.py = (int)sy;
                    const size_t idx = (size_t)sy * f.W + sx;
                    GFlags flags = FlagsAt(f.core, f.W, sx, sy);
                    if (flags.invalid || flags.emissive)
                    {
                        if (!fc.Accumulate || !fc.CameraStatic)
                            finalImg[idx] = f4(0, 0, 0, finalImg[idx].w);
                        s.inBounds = false;
                        continue;
                    }
                    Pixel p = LoadPixel(f, f.core, f.coat, sx, sy, false, sx, sy);
                    // RIS_InitialCandidates
                    s.rngGroup = RNG::Init4(sgx, sgy, fc.FrameNum, 1);
                    const uint3 state = RNG::PCG3d(uint3{ sx, sy, fc.FrameNum });
                    s.rngReplay = RNG::InitSeed(state.x);
                    s.rngThread = RNG::InitSeed(state.y);
                    s.seedReplay0 = state.x;
                    s.maxNumBounces = (int)(p.surface.specTr ? prm.maxGlossyTrBounces : prm.maxNonTrBounces);
                    s.li = f3(0);
                    s.r = Reservoir::Init();
                    s.rc = Reconnection::Init();
                    s.bsdfSample = BSDF::SampleBSDF(p.normal, p.surface, s.rngReplay);
                    if (dot(s.bsdfSample.bsdfOverPdf, s.bsdfSample.bsdfOverPdf) == 0)
                    {
                        s.alive = false;    // returns an empty reservoir, li = 0
                        continue;
                    }
                    // one presampled set for all threads of this group (ReSTIR_PT_PathTrace.hlsl:406-408)
                    s.sampleSetIdx = s.rngGroup.UniformUintBounded_Faster(f.sc->numSampleSets);
                    // PathTrace prologue
                    s.pos = p.pos; s.normal = p.normal; s.surface = p.surface;
                    s.bounce = 0;
                    s.throughput = s.bsdfSample.bsdfOverPdf;
                    s.prevHit.alpha_lobe = BSDF::LobeAlpha(p.surface, s.bsdfSample.lobe);
                    s.prevHit.lobe = s.bsdfSample.lobe; s.prevHit.wi = s.bsdfSample.wi; s.prevHit.pdf = s.bsdfSample.pdf;
                    s.eta_curr = dot(p.normal, s.bsdfSample.wi) < 0 ? p.eta_next : BSDF::ETA_AIR;
                    s.throughput_k = f3(1);
                    s.inTranslucentMedium = s.eta_curr != BSDF::ETA_AIR;
                    s.nextHit = FindClosestEmissive(*f.sc, s.pos, s.normal, s.bsdfSample.wi, s.surface.Transmissive());
                    s.alive = true;
                }
                // lock-step bounce loop
                for (;;)
                {
                    bool any = false;
                    bool atRR[32];
                    for (int l = 0; l < 32; l++)
                    {
                        atRR[l] = false;
                        PTLane& s = lanes[l];
                        if (!s.inBounds || !s.alive) continue;
                        if (PT_PhaseA(*f.sc, s, prm) == 0) { s.alive = false; continue; }
                        atRR[l] = true; any = true;
                    }
                    if (!any) break;
                    // all lanes at the RR point share the same bounce count
                    float waveMax = -FLT_MAX_;
                    bool doRR = false;
                    for (int l = 0; l < 32; l++)
                        if (atRR[l])
                        {
                            doRR = prm.russianRoulette && (lanes[l].bounce >= 3);
                            waveMax = fmaxf(waveMax, Math::Luminance(lanes[l].throughput));
                        }
                    for (int l = 0; l < 32; l++)
                        if (atRR[l] && !PT_PhaseB(lanes[l], prm, doRR, waveMax))
                            lanes[l].alive = false;
                }
                // epilogue
                for (int l = 0; l < 32; l++)
                {
                    PTLane& s = lanes[l];
                    if (!s.inBounds) continue;
                    const size_t idx = (size_t)s.py * f.W + s.px;
                    Reservoir& r = s.r;
                    r.rc.seed_replay = s.seedReplay0;
                    float targetLum = Math::Luminance(r.target);
                    r.W = targetLum > 0 ? fmaxf(r.w_sum / targetLum, 1.0f) : 0;
                    if (temporalResample || resetTemporal)
                        r.Write(res[idx], 0);
                    if (temporalResample)
                    {
                        r.target = Math::Sanitize(r.target);
                        target[idx] = f4(r.target.x, r.target.y, r.target.z, target[idx].w);
                    }
                    else
                    {
                        float3 li = isnan3(s.li) ? f3(0) : s.li;
                        if (fc.Accumulate && fc.CameraStatic)
                        {
                            float4 prev = finalImg[idx];
                            finalImg[idx] = f4(prev.x + li.x, prev.y + li.y, prev.z + li.z, prev.w);
                        }
                        else
                            finalImg[idx] = f4(li.x, li.y, li.z, finalImg[idx].w);
                    }
                }
            }
        });
    }

    // -------------------------------------------------------------------------------------------
    // Temporal / spatial neighbour lookup shared by Sort, Replay and Reconnect
    // -------------------------------------------------------------------------------------------
    bool PrevPixel(const Frame& f, int x, int y, int& ppx, int& ppy)
    {
        const float2 renderDim = f2((float)f.W, (float)f.H);
        const float2 motionVec = unpack_snorm16x2(f.me[(size_t)y * f.W + x].x);
        const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / renderDim;
        const float2 prevUV = currUV - motionVec;
        float2 pp = prevUV * renderDim;
        ppx = (int)pp.x; ppy = (int)pp.y;
        if (prevUV.x < 0.0f || prevUV.y < 0.0f || prevUV.x > 1.0f || prevUV.y > 1.0f)
            return false;
        return true;
    }

    // ReSTIR_PT_Sort.hlsl. mode: 0 = CtT, 1 = TtC, 2 = CtS, 3 = StC
    void SortPass(const Frame& f, int mode, bool spatialResampleFlag, const zr_rpt_reservoir* resCurr, const zr_rpt_reservoir* resPrev,
        const uint16_t* neighbor, uint16_t* threadMap)
    {
        enum { SUCCESS = 0, INVALID_PIXEL = 1, NOT_FOUND = 2, EMPTY = 4 };
        const uint32_t dispX = (f.W + 31) / 32, dispY = (f.H + 31) / 32;
        for (uint32_t Gy = 0; Gy < dispY; Gy++)
            for (uint32_t Gx = 0; Gx < dispX; Gx++)
            {
                struct Item { int dx, dy; uint32_t result; bool skip, edge; int cls; uint32_t k; };
                // [wave][lane][i]
                static thread_local std::vector<Item> items;
                items.assign(256 * 4, Item());
                const bool againstEdge = (Gx == dispX - 1) || (Gy == dispY - 1);
                const bool lastGroup = (Gx == dispX - 1) && (Gy == dispY - 1);
                for (uint32_t Gidx = 0; Gidx < 256; Gidx++)
                {
                    const uint32_t GTx = Gidx % 16, GTy = Gidx / 16;
                    const int gtx[4] = { (int)GTx * 2, (int)GTx * 2 + 1, (int)GTx * 2, (int)GTx * 2 + 1 };
                    const int gty[4] = { (int)GTy * 2, (int)GTy * 2, (int)GTy * 2 + 1, (int)GTy * 2 + 1 };
                    for (int i = 0; i < 4; i++)
                    {
                        Item& it = items[Gidx * 4 + i];
                        it.dx = (int)(Gx * 32) + gtx[i]; it.dy = (int)(Gy * 32) + gty[i];
                        int nx = 0, ny = 0;
                        uint32_t err = SUCCESS;
                        if ((uint32_t)it.dx >= f.W || (uint32_t)it.dy >= f.H)
                            err = INVALID_PIXEL;
                        else
                        {
                            GFlags flags = FlagsAt(f.core, f.W, it.dx, it.dy);
                            if (flags.invalid || flags.emissive)
                                err = INVALID_PIXEL;
                            else if (mode == 1)
                            {
                                if (!PrevPixel(f, it.dx, it.dy, nx, ny)) err = NOT_FOUND;
                            }
                            else if (mode == 3)
                            {
                                uint16_t nb = neighbor[(size_t)it.dy * f.W + it.dx];
                                int ox = nb & 0xff, oy = nb >> 8;
                                if (ox == 0xff) err = NOT_FOUND;
                                else { nx = ox - 32 + it.dx; ny = oy - 32 + it.dy; }
                            }
                        }
                        it.skip = err != SUCCESS;
                        it.result = err;
                        // Reservoir::Init() => k = EMPTY unless loaded
                        uint32_t k = Reconnection::EMPTY;
                        if (err == SUCCESS)
                        {
                            const zr_rpt_reservoir* src; int sx, sy;
                            if (mode == 1) { src = resPrev; sx = nx; sy = ny; }
                            else if (mode == 3) { src = resCurr; sx = nx; sy = ny; }
                            else { src = resCurr; sx = it.dx; sy = it.dy; }
                            uint32_t kk = src[(size_t)sy * f.W + sx].meta & 0xf;
                            k = kk == Reconnection::EMPTY ? kk : kk + 2;
                        }
                        if (k == Reconnection::EMPTY)
                        {
                            it.result |= EMPTY;
                            it.skip = true;
                        }
                        it.edge = false;
                        if (it.skip && againstEdge && ((uint32_t)it.dx < f.W) && ((uint32_t)it.dy < f.H))
                        {
                            it.result = SUCCESS;
                            it.skip = false;
                            it.edge = true;
                        }
                        it.k = k;
                        it.cls = -1;
                        if (!it.skip)
                        {
                            if (k == 2) it.cls = 0;
                            else if (k == 3) it.cls = 1;
                            else if (k == 4) it.cls = 2;
                            else if (k >= 5 || it.edge) it.cls = 3;
                        }
                        else it.cls = 4;
                        // note: !skip with k outside {2,3,4,>=5} cannot happen (k >= 2 whenever non-empty)
                    }
                }
                auto writeOutput = [&](int dx, int dy, int mgx, int mgy, uint32_t result)
                {
                    if ((Gx == dispX - 1) && (Gy != dispY - 1)) { int t = mgx; mgx = mgy; mgy = t; }
                    int mx = (int)(Gx * 32) + mgx, my = (int)(Gy * 32) + mgy;
                    uint32_t error;
                    if (mode == 1)
                        error = result & (spatialResampleFlag ? (INVALID_PIXEL | NOT_FOUND) : INVALID_PIXEL);
                    else if (mode == 3)
                        error = result & INVALID_PIXEL;
                    else
                        error = result & (INVALID_PIXEL | EMPTY);
                    if ((uint32_t)mx < f.W && (uint32_t)my < f.H)
                        threadMap[(size_t)my * f.W + mx] = EncodeSorted(dx, dy, mx, my, error);
                };
                if (lastGroup)
                {
                    for (uint32_t Gidx = 0; Gidx < 256; Gidx++)
                    {
                        const uint32_t GTx = Gidx % 16, GTy = Gidx / 16;
                        const int gtx[4] = { (int)GTx * 2, (int)GTx * 2 + 1, (int)GTx * 2, (int)GTx * 2 + 1 };
                        const int gty[4] = { (int)GTy * 2, (int)GTy * 2, (int)GTy * 2 + 1, (int)GTy * 2 + 1 };
                        for (int i = 0; i < 4; i++)
                        {
                            const Item& it = items[Gidx * 4 + i];
                            writeOutput(it.dx, it.dy, gtx[i], gty[i], it.result);
                        }
                    }
                    continue;
                }
                // class totals, then ranks: class-major, wave order, lane order, 2x2 order
                uint32_t count[5] = { 0, 0, 0, 0, 0 };
                for (auto& it : items) count[it.cls]++;
                uint32_t base[5];
                base[0] = 0; base[1] = count[0]; base[2] = count[0] + count[1]; base[3] = base[2] + count[2]; base[4] = base[3] + count[3];
                uint32_t running[5] = { 0, 0, 0, 0, 0 };
                for (uint32_t Gidx = 0; Gidx < 256; Gidx++)
                    for (int i = 0; i < 4; i++)
                    {
                        const Item& it = items[Gidx * 4 + i];
                        uint32_t rank = base[it.cls] + running[it.cls]++;
                        // GroupIndexToGTid over the 32-wide tile
                        int mgx = (int)(rank & 31), mgy = (int)(rank >> 5);
                        writeOutput(it.dx, it.dy, mgx, mgy, it.result);
                    }
            }
    }

    // ReSTIR_PT_SpatialSearch.hlsl
    const float* g_samplePattern = nullptr;  // 512 x (x, y), values already rounded to binary16

    void SpatialSearchPass(const Frame& f, uint16_t* neighbor, int nthreads)
    {
        const zr_frame_constants& fc = *f.fc;
        parallel_for(f.H, nthreads, [&](uint32_t y0, uint32_t y1)
        {
            for (uint32_t y = y0; y < y1; y++)
                for (uint32_t x = 0; x < f.W; x++)
                {
                    const size_t idx = (size_t)y * f.W + x;
                    float roughness;
                    GFlags flags = FlagsAt(f.core, f.W, x, y, &roughness);
                    if (flags.invalid || flags.emissive)
                        continue;       // output untouched
                    const float viewDepth = asfloat(f.core[idx].x);
                    const float2 renderDimF = f2((float)f.W, (float)f.H);
                    const float2 jitter = f2(fc.CurrCameraJitter[0], fc.CurrCameraJitter[1]);
                    const float3 pos = Math::WorldPosFromScreenSpace(f2((float)x, (float)y), renderDimF, viewDepth, fc.TanHalfFOV,
                        fc.AspectRatio, fc.CurrViewInv, jitter);
                    const float3 normal = Math::DecodeUnitVector(Math::DecodeUNorm2(f.core[idx].y));
                    uint3 h = RNG::PCG3d(uint3{ x, y, fc.FrameNum });
                    RNG rng = RNG::Init(h.x, h.y, fc.FrameNum);
                    const float u0 = rng.Uniform();
                    const uint32_t offset = rng.UniformUint();
                    const float theta = u0 * TWO_PI;
                    float sinTheta, cosTheta;
                    zr_sincosf(theta, &sinTheta, &cosTheta);
                    int foundX = 0xffff, foundY = 0xffff;
                    for (uint32_t i = 0; i < 3; i++)
                    {
                        const uint32_t si = (offset + i) & 511;
                        const float2 sampleUV = f2(g_samplePattern[si * 2], g_samplePattern[si * 2 + 1]);
                        float2 rotated = f2(dot(sampleUV, f2(cosTheta, -sinTheta)), dot(sampleUV, f2(sinTheta, cosTheta)));
                        rotated = rotated * 15.0f;
                        const int sxp = (int)rintf((float)x + rotated.x), syp = (int)rintf((float)y + rotated.y);
                        if (sxp < 0 || syp < 0 || sxp >= (int)f.W || syp >= (int)f.H) continue;
                        if (sxp == (int)x && syp == (int)y) continue;
                        float sampleRoughness;
                        GFlags sf = FlagsAt(f.core, f.W, sxp, syp, &sampleRoughness);
                        if (sf.invalid || sf.emissive) continue;
                        if (flags.metallic != sf.metallic) continue;
                        if (flags.transmissive != sf.transmissive) continue;
                        if (fabsf(sampleRoughness - roughness) > 0.05f) continue;
                        const size_t sidx = (size_t)syp * f.W + sxp;
                        const float sampleDepth = asfloat(f.core[sidx].x);
                        const float3 samplePos = Math::WorldPosFromScreenSpace(f2((float)sxp, (float)syp), renderDimF, sampleDepth,
                            fc.TanHalfFOV, fc.AspectRatio, fc.CurrViewInv, jitter);
                        const float3 sampleNormal = Math::DecodeUnitVector(Math::DecodeUNorm2(f.core[sidx].y));
                        // PlaneHeuristic(samplePos, normal, pos, viewDepth, 0.01)
                        float planeDist = fabsf(dot(normal, samplePos - pos));
                        if (!(planeDist <= 0.01f * viewDepth)) continue;
                        if (dot(sampleNormal, normal) < 0.9f) continue;
                        foundX = sxp; foundY = syp;
                        break;
                    }
                    uint32_t mx, my;
                    if (foundX == 0xffff) { mx = 0xff; my = 0xff; }
                    else { mx = (uint32_t)(foundX - (int)x + 32); my = (uint32_t)(foundY - (int)y + 32); }
                    neighbor[idx] = (uint16_t)((mx & 0xff) | ((my & 0xff) << 8));
                }
        });
    }

    // map a dispatch thread to the pixel it works on (group swizzle + optional sorted thread map)
    struct LaneMap { bool active; int x, y; };
    LaneMap MapLane(const Frame& f, uint32_t Gx, uint32_t Gy, uint32_t GTx, uint32_t GTy, uint32_t gdx, uint32_t gdy,
        uint32_t dispX, uint32_t dispY, bool sorted, const uint16_t* threadMap)
    {
        uint32_t sx, sy, sgx, sgy;
        SwizzleThreadGroup(Gx, Gy, GTx, GTy, gdx, gdy, dispX, 16, 4, 16 * dispY, sx, sy, sgx, sgy);
        LaneMap m; m.active = false; m.x = (int)sx; m.y = (int)sy;
        if (sx >= f.W || sy >= f.H) return m;
        if (sorted)
        {
            bool error; int ox, oy;
            DecodeSorted((int)sx, (int)sy, threadMap[(size_t)sy * f.W + sx], ox, oy, error);
            if (error) return m;
            m.x = ox; m.y = oy;
        }
        m.active = true;
        return m;
    }

    bool PlaneHeuristic(float3 prevPos, float3 normal, float3 pos, float linearDepth, float th)
    {
        float planeDist = fabsf(dot(normal, prevPos - pos));
        return planeDist <= th * linearDepth;
    }

    // moves x_k between the current and previous transforms of its mesh (Reconnect_CtT.hlsl:258-272, TtC :309-329)
    void XkToPrev(const Scene& sc, Reconnection& rc)
    {
        const zr_mesh_instance& md = sc.instances[rc.meshIdx];
        float4 q_curr = normalize(Math::DecodeNormalized4(md.Rotation));
        float3 T = f3(md.Translation[0], md.Translation[1], md.Translation[2]);
        float3 x_local = Math::InverseTransformTRS(rc.x_k, T, q_curr, Scene::h3(md.Scale));
        float3 prevTranslation = T - Scene::h3(md.dTranslation);
        float4 q_prev = normalize(Math::DecodeNormalized4(md.PrevRotation));
        rc.x_k = Math::TransformTRS(x_local, prevTranslation, q_prev, Scene::h3(md.PrevScale));
    }
    void XkToCurr(const Scene& sc, Reconnection& rc)
    {
        const zr_mesh_instance& md = sc.instances[rc.meshIdx];
        float3 T = f3(md.Translation[0], md.Translation[1], md.Translation[2]);
        float3 dT = Scene::h3(md.dTranslation);
        float3 prevTranslation = T - dT;
        float4 q_prev = normalize(Math::DecodeNormalized4(md.PrevRotation));
        float3 prevScale = Scene::h3(md.PrevScale), scale = Scene::h3(md.Scale);
        float3 x_local = Math::InverseTransformTRS(rc.x_k, prevTranslation, q_prev, prevScale);
        float4 q_curr = normalize(Math::DecodeNormalized4(md.Rotation));
        rc.x_k = Math::TransformTRS(x_local, T, q_curr, scale);
        float4 dRot = f4(q_prev.x - q_curr.x, q_prev.y - q_curr.y, q_prev.z - q_curr.z, q_prev.w - q_curr.w);
        float3 dScale = prevScale - scale;
        rc.x_k_in_motion = dot(dT, dT) > 0;
        rc.x_k_in_motion = rc.x_k_in_motion || dot(dRot, dRot) > 0;
        rc.x_k_in_motion = rc.x_k_in_motion || dot(dScale, dScale) > 0;
    }

    // Temporal validity shared by Replay (plane threshold 0.01) and Reconnect (threshold 1)
    struct TemporalCtx { bool ok; int ppx, ppy; Pixel cur, prev; };
    TemporalCtx TemporalSetup(const Frame& f, int x, int y, float planeTh)
    {
        TemporalCtx t; t.ok = false;
        if (!PrevPixel(f, x, y, t.ppx, t.ppy)) return t;
        const float prevViewDepth = asfloat(f.pcore[(size_t)t.ppy * f.W + t.ppx].x);
        if (prevViewDepth == FLT_MAX_) return t;
        t.cur = LoadPixel(f, f.core, f.coat, x, y, false, x, y);
        // ShiftCurrentToTemporal reads the coat plane at the CURRENT pixel (Reconnect_CtT.hlsl:88)
        t.prev = LoadPixel(f, f.pcore, f.pcoat, t.ppx, t.ppy, true, x, y);
        if (!PlaneHeuristic(t.prev.pos, t.cur.normal, t.cur.pos, t.cur.z, planeTh)) return t;
        if (t.prev.flags.emissive || (fabsf(t.prev.roughness - t.cur.roughness) > 0.3f) || (t.prev.flags.transmissive != t.cur.flags.transmissive))
            return t;
        t.ok = true;
        return t;
    }

    // Replay + Reconnect_CtT fused per pixel
    void ReconnectCtT(const Frame& f, const Params& prm, zr_rpt_reservoir* resCurr, const zr_rpt_reservoir* resPrev,
        const uint16_t* threadMap, int nthreads)
    {
        const uint32_t dispX = (f.W + 15) / 16, dispY = (f.H + 7) / 8;
        parallel_for(dispX * dispY, nthreads, [&](uint32_t g0, uint32_t g1)
        {
            for (uint32_t g = g0; g < g1; g++)
                for (uint32_t t = 0; t < 128; t++)
                {
                    LaneMap m = MapLane(f, g % dispX, g / dispX, t % 16, t / 16, 16, 8, dispX, dispY, prm.sortTemporal != 0, threadMap);
                    if (!m.active) continue;
                    GFlags flags = FlagsAt(f.core, f.W, m.x, m.y);
                    if (flags.invalid || flags.emissive) continue;
                    TemporalCtx tc = TemporalSetup(f, m.x, m.y, 1.0f);
                    if (!tc.ok) continue;
                    const size_t idx = (size_t)m.y * f.W + m.x;
                    Reservoir r_curr = Reservoir::Load_NonReconnection(resCurr[idx]);
                    Reservoir r_prev = Reservoir::Init();
                    r_prev.UnpackMetadata(resPrev[(size_t)tc.ppy * f.W + tc.ppx].meta);
                    if (r_curr.w_sum != 0 && r_prev.M > 0 && !r_curr.rc.Empty())
                    {
                        r_curr.Load_Reconnection(resCurr[idx]);
                        if (r_curr.rc.IsCase1() || r_curr.rc.IsCase2())
                            XkToPrev(*f.sc, r_curr.rc);
                        OffsetPathContext ctx; const OffsetPathContext* pctx = nullptr;
                        if (r_curr.rc.k > 2)
                        {
                            // Replay_CtT runs with the tighter plane test (ReSTIR_PT_Replay.hlsl:404)
                            TemporalCtx tr = TemporalSetup(f, m.x, m.y, 0.01f);
                            ctx = OffsetPathContext::Init();
                            if (tr.ok)
                            {
                                Reconnection rcOrig = Reservoir::Load(resCurr[idx]).rc;   // replay sees the untransformed x_k (unused by replay)
                                ctx = Replay_kGt2(*f.sc, tc.prev.pos, tc.prev.normal, tc.prev.eta_next, tc.prev.surface, rcOrig, prm.alpha_min).Quantize();
                            }
                            pctx = &ctx;
                        }
                        OffsetPath shift = Shift2(*f.sc, tc.prev.pos, tc.prev.normal, tc.prev.eta_next, tc.prev.surface, r_curr.rc, pctx, prm.alpha_min);
                        float target_prev = Math::Luminance(shift.target);
                        if (target_prev > 0)
                        {
                            float targetLum_curr = r_curr.W > 0 ? r_curr.w_sum / r_curr.W : 0;
                            float jacobian = r_curr.rc.partialJacobian > 0 ? shift.partialJacobian / r_curr.rc.partialJacobian : 0;
                            float m_curr = targetLum_curr / (targetLum_curr + (float)r_prev.M * target_prev * jacobian);
                            r_curr.w_sum *= m_curr;
                            resCurr[idx].w_sum = r_curr.w_sum;
                        }
                    }
                }
        });
    }

    void ReconnectTtC(const Frame& f, const Params& prm, bool spatialFlag, zr_rpt_reservoir* resCurr, const zr_rpt_reservoir* resPrev,
        float4* target, float4* finalImg, const uint16_t* threadMap, int nthreads)
    {
        const zr_frame_constants& fc = *f.fc;
        const uint32_t dispX = (f.W + 15) / 16, dispY = (f.H + 7) / 8;
        parallel_for(dispX * dispY, nthreads, [&](uint32_t g0, uint32_t g1)
        {
            for (uint32_t g = g0; g < g1; g++)
                for (uint32_t t = 0; t < 128; t++)
                {
                    LaneMap m = MapLane(f, g % dispX, g / dispX, t % 16, t / 16, 16, 8, dispX, dispY, prm.sortTemporal != 0, threadMap);
                    if (!m.active) continue;
                    GFlags flags = FlagsAt(f.core, f.W, m.x, m.y);
                    if (flags.invalid || flags.emissive) continue;
                    const size_t idx = (size_t)m.y * f.W + m.x;
                    Reservoir r_curr = Reservoir::Load_NonReconnection(resCurr[idx]);
                    r_curr.target = f3(target[idx].x, target[idx].y, target[idx].z);
                    TemporalCtx tc = TemporalSetup(f, m.x, m.y, 1.0f);
                    if (!tc.ok)
                    {
                        if (!spatialFlag)
                            WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
                        continue;
                    }
                    const zr_rpt_reservoir& sp = resPrev[(size_t)tc.ppy * f.W + tc.ppx];
                    Reservoir r_prev = Reservoir::Load_NonReconnection(sp);
                    const uint32_t M_new = r_curr.M + r_prev.M;
                    const uint32_t M_max = prm.M_max_temporal;
                    if (r_prev.rc.Empty())
                    {
                        float targetLum = Math::Luminance(r_curr.target);
                        r_curr.W = targetLum > 0 ? r_curr.w_sum / targetLum : 0;
                        r_curr.M = M_new;
                        // WriteReservoirData2: A.x and B.y
                        uint32_t k = r_curr.rc.Empty() ? r_curr.rc.k : (r_curr.rc.k > 2 ? r_curr.rc.k : 2) - 2;
                        uint32_t mm = r_curr.M < M_max ? r_curr.M : M_max;
                        resCurr[idx].meta = (resCurr[idx].meta & 0xffffff00u) | ((k | (mm << 4)) & 0xff);
                        resCurr[idx].W = r_curr.W;
                        if (!spatialFlag)
                            WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
                        continue;
                    }
                    r_prev.Load_Reconnection(sp);
                    Reconnection rcReplay = r_prev.rc;
                    if (r_prev.rc.IsCase1() || r_prev.rc.IsCase2())
                        XkToCurr(*f.sc, r_prev.rc);
                    OffsetPathContext ctx; const OffsetPathContext* pctx = nullptr;
                    if (r_prev.rc.k > 2)
                    {
                        TemporalCtx tr = TemporalSetup(f, m.x, m.y, 0.01f);
                        ctx = OffsetPathContext::Init();
                        if (tr.ok)
                            ctx = Replay_kGt2(*f.sc, tc.cur.pos, tc.cur.normal, tc.cur.eta_next, tc.cur.surface, rcReplay, prm.alpha_min).Quantize();
                        pctx = &ctx;
                    }
                    OffsetPath shift = Shift2(*f.sc, tc.cur.pos, tc.cur.normal, tc.cur.eta_next, tc.cur.surface, r_prev.rc, pctx, prm.alpha_min);
                    float targetLum_curr = Math::Luminance(shift.target);
                    float jacobian = r_prev.rc.partialJacobian > 0 ? shift.partialJacobian / r_prev.rc.partialJacobian : 0;
                    bool changed = false;
                    if (targetLum_curr > 1e-6f && jacobian > 1e-5f)
                    {
                        RNG rng = RNG::Init((uint32_t)m.y, (uint32_t)m.x, fc.FrameNum + 31);
                        float targetLum_prev = r_prev.W > 0 ? r_prev.w_sum / r_prev.W : 0;
                        float numerator = (float)r_prev.M * targetLum_prev;
                        float denom = numerator / jacobian + targetLum_curr;
                        float m_prev = denom > 0 ? numerator / denom : 0;
                        float w_prev = m_prev * r_prev.W * targetLum_curr;
                        if (r_curr.Update(w_prev, shift.target, r_prev.rc, rng))
                        {
                            r_curr.rc.partialJacobian = shift.partialJacobian;
                            changed = true;
                        }
                    }
                    float targetLum = Math::Luminance(r_curr.target);
                    r_curr.W = targetLum > 0 ? r_curr.w_sum / targetLum : 0;
                    r_curr.M = M_new;
                    if (changed)
                    {
                        r_curr.Write(resCurr[idx], M_max);
                        if (spatialFlag)
                        {
                            r_curr.target = Math::Sanitize(r_curr.target);
                            target[idx] = f4(r_curr.target.x, r_curr.target.y, r_curr.target.z, target[idx].w);
                        }
                    }
                    else
                        r_curr.WriteReservoirData(resCurr[idx], M_max);
                    if (!spatialFlag)
                        WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
                }
        });
    }

    bool NeighborOf(const Frame& f, const uint16_t* neighbor, int x, int y, int& nx, int& ny)
    {
        uint16_t nb = neighbor[(size_t)y * f.W + x];
        int ox = nb & 0xff, oy = nb >> 8;
        if (ox == 0xff) return false;
        nx = ox - 32 + x; ny = oy - 32 + y;
        return true;
    }

    // Replay_CtS + Reconnect_CtS fused: writes the scaled w_sum into the output buffer's B.x
    void ReconnectCtS(const Frame& f, const Params& prm, const zr_rpt_reservoir* resIn, zr_rpt_reservoir* resOut,
        const uint16_t* neighbor, const uint16_t* threadMap, int nthreads)
    {
        const uint32_t dispX = (f.W + 7) / 8, dispY = (f.H + 7) / 8;
        parallel_for(dispX * dispY, nthreads, [&](uint32_t g0, uint32_t g1)
        {
            for (uint32_t g = g0; g < g1; g++)
                for (uint32_t t = 0; t < 64; t++)
                {
                    LaneMap m = MapLane(f, g % dispX, g / dispX, t % 8, t / 8, 8, 8, dispX, dispY, prm.sortSpatial != 0, threadMap);
                    if (!m.active) continue;
                    int nx, ny;
                    if (!NeighborOf(f, neighbor, m.x, m.y, nx, ny)) continue;
                    GFlags flags = FlagsAt(f.core, f.W, m.x, m.y);
                    if (flags.invalid || flags.emissive) continue;
                    const size_t idx = (size_t)m.y * f.W + m.x;
                    Reservoir r_curr = Reservoir::Load_NonReconnection(resIn[idx]);
                    Reservoir r_spatial = Reservoir::Init();
                    r_spatial.UnpackMetadata(resIn[(size_t)ny * f.W + nx].meta);
                    if ((r_curr.w_sum != 0) && !r_curr.rc.Empty())
                    {
                        r_curr.Load_Reconnection(resIn[idx]);
                        // ShiftCurrentToSpatial reads the coat plane at the CURRENT pixel (Reconnect_CtS.hlsl:100)
                        Pixel pn = LoadPixel(f, f.core, f.coat, nx, ny, false, m.x, m.y);
                        OffsetPathContext ctx; const OffsetPathContext* pctx = nullptr;
                        if (r_curr.rc.k > 2)
                        {
                            Pixel pr = LoadPixel(f, f.core, f.coat, nx, ny, false, nx, ny);
                            ctx = Replay_kGt2(*f.sc, pr.pos, pr.normal, pr.eta_next, pr.surface, r_curr.rc, prm.alpha_min).Quantize();
                            pctx = &ctx;
                        }
                        OffsetPath shift = Shift2(*f.sc, pn.pos, pn.normal, pn.eta_next, pn.surface, r_curr.rc, pctx, prm.alpha_min);
                        float target_spatial = Math::Luminance(shift.target);
                        if (target_spatial > 0)
                        {
                            float targetLum_curr = r_curr.W > 0 ? r_curr.w_sum / r_curr.W : 0;
                            float jacobian = r_curr.rc.partialJacobian > 0 ? shift.partialJacobian / r_curr.rc.partialJacobian : 0;
                            float numerator = (float)r_curr.M * targetLum_curr;
                            float denom = numerator + (float)r_spatial.M * target_spatial * jacobian;
                            float m_curr = denom > 0 ? numerator / denom : 0;
                            r_curr.w_sum *= m_curr;
                        }
                        resOut[idx].w_sum = r_curr.w_sum;
                    }
                }
        });
    }

    // CopyToNextFrame (Reconnect_StC.hlsl:83-106)
    void CopyToNextFrame(const zr_rpt_reservoir& in, zr_rpt_reservoir& out, Reservoir r_curr, uint32_t M_max)
    {
        if (!r_curr.rc.Empty())
        {
            r_curr.Load_Reconnection(in);
            r_curr.Write(out, M_max);
        }
        else
            r_curr.WriteReservoirData(out, M_max);
    }

    void SuppressOutlier(float waveAvgExclusive, Reservoir& r)
    {
        if (r.w_sum > 50 * waveAvgExclusive)
        {
            r.M = 0; r.w_sum = 0; r.W = 0; r.rc.Clear();
        }
    }

    // Replay_StC + Reconnect_StC fused, wave by wave (8x8 groups => 2 waves of 8x4 lanes)
    void ReconnectStC(const Frame& f, const Params& prm, const zr_rpt_reservoir* resIn, zr_rpt_reservoir* resOut,
        const float4* target, float4* finalImg, const uint16_t* neighbor, const uint16_t* threadMap, int nthreads)
    {
        const zr_frame_constants& fc = *f.fc;
        const uint32_t dispX = (f.W + 7) / 8, dispY = (f.H + 7) / 8;
        parallel_for(dispX * dispY * 2, nthreads, [&](uint32_t w0, uint32_t w1)
        {
            for (uint32_t wv = w0; wv < w1; wv++)
            {
                const uint32_t g = wv / 2, wave = wv % 2;
                struct L { bool active; int x, y; size_t idx; Pixel p; Reservoir r; bool hasN; int nx, ny; Reservoir rs; uint32_t M_max, M_new;
                    int stage; bool changed; OffsetPath shift; };
                static thread_local std::vector<L> lanes;
                lanes.assign(32, L());
                float v[32];
                // ---- up to the first wave sum ----
                for (int l = 0; l < 32; l++)
                {
                    L& s = lanes[l];
                    LaneMap m = MapLane(f, g % dispX, g / dispX, l % 8, wave * 4 + l / 8, 8, 8, dispX, dispY, prm.sortSpatial != 0, threadMap);
                    s.active = false;
                    if (!m.active) continue;
                    GFlags flags = FlagsAt(f.core, f.W, m.x, m.y);
                    if (flags.invalid || flags.emissive) continue;
                    s.active = true; s.x = m.x; s.y = m.y; s.idx = (size_t)m.y * f.W + m.x;
                    s.p = LoadPixel(f, f.core, f.coat, m.x, m.y, false, m.x, m.y);
                    s.r = Reservoir::Load_NonReconnection(resIn[s.idx]);
                    s.r.target = f3(target[s.idx].x, target[s.idx].y, target[s.idx].z);
                    s.hasN = NeighborOf(f, neighbor, m.x, m.y, s.nx, s.ny);
                    s.stage = 0;
                }
                for (int l = 0; l < 32; l++) v[l] = lanes[l].active ? lanes[l].r.w_sum : 0.0f;
                float waveSum = WaveSum32(v);
                for (int l = 0; l < 32; l++) v[l] = lanes[l].active ? lanes[l].r.w_sum * (lanes[l].hasN ? 0.0f : 1.0f) : 0.0f;
                float waveSum2 = WaveSum32(v);
                // lanes without a neighbour finish here
                for (int l = 0; l < 32; l++)
                {
                    L& s = lanes[l];
                    if (!s.active) continue;
                    float waveAvgExclusive = (waveSum - s.r.w_sum) / 32.0f;
                    s.M_max = prm.M_max_spatial;
                    s.M_max = !s.r.rc.Empty() && s.r.rc.lobe_k_min_1 == BSDF::GLOSSY_T ? (s.M_max < 4 ? s.M_max : 4) : s.M_max;
                    if (!s.hasN)
                    {
                        if (prm.boilingSuppression) SuppressOutlier(waveAvgExclusive, s.r);
                        WriteOutputColor(fc, finalImg, s.idx, s.r.target * s.r.W);
                        CopyToNextFrame(resIn[s.idx], resOut[s.idx], s.r, s.M_max);
                        s.active = false;
                        continue;
                    }
                    s.rs = Reservoir::Load_NonReconnection(resIn[(size_t)s.ny * f.W + s.nx]);
                    if ((s.r.w_sum != 0) && (s.rs.M > 0) && !s.r.rc.Empty())
                        s.r.w_sum = resOut[s.idx].w_sum;        // LoadWSum: Reconnect_CtS's result
                    s.M_new = s.r.M + s.rs.M;
                }
                for (int l = 0; l < 32; l++) v[l] = lanes[l].active ? lanes[l].r.w_sum * (lanes[l].rs.rc.Empty() ? 1.0f : 0.0f) : 0.0f;
                float waveSum3 = WaveSum32(v);
                float waveSumAcc = waveSum2 + waveSum3;
                // The reference computes waveAvgExclusive once, before LoadWSum (Reconnect_StC.hlsl:221-222);
                // keep each lane's value from that point.
                float avgEx[32];
                for (int l = 0; l < 32; l++) avgEx[l] = 0;
                // recompute with the original (pre-LoadWSum) w_sum: it equals resIn's B.x
                for (int l = 0; l < 32; l++)
                    if (lanes[l].active) avgEx[l] = (waveSum - resIn[lanes[l].idx].w_sum) / 32.0f;
                for (int l = 0; l < 32; l++)
                {
                    L& s = lanes[l];
                    if (!s.active) continue;
                    if (s.rs.rc.Empty())
                    {
                        if (prm.boilingSuppression) SuppressOutlier(avgEx[l], s.r);
                        float targetLum = Math::Luminance(s.r.target);
                        s.r.W = targetLum > 0 ? s.r.w_sum / targetLum : 0;
                        s.r.M = s.M_new;
                        CopyToNextFrame(resIn[s.idx], resOut[s.idx], s.r, s.M_max);
                        WriteOutputColor(fc, finalImg, s.idx, s.r.target * s.r.W);
                        s.active = false;
                        continue;
                    }
                    s.M_max = s.rs.rc.x_k_in_motion ? (s.M_max < 4 ? s.M_max : 4) : s.M_max;
                    s.rs.rc.x_k_in_motion = false;
                    s.rs.Load_Reconnection(resIn[(size_t)s.ny * f.W + s.nx]);
                    OffsetPathContext ctx; const OffsetPathContext* pctx = nullptr;
                    if (s.rs.rc.k > 2)
                    {
                        ctx = Replay_kGt2(*f.sc, s.p.pos, s.p.normal, s.p.eta_next, s.p.surface, s.rs.rc, prm.alpha_min).Quantize();
                        pctx = &ctx;
                    }
                    s.shift = Shift2(*f.sc, s.p.pos, s.p.normal, s.p.eta_next, s.p.surface, s.rs.rc, pctx, prm.alpha_min);
                    float targetLum_curr = Math::Luminance(s.shift.target);
                    float targetLum_spatial = s.rs.W > 0 ? s.rs.w_sum / s.rs.W : 0;
                    float jacobian = s.rs.rc.partialJacobian > 0 ? s.shift.partialJacobian / s.rs.rc.partialJacobian : 0;
                    s.changed = false;
                    if (targetLum_curr > 1e-6f && jacobian > 1e-5f && jacobian < 100)
                    {
                        uint3 h = RNG::PCG3d(uint3{ (uint32_t)s.x, (uint32_t)s.y, (uint32_t)s.y });
                        RNG rng = RNG::Init(h.x, h.z, fc.FrameNum + 511);
                        float numerator = (float)s.rs.M * targetLum_spatial;
                        float denom = numerator / jacobian + (float)s.r.M * targetLum_curr;
                        float m_spatial = denom > 0 ? numerator / denom : 0;
                        float w_spatial = m_spatial * s.rs.W * targetLum_curr;
                        if (s.r.Update(w_spatial, s.shift.target, s.rs.rc, rng))
                        {
                            s.r.rc.partialJacobian = s.shift.partialJacobian;
                            s.changed = true;
                        }
                    }
                    float targetLum = Math::Luminance(s.r.target);
                    s.r.W = targetLum > 0 ? s.r.w_sum / targetLum : 0;
                    s.r.M = s.M_new;
                }
                if (prm.boilingSuppression)
                {
                    for (int l = 0; l < 32; l++) v[l] = lanes[l].active ? lanes[l].r.w_sum : 0.0f;
                    float waveSum4 = WaveSum32(v);
                    float total = waveSumAcc + waveSum4;
                    for (int l = 0; l < 32; l++)
                        if (lanes[l].active)
                            SuppressOutlier((total - lanes[l].r.w_sum) / 32.0f, lanes[l].r);
                }
                for (int l = 0; l < 32; l++)
                {
                    L& s = lanes[l];
                    if (!s.active) continue;
                    if (s.changed)
                    {
                        uint32_t M_max = s.shift.surfKMin1Tramsmissive ? (s.M_max < 4 ? s.M_max : 4) : s.M_max;
                        s.r.Write(resOut[s.idx], M_max);
                    }
                    else
                        CopyToNextFrame(resIn[s.idx], resOut[s.idx], s.r, s.M_max);
                    WriteOutputColor(fc, finalImg, s.idx, s.r.target * s.r.W);
                }
            }
        });
    }
}

extern "C"
{
    void orc_rpt_set_sample_pattern(const float* pattern512x2) { g_samplePattern = pattern512x2; }

    // One IndirectLighting::Render. state[0] = currTemporalIdx, state[1] = isTemporalReservoirValid,
    // state[2] = reset-temporal-textures flag (all updated). last_stage: 0 = whole frame, 1 = stop after
    // PathTrace, 2 = after temporal, 3 = after spatial.
    void orc_rpt_render(void* scene_, const zr_frame_constants* fc, const uint32_t* core_, const uint32_t* me_, const uint32_t* coat_,
        const uint32_t* pcore_, const uint32_t* pcoat_, const zr_indirect_params* p, orc_rpt_buffers* b, uint32_t* state, int last_stage, int nthreads)
    {
        const uint4* core = (const uint4*)core_;
        const uint2* me = (const uint2*)me_;
        const uint2* coat = (const uint2*)coat_;
        const uint4* pcore = (const uint4*)pcore_;
        const uint2* pcoat = (const uint2*)pcoat_;
        float4* target = (float4*)b->target;
        float4* finalImg = (float4*)b->finalImg;
        Frame f;
        f.sc = (Scene*)scene_; f.fc = fc; f.core = core; f.me = me; f.coat = coat; f.pcore = pcore; f.pcoat = pcoat;
        f.W = fc->RenderWidth; f.H = fc->RenderHeight;
        Params prm;
        prm.maxNonTrBounces = p->max_non_tr_bounces; prm.maxGlossyTrBounces = p->max_glossy_tr_bounces;
        prm.russianRoulette = p->russian_roulette; prm.M_max_temporal = p->M_max_temporal; prm.M_max_spatial = p->M_max_spatial;
        prm.boilingSuppression = p->boiling_suppression; prm.sortTemporal = p->sort_temporal; prm.sortSpatial = p->sort_spatial;
        prm.alpha_min = p->alpha_min;

        uint32_t cur = state[0];
        const bool doTemporal = p->temporal_resample && state[1];
        const bool doSpatial = (p->num_spatial_passes > 0) && doTemporal;
        zr_rpt_reservoir* resCurr = b->res[cur];
        zr_rpt_reservoir* resPrev = b->res[1 - cur];

        PathTracePass(f, prm, doTemporal, state[2] != 0, resCurr, target, finalImg, nthreads);
        if (doTemporal && last_stage != 1)
        {
            if (prm.sortTemporal)
            {
                SortPass(f, 1, doSpatial, resCurr, resPrev, nullptr, b->threadMapNtC);
                SortPass(f, 0, doSpatial, resCurr, resPrev, nullptr, b->threadMapCtN);
            }
            ReconnectCtT(f, prm, resCurr, resPrev, b->threadMapCtN, nthreads);
            ReconnectTtC(f, prm, doSpatial, resCurr, resPrev, target, finalImg, b->threadMapNtC, nthreads);
        }
        if (doSpatial && last_stage != 1 && last_stage != 2)
        {
            for (uint32_t pass = 0; pass < p->num_spatial_passes; pass++)
            {
                SpatialSearchPass(f, b->neighbor, nthreads);
                zr_rpt_reservoir* in = b->res[cur];
                zr_rpt_reservoir* out = b->res[1 - cur];
                cur = 1 - cur;
                if (prm.sortSpatial)
                {
                    SortPass(f, 2, true, in, nullptr, b->neighbor, b->threadMapCtN);
                    SortPass(f, 3, true, in, nullptr, b->neighbor, b->threadMapNtC);
                }
                ReconnectCtS(f, prm, in, out, b->neighbor, b->threadMapCtN, nthreads);
                ReconnectStC(f, prm, in, out, target, finalImg, b->neighbor, b->threadMapNtC, nthreads);
            }
        }
        state[1] = 1;
        state[0] = 1 - cur;
        state[2] = 0;
    }
}
