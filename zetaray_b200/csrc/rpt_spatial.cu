// rpt_spatial.cu -- ReSTIR PT spatial reuse as classify -> per-case shift queues -> TMA-staged streaming merge.
//
// Replaces ReSTIR_PT_Replay x2, ReSTIR_PT_Reconnect_CtS.hlsl:46-230 and ReSTIR_PT_Reconnect_StC.hlsl:150-352 and produces the oracle's
// bytes; the execution model is described in zr_rpt_spatial.h.
//
// Why the split: a fused kernel evaluates two hybrid shifts inline per pixel, so a warp idles on sky pixels, on pixels without a
// neighbour, on the other reconnection cases' phases (17 of 32 lanes active on the Cornell frame, 9 on the tunnel), and the 128 k
// instructions of both shifts + merge share one register allocation. Here
//   * the shifts run from queues holding (pixel, direction) items of ONE reconnection case and replay class, drained by
//     persistent blocks: every lane of every warp has work and the other cases' phases do not exist in the kernel;
//   * what remains per pixel -- MIS weights, reservoir update, boiling suppression, the 64-byte record and the colour -- is a
//     bandwidth-bound pass: the block's 32x32 tile of reservoirs arrives by TMA (cp.async.bulk.tensor.2d, double buffered, one
//     mbarrier per stage) while the previous tile is merged, every other access is a coalesced 128-bit row segment, and the wave
//     sums of the boiling filter are taken over the SAME 32 pixels as in the reference's sorted dispatch by routing the four
//     per-pixel terms through shared memory (pixel order -> sorted thread order -> xor-butterfly -> back).
#include "zr_rpt_spatial.h"
#include "zr_rpt_shift.cuh"
#include "zr_tma.cuh"

namespace zr
{
namespace
{
    using namespace RPT;

    // ---------------------------------------------------------------------------------------------------------------
    // classify: one thread per pixel of the owned rows
    // ---------------------------------------------------------------------------------------------------------------
    __global__ void __launch_bounds__(256) k_spatial_classify(FrameView f, RptParams prm, const zr_rpt_reservoir* __restrict__ resIn,
        const uint16_t* __restrict__ neighbor, uint32_t* __restrict__ queue, uint32_t* __restrict__ counters, uint32_t capacity)
    {
        __shared__ uint32_t s_count[SpatialQueued::NUM_CLASSES], s_base[SpatialQueued::NUM_CLASSES];
        const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31);
        const uint32_t y = prm.rowBegin + blockIdx.y * 8 + (threadIdx.x >> 5);
        if (threadIdx.x < SpatialQueued::NUM_CLASSES) s_count[threadIdx.x] = 0;
        __syncthreads();
        uint32_t cls[2] = { NO_ITEM, NO_ITEM };     // [0] current -> neighbour (CtS), [1] neighbour -> current (StC)
        if (x < f.W && y < f.H && y < prm.rowEnd)
        {
            const GFlags flags = FlagsAt(f.core, f.W, (int)x, (int)y);
            int nx = 0, ny = 0;
            if (!(flags.invalid || flags.emissive) && NeighborOf(f, neighbor, (int)x, (int)y, nx, ny))
            {
                const uint4 q0 = ld128(&resIn[(size_t)y * f.W + x]);
                const uint4 qn = ld128(&resIn[(size_t)ny * f.W + nx]);
                const bool selfEmpty = (q0.x & 0xf) == Reconnection::EMPTY, nEmpty = (qn.x & 0xf) == Reconnection::EMPTY;
                const uint32_t M_n = (qn.x >> 4) & 0xf;
                if (asfloat(q0.y) != 0 && !selfEmpty && M_n > 0) cls[0] = ShiftClass(q0.x);
                if (!nEmpty) cls[1] = ShiftClass(qn.x);
            }
        }
        const uint32_t item[2] = { x | (y << 16), x | (y << 16) | (1u << 31) };
        AppendItems(cls, item, queue, counters, capacity, s_count, s_base);
    }

    // ---------------------------------------------------------------------------------------------------------------
    // merge: persistent blocks, one 32x32 tile per iteration
    // ---------------------------------------------------------------------------------------------------------------
    struct MergeSmem
    {
        uint4 rec[2][1024][4];      // stage x pixel-of-tile x 64-byte record (TMA destination: 32 rows of 2048 bytes)
        float val[2][1024];         // [0] w_sum on entry, [1] the pixel's term of the final sum
        float sum[2][1024];         // [0] wave sum of val[0], [1] wave total of the final sums
        uint8_t cls[1024];          // which of the three final sums the pixel contributes to (0 = none)
        uint8_t visited[1024];      // a thread position of the sorted dispatch maps to this pixel
        unsigned long long bar[2];
    };

    __global__ void __launch_bounds__(1024, 1) k_spatial_merge(const CUtensorMap* __restrict__ pMapIn, FrameView f, RptParams prm,
        const zr_rpt_reservoir* __restrict__ resIn, zr_rpt_reservoir* __restrict__ resOut, const float4* __restrict__ target,
        float4* __restrict__ finalImg, const uint16_t* __restrict__ neighbor, const uint16_t* __restrict__ threadMap,
        const ShiftResult* __restrict__ shiftRes, uint32_t tilesX, uint32_t tileRow0, uint32_t numTiles, uint32_t swizzled)
    {
        extern __shared__ __align__(1024) unsigned char smemRaw[];
        MergeSmem& sm = *reinterpret_cast<MergeSmem*>(smemRaw);
        const zr_frame_constants& fc = f.fc;
        const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
        constexpr uint32_t TILE_BYTES = 1024 * 64;

        if (t == 0)
        {
            tma::MbarInit(reinterpret_cast<uint64_t*>(&sm.bar[0]), 1);
            tma::MbarInit(reinterpret_cast<uint64_t*>(&sm.bar[1]), 1);
            tma::FenceBarrierInit();
        }
        __syncthreads();
        auto issue = [&](uint32_t tile, uint32_t stage)
        {
            const uint32_t tx = tile % tilesX, ty = tileRow0 + tile / tilesX;
            uint64_t* bar = reinterpret_cast<uint64_t*>(&sm.bar[stage]);
            tma::MbarArriveExpectTx(bar, TILE_BYTES);
            if (swizzled) tma::Load3D(&sm.rec[stage][0][0], pMapIn, bar, 0, (int32_t)(tx * 16), (int32_t)(ty * 32));
            else tma::Load2D(&sm.rec[stage][0][0], pMapIn, bar, (int32_t)(tx * 32 * 8), (int32_t)(ty * 32));
        };
        if (t == 0 && blockIdx.x < numTiles)
            issue(blockIdx.x, 0);

        // Software pipeline across tiles: the first-level loads of a tile (flag word, neighbour code, target; thread-map entry of the
        // thread position this thread plays in phase 2) are issued one iteration ahead and carried in registers, so that at the top of
        // an iteration the dependent gathers (neighbour record, shift results) go out at once.
        uint32_t pfFlags = 0xff, pfNb = 0xffff, pfMap = 0x8000;
        float4 pfTg = f4(0, 0, 0, 0);
        auto prefetch = [&](uint32_t tile)
        {
            const uint32_t tX = tile % tilesX, tY = tileRow0 + tile / tilesX;
            const uint32_t px = tX * 32 + lane, py = tY * 32 + warp;
            pfFlags = 0xff; pfNb = 0xffff; pfMap = 0x8000;      // invalid | emissive, no neighbour, thread position without a pixel
            if (px < f.W && py < f.H && py >= prm.rowBegin && py < prm.rowEnd)
            {
                const size_t i = (size_t)py * f.W + px;
                pfFlags = __ldg(&f.core[i].w) & 0xff;
                pfNb = __ldg(&neighbor[i]);
                pfTg = __ldg(&target[i]);
            }
            const uint32_t sx = tX * 32 + (warp & 3) * 8 + (lane & 7), sy = tY * 32 + (warp >> 2) * 4 + (lane >> 3);
            if (sx < f.W && sy < f.H)
                pfMap = prm.sortSpatial ? __ldg(&threadMap[(size_t)sy * f.W + sx]) : (31u | (31u << 7));
        };
        if (blockIdx.x < numTiles)
            prefetch(blockIdx.x);

        uint32_t it = 0;
        for (uint32_t tile = blockIdx.x; tile < numTiles; tile += gridDim.x, it++)
        {
            const uint32_t stage = it & 1, parity = (it >> 1) & 1;
            const uint32_t tileX = tile % tilesX, tileY = tileRow0 + tile / tilesX;
            // prefetch the next tile into the other stage (its readers finished at the end of the previous iteration)
            if (t == 0 && tile + gridDim.x < numTiles)
            {
                tma::FenceProxyAsync();
                issue(tile + gridDim.x, stage ^ 1);
            }
            // ---- phase 1 (pixel order): everything but the wave sums ----
            const int x = (int)(tileX * 32 + lane), y = (int)(tileY * 32 + warp);
            const bool inImage = (uint32_t)x < f.W && (uint32_t)y < f.H;
            const size_t idx = inImage ? (size_t)y * f.W + x : 0;
            bool act = false;
            {
                const GFlags flags = DecodeFlags(pfFlags);
                act = !(flags.invalid || flags.emissive);       // out-of-strip / out-of-image pixels were prefetched as invalid
            }
            int nx = 0, ny = 0;
            bool hasN = false;
            const float4 tg = pfTg;
            const uint32_t mapEnc = pfMap;
            uint4 sh0 = make_uint4(0, 0, 0, 0);
            float2 sh1 = f2(0, 0);
            uint4 n0 = make_uint4(Reconnection::EMPTY, 0, 0, 0), n1 = make_uint4(0, 0, 0, 0);
            if (act)
            {
                const uint32_t ox = pfNb & 0xff, oy = pfNb >> 8;
                hasN = ox != 0xff;
                nx = (int)ox - 32 + x; ny = (int)oy - 32 + y;
                if (hasN)
                {
                    const uint4* nrec = reinterpret_cast<const uint4*>(&resIn[(size_t)ny * f.W + nx]);
                    n0 = __ldg(&nrec[0]); n1 = __ldg(&nrec[1]);
                    // second half of the neighbour's record (read only if its sample is accepted, after the RNG draw): brought into L1 now so
                    // that the slowest warp of the block does not add a second gather round trip before the barrier
                    asm volatile("prefetch.global.L1 [%0];" :: "l"(nrec + 2));
                    const uint4* sp = reinterpret_cast<const uint4*>(&shiftRes[idx]);
                    sh0 = __ldg(&sp[0]);
                    sh1 = __ldg(reinterpret_cast<const float2*>(&sp[1]));
                }
            }
            if (tile + gridDim.x < numTiles)
                prefetch(tile + gridDim.x);
            sm.visited[t] = 0;
            tma::MbarWait(reinterpret_cast<uint64_t*>(&sm.bar[stage]), parity);

            zr_rpt_reservoir rec;
            {
                // the record pair of pixels (2p, 2p + 1) is one 128-byte line; with the swizzled map its 16-byte chunk c sits at c ^ (p & 7)
                const uint4* line = &sm.rec[stage][t & ~1u][0];
                const uint32_t c0 = (t & 1u) * 4u, sw = swizzled ? ((t >> 1) & 7u) : 0u;
                uint4 v[4] = { line[(c0 + 0) ^ sw], line[(c0 + 1) ^ sw], line[(c0 + 2) ^ sw], line[(c0 + 3) ^ sw] };
                memcpy(&rec, v, 64);
            }
            Reservoir r_curr = Reservoir::Load_NonReconnection(rec);
            r_curr.target = f3(tg.x, tg.y, tg.z);
            const float wsum0 = act ? r_curr.w_sum : 0.0f;
            uint32_t M_max = prm.M_max_spatial;
            M_max = !r_curr.rc.Empty() && r_curr.rc.lobe_k_min_1 == BSDF::GLOSSY_T ? (M_max < 4 ? M_max : 4) : M_max;
            // class 1: no neighbour; class 2: neighbour's reservoir holds no sample; class 3: full merge
            uint32_t cls = 0, M_new = 0;
            bool changed = false, surfKMin1Tr = false;
            zr_rpt_reservoir recN;
            Reservoir r_spatial = Reservoir::Init();
            if (act && !hasN)
                cls = 1;
            else if (act)
            {
                memset(&recN, 0, sizeof(recN));
                memcpy(&recN, &n0, 16); memcpy(reinterpret_cast<unsigned char*>(&recN) + 16, &n1, 16);
                r_spatial = Reservoir::Load_NonReconnection(recN);
                // Reconnect_CtS: MIS weight of the current sample among (current, neighbour)
                if ((r_curr.w_sum != 0) && !r_curr.rc.Empty() && (r_spatial.M > 0))
                {
                    const float target_spatial = sh1.x;
                    if (target_spatial > 0)
                    {
                        const float selfJ = (r_curr.rc.IsCase3() && r_curr.rc.lobe_k_min_1 == BSDF::ALL) ? 1.0f : asfloat(rec.jacobian_or_seed_nee);
                        const float targetLum_curr = r_curr.W > 0 ? r_curr.w_sum / r_curr.W : 0;
                        const float jacobian = selfJ > 0 ? sh1.y / selfJ : 0;
                        const float numerator = (float)r_curr.M * targetLum_curr;
                        const float denom = numerator + (float)r_spatial.M * target_spatial * jacobian;
                        const float m_curr = denom > 0 ? numerator / denom : 0;
                        r_curr.w_sum *= m_curr;
                    }
                }
                M_new = r_curr.M + r_spatial.M;
                if (r_spatial.rc.Empty())
                    cls = 2;                // W and M are set after the outlier test (phase 3)
                else
                {
                    cls = 3;
                    M_max = r_spatial.rc.x_k_in_motion ? (M_max < 4 ? M_max : 4) : M_max;
                    r_spatial.rc.x_k_in_motion = false;
                    const float nJ = (r_spatial.rc.IsCase3() && r_spatial.rc.lobe_k_min_1 == BSDF::ALL) ? 1.0f : asfloat(recN.jacobian_or_seed_nee);
                    const float3 shTarget = f3(asfloat(sh0.x), asfloat(sh0.y), asfloat(sh0.z));
                    const float shJ = fabsf(asfloat(sh0.w));
                    surfKMin1Tr = (sh0.w >> 31) != 0;
                    const float targetLum_curr = Math::Luminance(shTarget);
                    const float targetLum_spatial = r_spatial.W > 0 ? r_spatial.w_sum / r_spatial.W : 0;
                    const float jacobian = nJ > 0 ? shJ / nJ : 0;
                    if (targetLum_curr > 1e-6f && jacobian > 1e-5f && jacobian < 100)
                    {
                        const uint3 h = RNG::PCG3d(make_uint3((uint32_t)x, (uint32_t)y, (uint32_t)y));
                        RNG rng = RNG::Init(h.x, h.z, fc.FrameNum + 511);
                        const float numerator = (float)r_spatial.M * targetLum_spatial;
                        const float denom = numerator / jacobian + (float)r_curr.M * targetLum_curr;
                        const float m_spatial = denom > 0 ? numerator / denom : 0;
                        const float w_spatial = m_spatial * r_spatial.W * targetLum_curr;
                        if (r_curr.Update(w_spatial, shTarget, r_spatial.rc, rng))
                        {
                            // the accepted sample is the neighbour's: the rest of its record (second 32 bytes)
                            const uint4* nrec = reinterpret_cast<const uint4*>(&resIn[(size_t)ny * f.W + nx]);
                            const uint4 n2 = __ldg(&nrec[2]), n3 = __ldg(&nrec[3]);
                            memcpy(reinterpret_cast<unsigned char*>(&recN) + 32, &n2, 16);
                            memcpy(reinterpret_cast<unsigned char*>(&recN) + 48, &n3, 16);
                            r_spatial.Load_Reconnection(recN);
                            r_curr.rc = r_spatial.rc;
                            r_curr.rc.partialJacobian = shJ;
                            changed = true;
                        }
                    }
                    const float targetLum = Math::Luminance(r_curr.target);
                    r_curr.W = targetLum > 0 ? r_curr.w_sum / targetLum : 0;
                    r_curr.M = M_new;
                }
            }
            sm.val[0][t] = wsum0;
            sm.val[1][t] = act ? r_curr.w_sum : 0.0f;
            sm.cls[t] = (uint8_t)cls;
            __syncthreads();

            // ---- phase 2 (sorted thread order): thread position -> pixel, xor-butterfly over the reference's waves ----
            {
                const int sx = (int)(tileX * 32 + (warp & 3) * 8 + (lane & 7)), sy = (int)(tileY * 32 + (warp >> 2) * 4 + (lane >> 3));
                bool on = (uint32_t)sx < f.W && (uint32_t)sy < f.H;
                int lx = sx - (int)(tileX * 32), ly = sy - (int)(tileY * 32);
                if (mapEnc & (1u << 15)) on = false;        // error bit (or a position outside the image: prefetched as such)
                lx += (int)(mapEnc & 0x3f) - 31;
                ly += (int)((mapEnc >> 7) & 0x3f) - 31;
                if (on && ((uint32_t)lx >= 32u || (uint32_t)ly >= 32u)) on = false;      // cannot happen: the sort permutes within a tile
                const uint32_t lp = on ? (uint32_t)(ly * 32 + lx) : 0;
                const float v0 = on ? sm.val[0][lp] : 0.0f, v1 = on ? sm.val[1][lp] : 0.0f;
                const uint32_t c = on ? sm.cls[lp] : 0;
                const float waveSum = WaveSum32(v0);
                float waveAcc = WaveSum32(c == 1 ? v1 : 0.0f);
                waveAcc += WaveSum32(c == 2 ? v1 : 0.0f);
                const float total = waveAcc + WaveSum32(c == 3 ? v1 : 0.0f);
                if (on)
                {
                    sm.sum[0][lp] = waveSum; sm.sum[1][lp] = total;
                    sm.visited[lp] = 1;
                }
            }
            __syncthreads();

            // ---- phase 3 (pixel order): boiling suppression, record, colour ----
            if (act && sm.visited[t])
            {
                const float avgEx0 = (sm.sum[0][t] - wsum0) / 32.0f;
                if (cls == 1)
                {
                    if (prm.boilingSuppression) SuppressOutlier(avgEx0, r_curr);
                    WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
                    CopyToNextFrame(rec, &resOut[idx], r_curr, M_max);
                }
                else if (cls == 2)
                {
                    if (prm.boilingSuppression) SuppressOutlier(avgEx0, r_curr);
                    const float targetLum = Math::Luminance(r_curr.target);
                    r_curr.W = targetLum > 0 ? r_curr.w_sum / targetLum : 0;
                    r_curr.M = M_new;
                    CopyToNextFrame(rec, &resOut[idx], r_curr, M_max);
                    WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
                }
                else
                {
                    if (prm.boilingSuppression)
                        SuppressOutlier((sm.sum[1][t] - r_curr.w_sum) / 32.0f, r_curr);
                    if (changed)
                    {
                        const uint32_t mmax = surfKMin1Tr ? (M_max < 4 ? M_max : 4) : M_max;
                        zr_rpt_reservoir out;
                        r_curr.Write(out, mmax);
                        StoreRecord(&resOut[idx], out);
                    }
                    else
                        CopyToNextFrame(rec, &resOut[idx], r_curr, M_max);
                    WriteOutputColor(fc, finalImg, idx, r_curr.target * r_curr.W);
                }
            }
            __syncthreads();        // the stage's records and the exchange arrays are free again
        }
    }
}

// -------------------------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------------------------
zr_status ShiftStreams::Init()
{
    int dev = 0;
    ZR_CUDA(cudaGetDevice(&dev));
    ZR_CUDA(cudaDeviceGetAttribute(&numSMs, cudaDevAttrMultiProcessorCount, dev));
    ZR_CUDA(cudaFuncSetAttribute(k_spatial_merge, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MergeSmem)));
    ZR_TRY(SetupShifts<false>());
    ZR_TRY(SetupTemporalShifts());
    // the greatest priority: in the renderer's frame the shift stages are on the critical path, and DirectLighting runs beside them at
    // the least (renderer.cu); a pass driven on a stream of the default priority loses nothing by it
    int leastPriority = 0, greatestPriority = 0;
    ZR_CUDA(cudaDeviceGetStreamPriorityRange(&leastPriority, &greatestPriority));
    for (int i = 0; i < 2; i++)
    {
        ZR_CUDA(cudaStreamCreateWithPriority(&aux[i], cudaStreamNonBlocking, greatestPriority));
        ZR_CUDA(cudaEventCreateWithFlags(&evJoin[i], cudaEventDisableTiming));
    }
    ZR_CUDA(cudaEventCreateWithFlags(&evFork, cudaEventDisableTiming));
    return ZR_OK;
}

ShiftStreams::~ShiftStreams()
{
    for (int i = 0; i < 2; i++)
    {
        if (aux[i]) cudaStreamDestroy(aux[i]);
        if (evJoin[i]) cudaEventDestroy(evJoin[i]);
    }
    if (evFork) cudaEventDestroy(evFork);
}

zr_status SpatialQueued::Build(uint32_t w, uint32_t h, const zr_rpt_reservoir* res0, const zr_rpt_reservoir* res1)
{
    width = w; height = h;
    const size_t n = (size_t)w * h;
    capacity = 2 * n;
    ZR_TRY(planes.Alloc(d_queue, NUM_CLASSES * capacity, false));
    ZR_TRY(planes.Alloc(d_counters, 16, false));
    ZR_TRY(planes.Alloc(d_shift, n));
    ZR_TRY(planes.Alloc(d_flags, n));
    ZR_TRY(planes.Alloc(d_maps, 2, false));
    const zr_rpt_reservoir* res[2] = { res0, res1 };
    CUtensorMap maps[2];
    swizzled = (w % 2) == 0;
    for (int i = 0; i < 2; i++)
    {
        mapBase[i] = res[i];
        bool ok;
        if (swizzled)
        {
            const uint64_t dims[3] = { 16, w / 2, h };
            const uint64_t strides[2] = { 128, (uint64_t)w * 64 };
            const uint32_t box[3] = { 16, 16, 32 };
            ok = tma::EncodeWords(&maps[i], res[i], 3, dims, strides, box, true);
        }
        else
            ok = tma::EncodePlane2D(&maps[i], res[i], w, h, 64, (uint64_t)w * 64, 32, 32);
        if (!ok)
        {
            set_error("zr_indirect_pass: cuTensorMapEncodeTiled failed for the %ux%u reservoir plane", w, h);
            return ZR_ERR_CUDA;
        }
    }
    ZR_CUDA(cudaMemcpy(d_maps, maps, sizeof(maps), cudaMemcpyHostToDevice));
    return planes.Clear();
}

zr_status SpatialQueued::Run(const ShiftStreams& ss, const SceneDev& sc, const FrameView& f, const RptParams& prm, const zr_rpt_reservoir* resIn,
    zr_rpt_reservoir* resOut, const float4* target, float4* finalImg, const uint16_t* neighbor, const uint16_t* threadMap, bool plain, cudaStream_t stream)
{
    const int plane = resIn == mapBase[0] ? 0 : (resIn == mapBase[1] ? 1 : -1);
    if (plane < 0) { set_error("zr_indirect_pass: spatial input is not one of the pass's reservoir planes"); return ZR_ERR_INVALID_ARG; }
    const uint32_t rows = prm.rowEnd - prm.rowBegin;
    ZR_CUDA(cudaMemsetAsync(d_counters, 0, 16 * sizeof(uint32_t), stream));
    {
        ZR_PROF("k_spatial_classify", stream);
        k_spatial_classify<<<dim3((width + 31) / 32, (rows + 7) / 8), 256, 0, stream>>>(f, prm, resIn, neighbor, d_queue, d_counters, (uint32_t)capacity);
        ZR_LAUNCH_CHECK();
    }
    {
        ZR_PROF("k_shift", stream);
        const zr_status ls = LaunchShifts<false>(*this, ss, sc, f, prm, resIn, nullptr, neighbor, plain, stream);
        zr::prof_after();
        if (ls != ZR_OK) return ls;
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return zr::cuda_fail(e, "k_shift launch");
    }
    {
        const uint32_t tilesX = (width + 31) / 32;
        const uint32_t tileRow0 = prm.rowBegin / 32, tileRow1 = (prm.rowEnd + 31) / 32;
        const uint32_t numTiles = tilesX * (tileRow1 - tileRow0);
        // A second form -- 512 threads x 2 co-resident blocks per SM, per-pixel state parked in shared memory between the phases -- was
        // bit-identical and no faster: the kernel waits for its global loads at 32 warps per
        // SM in either form. Removed again.
        const uint32_t grid = numTiles < (uint32_t)ss.numSMs ? numTiles : (uint32_t)ss.numSMs;
        ZR_PROF("k_spatial_merge", stream);
        k_spatial_merge<<<grid, 1024, sizeof(MergeSmem), stream>>>(d_maps + plane, f, prm, resIn, resOut, target, finalImg, neighbor, threadMap,
            d_shift, tilesX, tileRow0, numTiles, swizzled ? 1u : 0u);
        ZR_LAUNCH_CHECK();
    }
    return ZR_OK;
}
} // namespace zr
