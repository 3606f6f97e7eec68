// zr_rpt_spatial.h -- host interface of the queued spatial-reuse path (rpt_spatial.cu), used by zr_indirect_pass (rpt.cu).
//
// ReSTIR PT spatial reuse (Reconnect_CtS + Reconnect_StC with their replays, IndirectLighting.cpp:686-870) as
//   k_spatial_classify   per pixel: which of the two shifts (current -> neighbour, neighbour -> current) are needed at all, and
//                        their reconnection case / replay class; appends (pixel, direction) items to one queue per class
//   k_shift<case,replay> persistent blocks drain one queue each: every thread of a block runs the same shift code path on a
//                        full warp of work (no idle lanes for sky / empty / other-case pixels); result = 16 or 8 bytes per item
//   k_spatial_merge      streaming merge in pixel order: TMA-staged 32x32 tiles of 64-byte reservoirs, the MIS weights, the
//                        reservoir update, boiling-suppression wave sums taken in the sorted thread order through shared memory
// Results are bit-identical to the oracle.
#pragma once
#include <cuda.h>
#include "zr_planes.h"
#include "zr_rpt_io.cuh"

namespace zr
{
// per-pixel results of the two shifts: StC = neighbour's sample shifted to this pixel, CtS = this pixel's sample at the neighbour
struct ShiftResult
{
    float stcTarget[3];
    float stcJacobian;      // partial Jacobian of the shifted path; sign bit = x_{k-1} of the shifted path is transmissive
    float ctsTargetLum;
    float ctsJacobian;
    uint32_t pad[2];
};
static_assert(sizeof(ShiftResult) == 32, "ShiftResult is two 128-bit words");

// What the shift launches need whatever the frame size: created once with the pass (Init, which also sets k_spatial_merge's shared
// memory limit), released with it. The six class launches of a shift stage are independent (own queue, own claim cursor, disjoint result
// bytes): they are spread over the caller's stream and two forked ones of the greatest priority, so that short queues -- small classes,
// strip-sharded frames -- run side by side.
struct ShiftStreams
{
    int numSMs = 0;
    cudaStream_t aux[2] = { nullptr, nullptr };
    cudaEvent_t evFork = nullptr, evJoin[2] = { nullptr, nullptr };
    ShiftStreams() = default;
    ShiftStreams(const ShiftStreams&) = delete;
    ShiftStreams& operator=(const ShiftStreams&) = delete;
    ~ShiftStreams();
    zr_status Init();       // also sets up the shift kernels of both passes (SetupShifts in zr_rpt_shift.cuh)
};
// SetupShifts<true>: the temporal pass's shift kernels are instantiated in rpt_temporal.cu
zr_status SetupTemporalShifts();

// bits of SpatialQueued::d_flags
enum : uint8_t { TF_OK = 1, TF_REPLAY_OK = 2 };

// The queues, shift results and tensor maps of one frame size. Temporal reuse runs through the same queues, counters and shift-result
// plane (the two passes never overlap in a frame).
struct SpatialQueued
{
    static constexpr int NUM_CLASSES = 6;       // (case 1, 2, 3) x (k == 2, k > 2)
    Planes planes{ "zr_indirect_pass" };        // Build clears the shift results and the temporal flags, nothing else
    uint32_t width = 0, height = 0;
    uint32_t* d_queue = nullptr;                // NUM_CLASSES x capacity items: x | y << 16 | direction << 31
    uint32_t* d_counters = nullptr;             // [c] = items queued, [8 + c] = claim cursor of the persistent blocks
    ShiftResult* d_shift = nullptr;
    uint8_t* d_flags = nullptr;                 // temporal, per pixel: bit 0 = reuse valid, bit 1 = the replay's tighter plane test passed
    size_t capacity = 0;
    const void* mapBase[2] = { nullptr, nullptr };
    CUtensorMap* d_maps = nullptr;              // the two reservoir planes as [H][W] x 64 B, 32x32-pixel boxes (read from global memory)
    bool swizzled = false;                      // even widths: 3-D map {128-byte record pair, W / 2, H} with the 128-byte swizzle

    zr_status Build(uint32_t w, uint32_t h, const zr_rpt_reservoir* res0, const zr_rpt_reservoir* res1);
    // resIn must be one of the two planes given to Build. plain: the scene's materials use none of the features of BSDF::MF_ALL, so
    // the shifts run the kernels compiled without them.
    zr_status Run(const ShiftStreams& ss, const SceneDev& sc, const FrameView& f, const RptParams& prm, const zr_rpt_reservoir* resIn,
        zr_rpt_reservoir* resOut, const float4* target, float4* finalImg, const uint16_t* neighbor, const uint16_t* threadMap, bool plain,
        cudaStream_t stream);
    zr_status RunTemporal(const ShiftStreams& ss, const SceneDev& sc, const FrameView& f, const RptParams& prm, zr_rpt_reservoir* resCurr,
        const zr_rpt_reservoir* resPrev, float4* target, float4* finalImg, bool plain, cudaStream_t stream);
};
} // namespace zr
