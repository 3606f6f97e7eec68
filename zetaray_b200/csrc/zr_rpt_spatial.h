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

struct SpatialQueued
{
    static constexpr int NUM_CLASSES = 6;       // (case 1, 2, 3) x (k == 2, k > 2)
    uint32_t width = 0, height = 0;
    uint32_t* d_queue = nullptr;                // NUM_CLASSES x capacity items: x | y << 16 | direction << 31
    uint32_t* d_counters = nullptr;             // [c] = items queued, [8 + c] = claim cursor of the persistent blocks
    ShiftResult* d_shift = nullptr;
    size_t capacity = 0;
    CUtensorMap mapRes[2];                      // the two reservoir planes as [H][W] x 64 B, 32x32-pixel boxes
    const void* mapBase[2] = { nullptr, nullptr };
    CUtensorMap* d_maps = nullptr;              // device copy of mapRes (the kernel reads the descriptor from global memory)
    int numSMs = 0;
    bool ready = false;
    // the six class launches of a shift stage are independent (own queue, own claim cursor, disjoint result bytes): they are spread over
    // the caller's stream and two forked ones, so that short queues -- small classes, strip-sharded frames -- run side by side
    cudaStream_t aux[2] = { nullptr, nullptr };
    cudaEvent_t evFork = nullptr, evJoin[2] = { nullptr, nullptr };
    bool swizzled = false;                      // even widths: 3-D map {128-byte record pair, W / 2, H} with the 128-byte swizzle

    zr_status Resize(uint32_t w, uint32_t h, const zr_rpt_reservoir* res0, const zr_rpt_reservoir* res1);
    void Release();
    // resIn must be one of the two planes given to Resize
    zr_status Run(const SceneDev& sc, const FrameView& f, const RptParams& prm, const zr_rpt_reservoir* resIn, zr_rpt_reservoir* resOut,
        const float4* target, float4* finalImg, const uint16_t* neighbor, const uint16_t* threadMap, cudaStream_t stream);
};

// Temporal reuse through the same queues, counters and shift-result plane (the two passes never overlap in a frame).
struct TemporalQueued
{
    uint8_t* d_flags = nullptr;     // per pixel: bit 0 = temporal reuse valid, bit 1 = the replay's tighter plane test passed
    zr_status Resize(uint32_t w, uint32_t h);
    void Release();
    zr_status Run(SpatialQueued& q, const SceneDev& sc, const FrameView& f, const RptParams& prm, zr_rpt_reservoir* resCurr,
        const zr_rpt_reservoir* resPrev, float4* target, float4* finalImg, cudaStream_t stream);
};
} // namespace zr
