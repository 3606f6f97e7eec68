// zr_schedule.h -- host side: the rows a strip-sharded pass owns and its halo hook; which thread blocks a lighting kernel
// launches, and in which order.
//
// A lighting kernel's blocks differ in cost by orders of magnitude (sky vs. the inside of the box) and only one or
// two of them fit on an SM, so the hardware's in-order block dispatch leaves a tail in which a few SMs finish the
// last expensive blocks while the rest idle (ncu: 5-8 % of each kernel at 1080p, and a fixed cost that does not shrink
// when a frame is strip-sharded). The schedule lists the blocks that intersect the rows this device owns, most
// expensive 32-row band first (longest-processing-time-first), so the tail is made of cheap blocks; blocks outside
// the strip are not launched at all. Per-pixel results do not depend on the order.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>
#include "zr_common.cuh"

namespace zr
{
struct BlockSchedule
{
    uint32_t* d_order = nullptr;
    uint32_t count = 0;
    // key of the inputs the table was built from
    uint32_t rowBegin = 0xffffffffu, rowEnd = 0, costVersion = 0xffffffffu;

    BlockSchedule() = default;
    BlockSchedule(const BlockSchedule&) = delete;
    BlockSchedule& operator=(const BlockSchedule&) = delete;
    ~BlockSchedule() { Release(); }
    void Release() { if (d_order) cudaFree(d_order); d_order = nullptr; count = 0; rowBegin = 0xffffffffu; }
    bool UpToDate(uint32_t y0, uint32_t y1, uint32_t version) const { return d_order && rowBegin == y0 && rowEnd == y1 && costVersion == version; }
    cudaError_t Upload(const std::vector<uint32_t>& order, uint32_t y0, uint32_t y1, uint32_t version)
    {
        if (d_order) cudaFree(d_order);
        d_order = nullptr;
        count = (uint32_t)order.size();
        rowBegin = y0; rowEnd = y1; costVersion = version;
        if (!count) return cudaSuccess;
        cudaError_t e = cudaMalloc(&d_order, count * sizeof(uint32_t));
        if (e != cudaSuccess) return e;
        return cudaMemcpy(d_order, order.data(), count * sizeof(uint32_t), cudaMemcpyHostToDevice);
    }
};

// cost of the 32x32-pixel tile holding pixel (x, y); tiles are stored row-major, tilesX per row
struct TileCosts
{
    std::vector<double> cost;
    uint32_t tilesX = 0;
    uint32_t version = 0;       // bumped whenever the costs change
    double At(uint32_t x, uint32_t y) const
    {
        if (!tilesX) return 0.0;
        const size_t i = (size_t)(y >> 5) * tilesX + std::min(x >> 5, tilesX - 1);
        return i < cost.size() ? cost[i] : 0.0;
    }
};

inline void SortByCost(std::vector<uint32_t>& blocks, const std::vector<double>& key)
{
    std::vector<uint32_t> idx(blocks.size());
    for (uint32_t i = 0; i < idx.size(); i++) idx[i] = i;
    std::stable_sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return key[a] > key[b]; });
    std::vector<uint32_t> out(blocks.size());
    for (uint32_t i = 0; i < idx.size(); i++) out[i] = blocks[idx[i]];
    blocks.swap(out);
}

// Host copy of the thread-group swizzle (zr_common.cuh SwizzleThreadGroup, tile width 16, tile = all group rows):
// flattened group id -> group column / row after swizzling.
inline void SwizzledGroup(uint32_t flat, uint32_t dispX, uint32_t dispY, uint32_t& outX, uint32_t& outY)
{
    const uint32_t tileWidth = 16, numGroupsInTile = 16 * dispY;
    const uint32_t tileID = flat / numGroupsInTile, inTile = flat % numGroupsInTile;
    const uint32_t numFullTiles = dispX / tileWidth;
    uint32_t gx, gy;
    if (flat >= numFullTiles * numGroupsInTile)
    {
        const uint32_t lastW = dispX - tileWidth * numFullTiles;
        gx = inTile % lastW; gy = inTile / lastW;
    }
    else
    {
        gx = inTile & (tileWidth - 1); gy = inTile >> 4;
    }
    const uint32_t swz = gy * dispX + tileID * tileWidth + gx;
    outX = swz % dispX; outY = swz / dispX;
}

// Kernels whose block is `groupsPerBlock` consecutive flattened groups of groupW x groupH pixels each.
inline std::vector<uint32_t> ScheduleSwizzled(uint32_t dispX, uint32_t dispY, uint32_t groupW, uint32_t groupH, uint32_t groupsPerBlock,
    uint32_t rowBegin, uint32_t rowEnd, const TileCosts& costs)
{
    const uint32_t numGroups = dispX * dispY;
    const uint32_t numBlocks = (numGroups + groupsPerBlock - 1) / groupsPerBlock;
    std::vector<uint32_t> blocks;
    std::vector<double> key;
    for (uint32_t b = 0; b < numBlocks; b++)
    {
        bool inside = false;
        double c = 0;
        for (uint32_t g = b * groupsPerBlock; g < (b + 1) * groupsPerBlock && g < numGroups; g++)
        {
            uint32_t gx, gy;
            SwizzledGroup(g, dispX, dispY, gx, gy);
            const uint32_t r0 = gy * groupH;
            if (r0 + groupH > rowBegin && r0 < rowEnd) { inside = true; c = std::max(c, costs.At(gx * groupW, r0)); }
        }
        if (inside) { blocks.push_back(b); key.push_back(c); }
    }
    SortByCost(blocks, key);
    return blocks;
}

// What a pass that runs strip-sharded keeps (SURVEY 8e): the rows it owns and the hook that makes rows it just wrote coherent
// across strips. `pass` ("zr_direct_pass", ...) prefixes the error messages of the pass's set_* entry points.
struct StripRows
{
    const char* pass;
    uint32_t rowBegin = 0, rowEnd = 0xffffffffu;
    zr_halo_exchange_fn exchange = nullptr;
    void* exchangeUser = nullptr;

    explicit StripRows(const char* passName) : pass(passName) {}
    // after a resize: the rows described the old frame; the halo hook stays
    void ForgetRows() { rowBegin = 0; rowEnd = 0xffffffffu; }
    uint32_t ClampedRowEnd(uint32_t height) const { return rowEnd < height ? rowEnd : height; }

    zr_status SetRows(uint32_t y0, uint32_t y1, uint32_t height)
    {
        if (y0 >= y1 || y0 >= height) { set_error("%s_set_rows: empty row range", pass); return ZR_ERR_INVALID_ARG; }
        rowBegin = y0; rowEnd = y1;
        return ZR_OK;
    }
    zr_status SetHaloExchange(zr_halo_exchange_fn fn, void* user)
    {
        exchange = fn; exchangeUser = user;
        return ZR_OK;
    }
    // hands the hook n planes (their own pitches); nothing happens without a hook
    void Exchange(const zr_image2d* planes, int n, cudaStream_t stream) const
    {
        if (exchange) exchange(exchangeUser, planes, n, stream);
    }
    // one unpadded width x height plane of texelBytes-sized texels
    void Exchange(void* d_plane, uint32_t width, uint32_t height, uint32_t texelBytes, cudaStream_t stream) const
    {
        const zr_image2d plane{ d_plane, width, height, width * texelBytes, texelBytes };
        Exchange(&plane, 1, stream);
    }
};

// What a lighting pass keeps on top of its rows and hook: the optional cost map and tile costs, and its kernels' block table.
struct LightingStrip : StripRows
{
    unsigned long long* d_costMap = nullptr;
    TileCosts tileCosts;
    BlockSchedule sched[2];     // one block table per block shape; a pass whose kernels have two shapes uses both

    explicit LightingStrip(const char* passName) : StripRows(passName) {}
    // after a resize: the rows, cost map, tile costs and block table described the old frame; the halo hook stays
    void ForgetSize()
    {
        ForgetRows();
        d_costMap = nullptr;
        tileCosts = TileCosts{};
        sched[0].Release();
        sched[1].Release();
    }
    zr_status SetCostMap(void* d_cycles)
    {
        d_costMap = (unsigned long long*)d_cycles;
        return ZR_OK;
    }
    // h_tile_cost: ceil(width/32) x ceil(height/32) tiles, row-major, or nullptr for plain order
    zr_status SetScheduleCosts(const double* h_tile_cost, uint32_t tiles_x, uint32_t tiles_y, uint32_t width, uint32_t height)
    {
        if (h_tile_cost && (tiles_x != (width + 31) / 32 || tiles_y != (height + 31) / 32))
        {
            set_error("%s_set_schedule_costs: expected %u x %u tiles", pass, (width + 31) / 32, (height + 31) / 32);
            return ZR_ERR_INVALID_ARG;
        }
        tileCosts.cost.assign(h_tile_cost ? h_tile_cost : nullptr, h_tile_cost ? h_tile_cost + (size_t)tiles_x * tiles_y : nullptr);
        tileCosts.tilesX = h_tile_cost ? tiles_x : 0;
        tileCosts.version++;
        return ZR_OK;
    }
    // sched[shape] for a kernel whose blocks are groupsPerBlock swizzled groups of groupW x groupH pixels; the table is rebuilt and
    // uploaded only when the rows or the tile costs changed
    zr_status Schedule(uint32_t width, uint32_t height, uint32_t groupW, uint32_t groupH, uint32_t groupsPerBlock, int shape = 0)
    {
        const uint32_t y0 = rowBegin, y1 = ClampedRowEnd(height), v = tileCosts.version;
        BlockSchedule& s = sched[shape];
        if (!s.UpToDate(y0, y1, v))
            ZR_CUDA(s.Upload(ScheduleSwizzled((width + groupW - 1) / groupW, (height + groupH - 1) / groupH, groupW, groupH, groupsPerBlock,
                y0, y1, tileCosts), y0, y1, v));
        return ZR_OK;
    }
};
} // namespace zr
