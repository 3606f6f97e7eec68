// zr_bvh.h -- the acceleration structure's storage format and its host builder (plain C++, no CUDA).
//
// Stands in for what ZetaCore/RayTracing/RtAccelerationStructure.cpp gets from the DXR driver
// (BuildRaytracingAccelerationStructure for the static BLAS + TLAS): binned-SAH binary BVH over
// world-space triangles -> collapsed to 8-wide nodes -> child boxes quantised to 8 bits per plane,
// rounded outwards. Lives in its own translation unit so the builder can be exercised without a GPU
// (zr_bvh_build_host, tests/test_bvh_host.py).
#pragma once
#include <stdint.h>
#include <vector>

namespace zr
{
struct BVH8Node
{
    float px, py, pz;
    uint8_t ex, ey, ez, pad;
    uint32_t childBase;
    uint32_t triBase;
    uint8_t meta[8];        // bits 7..6: #tris of a leaf child (0 = not a leaf), bit 5: internal child, bits 4..0: offset
    uint8_t qlo[3][8];
    uint8_t qhi[3][8];
};
static_assert(sizeof(BVH8Node) == 80, "BVH8Node must be 80 bytes");

// Entries the node-group stack of zr_scene.cuh::Traverse holds. One entry stands for the unvisited hit inner children of one
// node and each tree level keeps at most one, so a tree of depth BvhBuild::maxDepth needs maxDepth - 1 entries (the 302 k-triangle
// atrium 8, the 1.03 M-triangle tunnel 7). Scene creation refuses a deeper tree, so the device never drops a node.
constexpr int BVH_STACK_ENTRIES = 32;
// How many of those entries (the top ones) Traverse keeps in registers; the rest live in a local array.
#ifndef ZR_BVH_STACK_REGS
#define ZR_BVH_STACK_REGS 1
#endif
constexpr int BVH_STACK_REGS = ZR_BVH_STACK_REGS;
static_assert(BVH_STACK_REGS >= 1 && BVH_STACK_REGS < BVH_STACK_ENTRIES, "BVH_STACK_REGS out of range");

struct BvhBuild
{
    std::vector<BVH8Node> nodes;
    std::vector<uint32_t> leafOrder;    // global triangle index per slot of the leaf-ordered triangle array
    uint32_t maxDepth = 0;              // of the 8-wide tree, the root at depth 1
    uint32_t maxStack = 0;              // worst-case occupancy of a stack of single nodes (reported only; Traverse stacks node groups)
};

// worldTris: 9 floats per triangle {v0, e1 = v1 - v0, e2 = v2 - v0}, the arithmetic k_world_tris produced.
void build_bvh8(const float* worldTris, uint32_t numTris, BvhBuild& out);
} // namespace zr
