// zr_planes.h -- host side: the device allocations a pass holds for one frame size, and the create / resize / reset / destroy
// bodies every pass's C entry points share.
//
// A pass keeps everything that depends on the frame size in one member that owns a Planes. OnWindowResized builds a complete new
// member (allocations, tensor maps, clears) and swaps it in only when all of it succeeded, so a failed resize leaves the pass exactly
// as it was; while a resize runs, the old and the new planes are both allocated.
#pragma once
#include <memory>
#include <utility>
#include <vector>
#include <cuda_runtime.h>
#include "zr_common.cuh"

#define ZR_TRY(expr) do { const zr_status s__ = (expr); if (s__ != ZR_OK) return s__; } while (0)

namespace zr
{
class Planes
{
public:
    explicit Planes(const char* passName) : pass(passName) {}
    Planes(Planes&& o) noexcept : pass(o.pass), blocks(std::move(o.blocks)) { o.blocks.clear(); }
    Planes& operator=(Planes&& o) noexcept { std::swap(pass, o.pass); std::swap(blocks, o.blocks); return *this; }
    Planes(const Planes&) = delete;
    Planes& operator=(const Planes&) = delete;
    ~Planes() { for (const Block& b : blocks) cudaFree(b.ptr); }

    // count elements of T; Clear() zeroes the plane only when `clear` is set
    template<typename T>
    zr_status Alloc(T*& p, size_t count, bool clear = true)
    {
        void* d = nullptr;
        const size_t bytes = count * sizeof(T);
        const cudaError_t e = cudaMalloc(&d, bytes);
        if (e != cudaSuccess)
        {
            cudaGetLastError();     // the failure is reported here, not by the next launch check
            set_error("%s: cannot allocate %zu bytes of device memory (%s)", pass, bytes, cudaGetErrorString(e));
            return e == cudaErrorMemoryAllocation ? ZR_ERR_OUT_OF_MEMORY : ZR_ERR_CUDA;
        }
        blocks.push_back(Block{ d, bytes, clear });
        p = (T*)d;
        return ZR_OK;
    }
    zr_status Clear() const
    {
        ZR_CLEAR_BEGIN();
        for (const Block& b : blocks)
            if (b.clear) ZR_CUDA(cudaMemset(b.ptr, 0, b.bytes));
        ZR_CLEAR_END();
        return ZR_OK;
    }

private:
    struct Block { void* ptr; size_t bytes; bool clear; };
    const char* pass;
    std::vector<Block> blocks;
};

// The lifecycle entry points. P has Setup() (size-independent, once), OnWindowResized(w, h) and ResetTemporal(); `name` is the
// entry points' prefix ("zr_direct_pass", ...).
template<typename P>
zr_status CreatePass(const char* name, uint32_t w, uint32_t h, P** out)
{
    if (!out || !w || !h) { set_error("%s_create: bad args", name); return ZR_ERR_INVALID_ARG; }
    *out = nullptr;
    std::unique_ptr<P> p(new P());
    ZR_TRY(p->Setup());
    ZR_TRY(p->OnWindowResized(w, h));
    *out = p.release();
    return ZR_OK;
}
template<typename P>
zr_status ResizePass(const char* name, P* p, uint32_t w, uint32_t h)
{
    if (!p || !w || !h) { set_error("%s_resize: null pass or zero size", name); return ZR_ERR_INVALID_ARG; }
    return p->OnWindowResized(w, h);
}
template<typename P>
zr_status ResetPass(P* p) { return p ? p->ResetTemporal() : ZR_ERR_INVALID_ARG; }
template<typename P, typename Params>
zr_status DefaultParams(Params* out)
{
    if (!out) return ZR_ERR_INVALID_ARG;
    *out = P::Defaults();
    return ZR_OK;
}
} // namespace zr
