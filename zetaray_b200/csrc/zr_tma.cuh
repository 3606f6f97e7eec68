// zr_tma.cuh -- Tensor Memory Accelerator plumbing for the streaming kernels (sm_90a).
//
// Host: tensor maps over pitched 2D planes ([H][W] records of 8..64 bytes), encoded through the driver entry point
// cuTensorMapEncodeTiled, which is fetched at run time with cudaGetDriverEntryPoint (the library links cudart only).
// Device: mbarrier + cp.async.bulk.tensor.2d wrappers (SASS: UTMALDG / UTMASTG, SYNCS). Tiles that stick out of the
// image are zero-filled on load and clipped on store by the hardware, so edge tiles need no special casing.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace zr
{
namespace tma
{
    // A plane of `width` x `height` records of `recordBytes` (multiple of 8) with a row pitch of `pitchBytes` (multiple of 16),
    // fetched in boxes of boxW x boxH records. The map describes the plane as rows of 64-bit words: boxW * recordBytes / 8 <= 256.
    inline bool EncodePlane2D(CUtensorMap* map, const void* base, uint32_t width, uint32_t height, uint32_t recordBytes,
        uint64_t pitchBytes, uint32_t boxW, uint32_t boxH)
    {
        typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
            const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
        static EncodeFn encode = nullptr;
        if (!encode)
        {
            void* fn = nullptr;
            cudaDriverEntryPointQueryResult qres;
            if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn ||
                qres != cudaDriverEntryPointSuccess)
                return false;
            encode = (EncodeFn)fn;
        }
        const uint32_t wordsPerRecord = recordBytes / 8;
        if (recordBytes % 8 || pitchBytes % 16 || boxW * wordsPerRecord > 256 || boxH > 256 || ((uintptr_t)base & 15))
            return false;
        const cuuint64_t dims[2] = { (cuuint64_t)width * wordsPerRecord, height };
        const cuuint64_t strides[1] = { pitchBytes };
        const cuuint32_t box[2] = { boxW * wordsPerRecord, boxH };
        const cuuint32_t elemStrides[2] = { 1, 1 };
        return encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<void*>(base), dims, strides, box, elemStrides,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    }

    // General form: `rank` dimensions of 64-bit words, dims[0] innermost (contiguous); stridesBytes[i] is the byte stride of
    // dimension i + 1 (multiples of 16). Used for strided-lattice views of an image: {phase_x, u, phase_y, v} with pixel
    // x = u * step + phase_x, y = v * step + phase_y turns every sub-lattice of an a-trous pass into a dense box.
    // swizzle128: CU_TENSOR_MAP_SWIZZLE_128B -- the innermost box extent must be 16 words (128 bytes) and the shared-memory tile 1024-byte
    // aligned; the 16-byte chunk c of the 128-byte line L of the tile then lives at chunk c ^ (L & 7) of that line, which makes a warp's
    // 128-bit reads of consecutive 64-byte records conflict-free.
    inline bool EncodeWords(CUtensorMap* map, const void* base, uint32_t rank, const uint64_t* dims, const uint64_t* stridesBytes, const uint32_t* box,
        bool swizzle128 = false)
    {
        typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
            const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
        static EncodeFn encode = nullptr;
        if (!encode)
        {
            void* fn = nullptr;
            cudaDriverEntryPointQueryResult qres;
            if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn ||
                qres != cudaDriverEntryPointSuccess)
                return false;
            encode = (EncodeFn)fn;
        }
        if (rank < 1 || rank > 5 || ((uintptr_t)base & 15) || (box[0] * 8) % 16) return false;
        cuuint64_t d[5]; cuuint64_t st[4]; cuuint32_t b[5]; cuuint32_t es[5];
        for (uint32_t i = 0; i < rank; i++) { d[i] = dims[i]; b[i] = box[i]; es[i] = 1; if (box[i] == 0 || box[i] > 256) return false; }
        for (uint32_t i = 0; i + 1 < rank; i++) { st[i] = stridesBytes[i]; if (st[i] % 16) return false; }
        if (swizzle128 && box[0] != 16) return false;
        return encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT64, rank, const_cast<void*>(base), d, st, b, es,
            CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    }

#ifdef __CUDACC__
    __device__ __forceinline__ uint32_t SmemAddr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

    __device__ __forceinline__ void MbarInit(uint64_t* bar, uint32_t arrivals)
    {
        asm volatile("mbarrier.init.shared::cta.b64 [%1], %0;" :: "r"(arrivals), "r"(SmemAddr(bar)) : "memory");
    }
    // makes the initialised barriers visible to the async (TMA) proxy; follow with __syncthreads()
    __device__ __forceinline__ void FenceBarrierInit() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    // orders generic-proxy shared-memory accesses (reads of a tile about to be overwritten, writes of a tile about to be
    // stored) against the async proxy
    __device__ __forceinline__ void FenceProxyAsync() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

    __device__ __forceinline__ void MbarArriveExpectTx(uint64_t* bar, uint32_t bytes)
    {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%1], %0;" :: "r"(bytes), "r"(SmemAddr(bar)) : "memory");
    }
    __device__ __forceinline__ void MbarWait(uint64_t* bar, uint32_t parity)
    {
        asm volatile(
            "{\n\t"
            ".reg .pred P1;\n\t"
            "LAB_WAIT:\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n\t"
            "@P1 bra DONE;\n\t"
            "bra LAB_WAIT;\n\t"
            "DONE:\n\t"
            "}" :: "r"(SmemAddr(bar)), "r"(parity), "r"(0x989680u) : "memory");
    }
    // box at (x0 in 64-bit words, y0 in rows) -> dense [boxH][boxW words] at `smem` (128-byte aligned); completes on `bar`
    __device__ __forceinline__ void Load2D(void* smem, const CUtensorMap* map, uint64_t* bar, int32_t x0, int32_t y0)
    {
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
            :: "r"(SmemAddr(smem)), "l"((uint64_t)map), "r"(SmemAddr(bar)), "r"(x0), "r"(y0) : "memory");
    }
    __device__ __forceinline__ void Store2D(const CUtensorMap* map, const void* smem, int32_t x0, int32_t y0)
    {
        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
            :: "l"((uint64_t)map), "r"(SmemAddr(smem)), "r"(x0), "r"(y0) : "memory");
    }
    __device__ __forceinline__ void Load3D(void* smem, const CUtensorMap* map, uint64_t* bar, int32_t c0, int32_t c1, int32_t c2)
    {
        asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
            :: "r"(SmemAddr(smem)), "l"((uint64_t)map), "r"(SmemAddr(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
    }
    __device__ __forceinline__ void Load4D(void* smem, const CUtensorMap* map, uint64_t* bar, int32_t c0, int32_t c1, int32_t c2, int32_t c3)
    {
        asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
            :: "r"(SmemAddr(smem)), "l"((uint64_t)map), "r"(SmemAddr(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
    }
    __device__ __forceinline__ void Store4D(const CUtensorMap* map, const void* smem, int32_t c0, int32_t c1, int32_t c2, int32_t c3)
    {
        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
            :: "l"((uint64_t)map), "r"(SmemAddr(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
    }
    __device__ __forceinline__ void StoreCommit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
    // all committed stores have finished READING shared memory (the tile may be reused)
    __device__ __forceinline__ void StoreWaitRead() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
    // all committed stores are complete
    __device__ __forceinline__ void StoreWaitAll() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
#endif
}
} // namespace zr
