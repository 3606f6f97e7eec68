// abi_core.cu -- error plumbing, asset files, launch accounting and host<->device helpers of the C-ABI.
#include "zr_common.cuh"
#include <dlfcn.h>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <atomic>
#include <vector>
#include <mutex>
#include <map>
#include <string>

namespace zr
{
    static thread_local char g_err[512] = { 0 };
    static std::atomic<uint64_t> g_launches{ 0 };

    void set_error(const char* fmt, ...)
    {
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(g_err, sizeof(g_err), fmt, ap);
        va_end(ap);
    }

    zr_status read_asset(const char* who, const char* name, void* dst, size_t bytes)
    {
        Dl_info info;
        std::string dir = ".";
        if (dladdr((void*)&read_asset, &info) && info.dli_fname)
        {
            const std::string lib = info.dli_fname;
            const size_t s = lib.find_last_of('/');
            if (s != std::string::npos) dir = lib.substr(0, s);
        }
        const std::string path = dir + "/assets/" + name;
        FILE* fp = fopen(path.c_str(), "rb");
        const bool ok = fp && fread(dst, 1, bytes, fp) == bytes;
        if (fp) fclose(fp);
        if (!ok)
        {
            set_error("%s: cannot read %s (tools/extract_reference_tables.py writes it)", who, path.c_str());
            return ZR_ERR_NOT_INITIALIZED;
        }
        return ZR_OK;
    }

    zr_status cuda_fail(cudaError_t e, const char* what)
    {
        set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
        return ZR_ERR_CUDA;
    }

    zr_status check_frame_size(const char* pass, const zr_frame_constants& frame, uint32_t width, uint32_t height)
    {
        if (frame.RenderWidth == width && frame.RenderHeight == height) return ZR_OK;
        set_error("%s_render: frame is %ux%u but the pass was sized %ux%u", pass, frame.RenderWidth, frame.RenderHeight, width, height);
        return ZR_ERR_INVALID_ARG;
    }

    void count_launch(uint64_t n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

    // Optional per-kernel timing (bench.py's roofline leg): an event pair around every launch while enabled.
    struct ProfRec { const char* name; cudaEvent_t a, b; };
    static bool g_profOn = false;
    static std::vector<ProfRec> g_prof;
    static std::mutex g_profMu;
    static thread_local ProfRec g_pending{ nullptr, nullptr, nullptr };
    static thread_local cudaStream_t g_pendingStream = nullptr;

    void prof_before(const char* name, cudaStream_t stream)
    {
        if (!g_profOn) return;
        ProfRec r; r.name = name;
        cudaEventCreate(&r.a); cudaEventCreate(&r.b);
        cudaEventRecord(r.a, stream);
        g_pending = r; g_pendingStream = stream;
    }
    void prof_after()
    {
        if (!g_profOn || !g_pending.name) return;
        cudaEventRecord(g_pending.b, g_pendingStream);
        std::lock_guard<std::mutex> lk(g_profMu);
        g_prof.push_back(g_pending);
        g_pending.name = nullptr;
    }
}

extern "C"
{
    const char* zr_last_error(void) { return zr::g_err; }
    // 1.5: - ZR_INDIRECT_THREADMAP_CTN (never written; ZR_INDIRECT_THREADMAP_NTC keeps its id 6); resize is all-or-nothing and
    //        allocation failures return ZR_ERR_OUT_OF_MEMORY
    // 1.4: - the stage-limited ReSTIR PT render and its stage enum (nothing called them)
    // 1.3: - zr_indirect_pass_set_execution, zr_compositing_pass_render_unfused (measurement and test hooks; nothing else called them)
    uint32_t zr_abi_version(void) { return (1u << 16) | 11u; }    // 1.11: + zr_indirect_pass_set_debug_view; 1.10: + zr_gbuffer_pass_pick / get_pick, zr_display_pass_set_view / set_picked; 1.9: + zr_scene_update_materials, zr_scene_get_tables; 1.8: + zr_svgf_pass_set_rows / set_halo_exchange, sharded SVGF stage; 1.7: + zr_comm_create_transport; 1.6: + AutoExposure and Display passes, zr_renderer_set_display, zr_comm_allreduce_u32; 1.2: + SVGF pass, zr_comm, sharded renderer, zr_gi_pass_set_rows / set_halo_exchange; 1.1: + zr_bvh_build_host, zr_renderer_set_integrator / get_gi_pass / apply_scene_settings, zr_gi_pass_set_method
    uint64_t zr_kernel_launch_count(void) { return zr::g_launches.load(); }

    zr_status zr_profile_enable(int on)
    {
        std::lock_guard<std::mutex> lk(zr::g_profMu);
        zr::g_profOn = on != 0;
        return ZR_OK;
    }
    // Synchronises the device, then writes "name:calls:total_ms;..." for every kernel timed since the last collect.
    zr_status zr_profile_collect(char* buf, size_t bufSize)
    {
        if (!buf || !bufSize) return ZR_ERR_INVALID_ARG;
        ZR_CUDA(cudaDeviceSynchronize());
        std::lock_guard<std::mutex> lk(zr::g_profMu);
        std::map<std::string, std::pair<int, double>> agg;
        for (auto& r : zr::g_prof)
        {
            float ms = 0;
            cudaEventElapsedTime(&ms, r.a, r.b);
            auto& e = agg[r.name];
            e.first++; e.second += ms;
            cudaEventDestroy(r.a); cudaEventDestroy(r.b);
        }
        zr::g_prof.clear();
        std::string out;
        for (auto& kv : agg)
        {
            char line[160];
            snprintf(line, sizeof(line), "%s:%d:%.6f;", kv.first.c_str(), kv.second.first, kv.second.second);
            out += line;
        }
        if (out.size() + 1 > bufSize) { zr::set_error("zr_profile_collect: buffer too small"); return ZR_ERR_INVALID_ARG; }
        memcpy(buf, out.c_str(), out.size() + 1);
        return ZR_OK;
    }

    zr_status zr_device_malloc(void** d_ptr, size_t bytes)
    {
        if (!d_ptr) { zr::set_error("zr_device_malloc: null out pointer"); return ZR_ERR_INVALID_ARG; }
        cudaError_t e = cudaMalloc(d_ptr, bytes ? bytes : 1);
        if (e != cudaSuccess) { zr::cuda_fail(e, "cudaMalloc"); return e == cudaErrorMemoryAllocation ? ZR_ERR_OUT_OF_MEMORY : ZR_ERR_CUDA; }
        return ZR_OK;
    }
    void zr_device_free(void* d_ptr) { if (d_ptr) cudaFree(d_ptr); }
    zr_status zr_memcpy_h2d(void* d_dst, const void* h_src, size_t bytes, void* stream)
    {
        ZR_CUDA(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
        return ZR_OK;
    }
    zr_status zr_memcpy_d2h(void* h_dst, const void* d_src, size_t bytes, void* stream)
    {
        ZR_CUDA(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
        return ZR_OK;
    }
    zr_status zr_memset_d(void* d_dst, int value, size_t bytes, void* stream)
    {
        ZR_CUDA(cudaMemsetAsync(d_dst, value, bytes, (cudaStream_t)stream));
        return ZR_OK;
    }
    zr_status zr_stream_synchronize(void* stream)
    {
        ZR_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
        return ZR_OK;
    }
}
