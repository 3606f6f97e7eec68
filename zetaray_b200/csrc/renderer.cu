// renderer.cu -- the frame: which passes run, in which order, on which stream (host code only, no kernels).
//
// Headless counterpart of ZetaRenderer/Default: DefaultRenderer::Update/Render (DefaultRenderer.cpp:304-520) decide what
// a frame contains, PathTracer::Register/AddAdjacencies (PathTracer.cpp:149-563) and the GBuffer / PostProcessor
// equivalents put the passes into the render graph, and the graph runs them in dependency order with DirectLighting and
// IndirectLighting as independent compute nodes (both read only the G-buffer). Here that schedule is fixed:
//
//   frame 1 only      zr_prelighting_render        power estimate + alias table (on device, so no one-frame read-back delay)
//   every frame       zr_presample_emissives       when presampling is on (the reference: >= 13107 emissive triangles)
//                     GBufferRT -> IndirectLighting               `chain` stream, the greatest priority
//                     DirectLighting                              `side` stream, the least priority, after GBufferRT
//                     Compositing (+ firefly filter) -> [SVGF denoise, zr_renderer_set_denoiser] -> TAA
//                     with zr_renderer_set_display: AutoExposure on the TAA input before TAA, Display on its output after it
//                     with zr_renderer_set_sky: the sky-view LUT on `side`, before DirectLighting
//
// Streams (two_streams != 0; otherwise every pass runs on the caller's stream in the order above). `chain` is forked from the caller's
// stream by an event and holds the frame's critical path: GBufferRT and IndirectLighting, whose shift stages fork two more streams of
// the same priority (ShiftStreams, rpt_spatial.cu). DirectLighting is the shorter of the two lighting passes and needs only the
// G-buffer, so it runs at the least priority: the block scheduler hands an SM to a pending DirectLighting block only when no chain
// kernel has a block waiting, and DirectLighting fills the SM time the chain leaves idle (the last wave of k_pathtrace, the drain of the
// persistent shift launches, the ramps and gaps of the short kernels) instead of delaying the chain. Both streams join the caller's
// stream before Compositing, and everything from Compositing on -- SVGF, AutoExposure, TAA, Display, the post-lighting halo exchange and
// the gathers -- runs on the caller's stream, so the caller's stream is ordered after the whole frame. Strip-sharded, DirectLighting's
// halo exchange uses communicator 1 on `side`; IndirectLighting's use communicator 0 on `chain`, and the caller's stream uses
// communicator 0 after the join, which orders the two.
//
// The renderer owns the double-buffered G-buffers (DefaultRendererImpl.h:111-121) and the pass objects; callers reach
// the passes through zr_renderer_get_*_pass to set parameters, exactly like the reference's UI callbacks do.
#include <cuda_runtime.h>
#include <vector>
#include "../../include/zr_abi.h"
#include "zr_common.cuh"

struct zr_renderer
{
    uint32_t width = 0, height = 0;
    zr_scene* scene = nullptr;              // not owned
    zr_gbuffer gbuffer[2]{};
    int curr = 0;
    uint64_t framesRendered = 0;
    zr_gbuffer_pass* gbufferPass = nullptr;
    zr_direct_pass* direct = nullptr;
    zr_indirect_pass* indirect = nullptr;
    zr_gi_pass* gi = nullptr;                       // created on the first SetMethod(ReSTIR_GI / PATH_TRACING)
    zr_integrator integrator = ZR_INTEGRATOR_RESTIR_PT;     // RenderSettings::Indirect default, DefaultRendererImpl.h:64
    zr_compositing_pass* compositing = nullptr;
    zr_taa_pass* taa = nullptr;
    zr_svgf_pass* svgf = nullptr;                   // optional denoise stage between Compositing and TAA (BASELINE config 3)
    zr_auto_exposure_pass* ae = nullptr;            // optional post-processing (PostProcessor.cpp): both or neither
    zr_display_pass* display = nullptr;
    zr_sky_pass* sky = nullptr;                     // optional sky-view LUT, read by DirectLighting and Compositing (zr_renderer_set_sky)
    cudaStream_t chain = nullptr;           // GBufferRT + IndirectLighting when twoStreams, the greatest priority
    cudaStream_t side = nullptr;            // DirectLighting when twoStreams, the least priority
    cudaEvent_t evFork = nullptr, evGBuffer = nullptr, evChain = nullptr, evDirect = nullptr;
    bool twoStreams = true;
    // strip-sharded frames
    zr_comm* comm = nullptr;                // not owned
    int rank = 0, world = 1;
    std::vector<uint32_t> bounds;
    bool gatherOutput = true;
    static constexpr uint32_t HALO = 32;
    struct HookCtx { zr_renderer* r; int whichComm; } hookMain{ this, 0 }, hookSide{ this, 1 };
    zr_status hookStatus = ZR_OK;
    static void HaloHook(void* user, const zr_image2d* planes, int n, void* stream)
    {
        HookCtx* h = (HookCtx*)user;
        zr_renderer* r = h->r;
        // DirectLighting runs on `side` when twoStreams, concurrently with the chain's exchanges: it gets its own communicator
        const int which = (r->twoStreams && stream == (void*)r->side) ? 1 : 0;
        const zr_status s = zr_comm_exchange_halos(r->comm, which, r->bounds.data(), HALO, planes, n, stream);
        if (s != ZR_OK) r->hookStatus = s;
    }
    // AutoExposure's bins: every rank's strip histogram summed in place, so every rank derives the same exposure
    static void ReduceHook(void* user, uint32_t* d_values, uint32_t n, void* stream)
    {
        zr_renderer* r = (zr_renderer*)user;
        const zr_status s = zr_comm_allreduce_u32(r->comm, 0, d_values, n, stream);
        if (s != ZR_OK) r->hookStatus = s;
    }

    // Applies the current strip to every pass that exists: zr_renderer_set_shard, and the entry points that create the GI, SVGF and
    // display passes (possibly after the cut). Sharded, each pass gets the rows it computes and its hook; otherwise the whole frame
    // and no hook. Re-applying unchanged rows and hooks rebuilds nothing.
    zr_status ApplyShard()
    {
        const bool sharded = comm && world > 1;
        const uint32_t y0 = sharded ? bounds[rank] : 0, y1 = sharded ? bounds[rank + 1] : height;
        zr_halo_exchange_fn hook = sharded ? HaloHook : nullptr;
        // the G-buffer halo is re-rendered locally; the TAA neighbourhood reads the composited signal one row beyond the strip
        zr_status s = zr_gbuffer_pass_set_rows(gbufferPass, y0 > HALO ? y0 - HALO : 0, y1 + HALO < height ? y1 + HALO : height);
        if (s == ZR_OK) s = zr_direct_pass_set_rows(direct, y0, y1);
        if (s == ZR_OK) s = zr_indirect_pass_set_rows(indirect, y0, y1);
        if (s == ZR_OK) s = zr_compositing_pass_set_rows(compositing, y0 > 0 ? y0 - 1 : 0, y1 + 1 < height ? y1 + 1 : height);
        if (s == ZR_OK) s = zr_taa_pass_set_rows(taa, y0, y1);
        if (s == ZR_OK) s = zr_direct_pass_set_halo_exchange(direct, hook, &hookSide);
        if (s == ZR_OK) s = zr_indirect_pass_set_halo_exchange(indirect, hook, &hookMain);
        if (s == ZR_OK && gi) s = zr_gi_pass_set_rows(gi, y0, y1);
        if (s == ZR_OK && gi) s = zr_gi_pass_set_halo_exchange(gi, hook, &hookMain);
        if (s == ZR_OK && svgf) s = zr_svgf_pass_set_rows(svgf, y0, y1);
        if (s == ZR_OK && svgf) s = zr_svgf_pass_set_halo_exchange(svgf, hook, &hookMain);
        if (s == ZR_OK && ae) s = zr_auto_exposure_pass_set_rows(ae, y0, y1);
        if (s == ZR_OK && ae) s = zr_auto_exposure_pass_set_reduce(ae, sharded ? ReduceHook : nullptr, this);
        if (s == ZR_OK && display) s = zr_display_pass_set_rows(display, y0, y1);
        return s;
    }
    // an error a hook met during the stage that just ran; reported once
    zr_status TakeHookStatus()
    {
        const zr_status s = hookStatus;
        hookStatus = ZR_OK;
        return s;
    }
    void ReleaseDisplay()
    {
        if (ae) zr_auto_exposure_pass_destroy(ae);
        if (display) zr_display_pass_destroy(display);
        ae = nullptr; display = nullptr;
    }

    // detaches the LUT from the passes that read it, then frees it
    void ReleaseSky()
    {
        if (direct) zr_direct_pass_set_sky(direct, nullptr);
        if (compositing) zr_compositing_pass_set_sky(compositing, nullptr);
        if (sky) zr_sky_pass_destroy(sky);
        sky = nullptr;
    }

    void Release()
    {
        ReleaseSky();
        if (gbufferPass) zr_gbuffer_pass_destroy(gbufferPass);
        if (direct) zr_direct_pass_destroy(direct);
        if (indirect) zr_indirect_pass_destroy(indirect);
        if (gi) zr_gi_pass_destroy(gi);
        gi = nullptr;
        if (compositing) zr_compositing_pass_destroy(compositing);
        if (taa) zr_taa_pass_destroy(taa);
        if (svgf) zr_svgf_pass_destroy(svgf);
        svgf = nullptr;
        ReleaseDisplay();
        gbufferPass = nullptr; direct = nullptr; indirect = nullptr; compositing = nullptr; taa = nullptr;
        for (int i = 0; i < 2; i++) zr_gbuffer_free(&gbuffer[i]);
        if (chain) cudaStreamDestroy(chain);
        if (side) cudaStreamDestroy(side);
        for (cudaEvent_t e : { evFork, evGBuffer, evChain, evDirect })
            if (e) cudaEventDestroy(e);
        chain = side = nullptr; evFork = evGBuffer = evChain = evDirect = nullptr;
    }
};

extern "C"
{
    zr_status zr_renderer_create(const zr_renderer_desc* desc, zr_scene* scene, zr_renderer** out)
    {
        if (!desc || !scene || !out || !desc->width || !desc->height)
        {
            zr::set_error("zr_renderer_create: bad args");
            return ZR_ERR_INVALID_ARG;
        }
        zr_renderer* r = new zr_renderer();
        r->width = desc->width; r->height = desc->height; r->scene = scene; r->twoStreams = desc->two_streams != 0;
        zr_status s = ZR_OK;
        for (int i = 0; i < 2 && s == ZR_OK; i++) s = zr_gbuffer_alloc(desc->width, desc->height, desc->with_tridiff, &r->gbuffer[i]);
        if (s == ZR_OK) s = zr_gbuffer_pass_create(&r->gbufferPass);
        if (s == ZR_OK) s = zr_direct_pass_create(desc->width, desc->height, &r->direct);
        if (s == ZR_OK) s = zr_indirect_pass_create(desc->width, desc->height, &r->indirect);
        if (s == ZR_OK) s = zr_compositing_pass_create(desc->width, desc->height, &r->compositing);
        if (s == ZR_OK) s = zr_taa_pass_create(desc->width, desc->height, &r->taa);
        int leastPriority = 0, greatestPriority = 0;
        if (s == ZR_OK && cudaDeviceGetStreamPriorityRange(&leastPriority, &greatestPriority) != cudaSuccess) s = ZR_ERR_CUDA;
        if (s == ZR_OK && cudaStreamCreateWithPriority(&r->chain, cudaStreamNonBlocking, greatestPriority) != cudaSuccess) s = ZR_ERR_CUDA;
        if (s == ZR_OK && cudaStreamCreateWithPriority(&r->side, cudaStreamNonBlocking, leastPriority) != cudaSuccess) s = ZR_ERR_CUDA;
        for (cudaEvent_t* e : { &r->evFork, &r->evGBuffer, &r->evChain, &r->evDirect })
            if (s == ZR_OK && cudaEventCreateWithFlags(e, cudaEventDisableTiming) != cudaSuccess) s = ZR_ERR_CUDA;
        if (s != ZR_OK) { r->Release(); delete r; return s; }
        *out = r;
        return ZR_OK;
    }

    void zr_renderer_destroy(zr_renderer* r)
    {
        if (!r) return;
        r->Release();
        delete r;
    }

    // One frame == DefaultRenderer::Update + Render for the emissive-lit path-tracing configuration.
    zr_status zr_renderer_render(zr_renderer* r, const zr_frame_constants* fc, void* stream_)
    {
        if (!r || !fc) return ZR_ERR_INVALID_ARG;
        if (fc->RenderWidth != r->width || fc->RenderHeight != r->height)
        {
            zr::set_error("zr_renderer_render: frame is %ux%u but the renderer was sized %ux%u", fc->RenderWidth, fc->RenderHeight,
                r->width, r->height);
            return ZR_ERR_INVALID_ARG;
        }
        cudaStream_t stream = (cudaStream_t)stream_;
        zr_status s;
        if (r->framesRendered == 0)
        {
            s = zr_prelighting_render(r->scene, stream);
            if (s != ZR_OK) return s;
        }
        s = zr_presample_emissives(r->scene, fc->FrameNum, stream);
        if (s != ZR_OK) return s;
        s = zr_build_light_voxel_grid(r->scene, fc, stream);        // no-op unless the grid is enabled (ReSTIR GI's LVG variant)
        if (s != ZR_OK) return s;

        r->curr ^= 1;       // GlobalIdxForDoubleBufferedResources
        zr_frame_inputs in;
        in.frame = *fc;
        in.curr = r->gbuffer[r->curr];
        in.prev = r->gbuffer[r->curr ^ 1];
        in.scene = r->scene;

        cudaStream_t chainStream = stream, directStream = stream;
        if (r->twoStreams)
        {
            ZR_CUDA(cudaEventRecord(r->evFork, stream));
            ZR_CUDA(cudaStreamWaitEvent(r->chain, r->evFork, 0));
            chainStream = r->chain;
            directStream = r->side;
        }
        s = zr_gbuffer_pass_render(r->gbufferPass, &in, chainStream);
        if (s != ZR_OK) return s;
        if (r->twoStreams)
        {
            ZR_CUDA(cudaEventRecord(r->evGBuffer, chainStream));
            ZR_CUDA(cudaStreamWaitEvent(r->side, r->evGBuffer, 0));
        }
        // the chain is enqueued first: were DirectLighting first, a device that has caught up with the host would start its blocks
        // before the chain's kernels exist, and no priority could give those SMs back
        s = r->integrator != ZR_INTEGRATOR_RESTIR_PT ? zr_gi_pass_render(r->gi, &in, chainStream)
                                                     : zr_indirect_pass_render(r->indirect, &in, chainStream);
        if (s != ZR_OK) return s;
        if (r->sky)
        {
            // the LUT follows the frame's sun and atmosphere, so it is recomputed every frame (PathTracer.cpp:343-362)
            s = zr_sky_pass_render(r->sky, &in, directStream);
            if (s != ZR_OK) return s;
        }
        s = zr_direct_pass_render(r->direct, &in, directStream);
        if (s != ZR_OK) return s;
        if (r->twoStreams)
        {
            ZR_CUDA(cudaEventRecord(r->evChain, chainStream));
            ZR_CUDA(cudaEventRecord(r->evDirect, directStream));
            ZR_CUDA(cudaStreamWaitEvent(stream, r->evChain, 0));
            ZR_CUDA(cudaStreamWaitEvent(stream, r->evDirect, 0));
        }
        s = r->TakeHookStatus();
        if (s != ZR_OK) return s;
        zr_image2d di, ind, comp;
        s = zr_direct_pass_get_output(r->direct, ZR_DIRECT_FINAL, &di);
        if (s != ZR_OK) return s;
        s = r->integrator != ZR_INTEGRATOR_RESTIR_PT ? zr_gi_pass_get_output(r->gi, ZR_GI_FINAL, &ind)
                                                     : zr_indirect_pass_get_output(r->indirect, ZR_INDIRECT_FINAL, &ind);
        if (s != ZR_OK) return s;
        if (r->comm && r->world > 1)
        {
            // the firefly stencil and TAA read the finals / the history one to two rows beyond the strip
            zr_image2d planes[3] = { di, ind, zr_image2d{} };
            s = zr_taa_pass_get_output(r->taa, &planes[2]);
            if (s != ZR_OK) return s;
            s = zr_comm_exchange_halos(r->comm, 0, r->bounds.data(), zr_renderer::HALO, planes, 3, stream);
            if (s != ZR_OK) return s;
        }
        s = zr_compositing_pass_render(r->compositing, &in, di.d_ptr, ind.d_ptr, stream);
        if (s != ZR_OK) return s;
        s = zr_compositing_pass_get_output(r->compositing, &comp);
        if (s != ZR_OK) return s;
        if (r->svgf)
        {
            s = zr_svgf_pass_render(r->svgf, &in, comp.d_ptr, stream);
            if (s != ZR_OK) return s;
            s = r->TakeHookStatus();
            if (s != ZR_OK) return s;
            s = zr_svgf_pass_get_output(r->svgf, ZR_SVGF_DENOISED, &comp);
            if (s != ZR_OK) return s;
        }
        zr_image2d exposure{};
        if (r->ae)
        {
            s = zr_auto_exposure_pass_render(r->ae, &in, comp.d_ptr, stream);
            if (s != ZR_OK) return s;
            s = r->TakeHookStatus();
            if (s != ZR_OK) return s;
            s = zr_auto_exposure_pass_get_output(r->ae, &exposure);
            if (s != ZR_OK) return s;
        }
        s = zr_taa_pass_render(r->taa, &in, comp.d_ptr, stream);
        if (s != ZR_OK) return s;
        zr_image2d img;
        s = zr_taa_pass_get_output(r->taa, &img);
        if (s != ZR_OK) return s;
        zr_image2d shown{};
        if (r->display)
        {
            s = zr_display_pass_render(r->display, &in, img.d_ptr, exposure.d_ptr, stream);
            if (s != ZR_OK) return s;
            s = zr_display_pass_get_output(r->display, &shown);
            if (s != ZR_OK) return s;
        }
        if (r->comm && r->world > 1 && r->gatherOutput)
        {
            s = zr_comm_gather_rows(r->comm, r->bounds.data(), &img, 0, stream);
            if (s != ZR_OK) return s;
            if (r->display) s = zr_comm_gather_rows(r->comm, r->bounds.data(), &shown, 0, stream);
            if (s != ZR_OK) return s;
        }
        r->framesRendered++;
        return ZR_OK;
    }

    // IndirectLighting::SetMethod (IndirectLighting.cpp:203-235, called from DefaultRenderer.cpp:243): switching the
    // integrator drops the temporal history of the one switched to.
    zr_status zr_renderer_set_integrator(zr_renderer* r, zr_integrator method)
    {
        if (!r) return ZR_ERR_INVALID_ARG;
        if (method != ZR_INTEGRATOR_PATH_TRACING && method != ZR_INTEGRATOR_RESTIR_GI && method != ZR_INTEGRATOR_RESTIR_PT)
        {
            zr::set_error("zr_renderer_set_integrator: unknown integrator %d (path tracing = 0, ReSTIR GI = 1, ReSTIR PT = 2)", (int)method);
            return ZR_ERR_INVALID_ARG;
        }
        if (method == r->integrator) return ZR_OK;
        zr_status s = ZR_OK;
        if (method != ZR_INTEGRATOR_RESTIR_PT)
        {
            // the plain path tracer and ReSTIR GI share one pass object (both read cb_ReSTIR_GI in the reference)
            if (!r->gi) s = zr_gi_pass_create(r->width, r->height, &r->gi);
            else s = zr_gi_pass_reset_temporal(r->gi);
            if (s == ZR_OK) s = zr_gi_pass_set_method(r->gi, method);
            if (s == ZR_OK) s = r->ApplyShard();
        }
        else
            s = zr_indirect_pass_reset_temporal(r->indirect);
        if (s != ZR_OK) return s;
        r->integrator = method;
        return ZR_OK;
    }
    // SVGF between Compositing and TAA (enable != 0 creates the pass with its defaults; 0 removes it and its history)
    zr_status zr_renderer_set_denoiser(zr_renderer* r, int enable, zr_svgf_pass** out_pass)
    {
        if (!r) return ZR_ERR_INVALID_ARG;
        zr_status s = ZR_OK;
        if (enable && !r->svgf)
        {
            s = zr_svgf_pass_create(r->width, r->height, &r->svgf);
            if (s == ZR_OK) s = r->ApplyShard();
            if (s != ZR_OK && r->svgf) { zr_svgf_pass_destroy(r->svgf); r->svgf = nullptr; }
        }
        if (!enable && r->svgf) { zr_svgf_pass_destroy(r->svgf); r->svgf = nullptr; }
        if (out_pass) *out_pass = r->svgf;
        return s;
    }
    // AutoExposure + Display after TAA (enable != 0 creates both with their defaults; 0 removes both and the exposure history)
    zr_status zr_renderer_set_display(zr_renderer* r, int enable, zr_auto_exposure_pass** out_ae, zr_display_pass** out_display)
    {
        if (!r) return ZR_ERR_INVALID_ARG;
        zr_status s = ZR_OK;
        if (enable && !r->ae)
        {
            s = zr_auto_exposure_pass_create(r->width, r->height, &r->ae);
            if (s == ZR_OK) s = zr_display_pass_create(r->width, r->height, &r->display);
            if (s == ZR_OK) s = r->ApplyShard();
            if (s != ZR_OK) r->ReleaseDisplay();
        }
        if (!enable) r->ReleaseDisplay();
        if (out_ae) *out_ae = r->ae;
        if (out_display) *out_display = r->display;
        return s;
    }
    // Sky (PathTracer.cpp:165-185): enable != 0 creates a 256 x 128 sky-view LUT (DefaultRendererImpl.h:165-166) that every frame
    // recomputes before DirectLighting, on DirectLighting's stream, and that DirectLighting and Compositing read for the background of
    // pixels without geometry; 0 detaches it and frees it. A strip-sharded frame computes the whole LUT on every rank.
    zr_status zr_renderer_set_sky(zr_renderer* r, int enable, zr_sky_pass** out_pass)
    {
        if (!r) return ZR_ERR_INVALID_ARG;
        zr_status s = ZR_OK;
        if (enable && !r->sky)
        {
            zr_image2d lut{};
            s = zr_sky_pass_create(256, 128, &r->sky);
            if (s == ZR_OK) s = zr_sky_pass_get_output(r->sky, &lut);
            if (s == ZR_OK) s = zr_direct_pass_set_sky(r->direct, &lut);
            if (s == ZR_OK) s = zr_compositing_pass_set_sky(r->compositing, &lut);
            if (s != ZR_OK) r->ReleaseSky();
        }
        if (!enable) r->ReleaseSky();
        if (out_pass) *out_pass = r->sky;
        return s;
    }
    zr_status zr_renderer_get_display_output(zr_renderer* r, zr_image2d* out)
    {
        if (!r || !out) return ZR_ERR_INVALID_ARG;
        if (!r->display) { zr::set_error("zr_renderer_get_display_output: the display stage is off (zr_renderer_set_display)"); return ZR_ERR_NOT_INITIALIZED; }
        return zr_display_pass_get_output(r->display, out);
    }
    zr_status zr_renderer_set_shard(zr_renderer* r, zr_comm* comm, const uint32_t* bounds, int gather_output)
    {
        if (!r) return ZR_ERR_INVALID_ARG;
        if (!comm)
        {
            r->comm = nullptr; r->world = 1; r->rank = 0; r->bounds.clear();
            return r->ApplyShard();
        }
        if (!bounds) { zr::set_error("zr_renderer_set_shard: bounds missing"); return ZR_ERR_INVALID_ARG; }
        int rank = 0, world = 1;
        zr_status s = zr_comm_rank(comm, &rank, &world);
        if (s != ZR_OK) return s;
        if (bounds[0] != 0 || bounds[world] != r->height) { zr::set_error("zr_renderer_set_shard: bounds must cover [0, height)"); return ZR_ERR_INVALID_ARG; }
        for (int q = 0; q < world; q++)
            if (bounds[q + 1] <= bounds[q] || (q + 1 < world && bounds[q + 1] % 32 != 0))
            {
                zr::set_error("zr_renderer_set_shard: strip bounds must increase and be multiples of 32 rows");
                return ZR_ERR_INVALID_ARG;
            }
        r->comm = comm; r->rank = rank; r->world = world; r->gatherOutput = gather_output != 0;
        r->bounds.assign(bounds, bounds + world + 1);
        return r->ApplyShard();
    }
    zr_status zr_renderer_get_gi_pass(zr_renderer* r, zr_gi_pass** gi)
    {
        if (!r || !gi) return ZR_ERR_INVALID_ARG;
        *gi = r->gi;        // NULL until ReSTIR GI has been selected once
        return ZR_OK;
    }
    // The host decisions of DefaultRenderer::Update for an emissive-lit scene (DefaultRenderer.cpp:361-363, 439-478 with
    // the constants of DefaultRendererImpl.h:37-43): presampled sets 128 x 512 iff the scene has at least
    // 0.5 MB / sizeof(PresampledEmissiveTriangle) = 13107 emissive triangles; the light voxel grid (32 x 8 x 40 voxels of
    // half-extents 0.6 x 0.45 x 0.6, y offset 0.1) only together with presampling.
    zr_status zr_renderer_apply_scene_settings(zr_renderer* r, int use_lvg, uint32_t out_applied[2])
    {
        if (!r) return ZR_ERR_INVALID_ARG;
        const zr_alias_entry* table = nullptr; uint32_t numEmissive = 0;
        zr_status s = zr_scene_get_alias_table(r->scene, &table, &numEmissive);
        if (s != ZR_OK) return s;
        constexpr uint32_t MIN_NUM_LIGHTS_PRESAMPLING = (uint32_t)((0.5 * 1024 * 1024) / sizeof(zr_presampled_tri));
        static_assert(MIN_NUM_LIGHTS_PRESAMPLING == 13107, "sizeof(PresampledEmissiveTriangle) must be 40");
        const bool presampling = numEmissive >= MIN_NUM_LIGHTS_PRESAMPLING;
        const bool lvg = use_lvg && presampling;
        s = presampling ? zr_scene_set_presampling(r->scene, 128, 512) : zr_scene_set_presampling(r->scene, 0, 0);
        if (s != ZR_OK) return s;
        const uint32_t dim[3] = { 32, 8, 40 }, none[3] = { 0, 0, 0 };
        const float ext[3] = { 0.6f, 0.45f, 0.6f };
        s = zr_scene_set_light_voxel_grid(r->scene, lvg ? dim : none, ext, 0.1f);
        if (s != ZR_OK) return s;
        if (out_applied) { out_applied[0] = presampling; out_applied[1] = lvg; }
        return ZR_OK;
    }

    zr_status zr_renderer_get_output(zr_renderer* r, zr_image2d* out)
    {
        if (!r || !out) return ZR_ERR_INVALID_ARG;
        return zr_taa_pass_get_output(r->taa, out);
    }
    zr_status zr_renderer_get_passes(zr_renderer* r, zr_gbuffer_pass** g, zr_direct_pass** d, zr_indirect_pass** i,
        zr_compositing_pass** c, zr_taa_pass** t)
    {
        if (!r) return ZR_ERR_INVALID_ARG;
        if (g) *g = r->gbufferPass;
        if (d) *d = r->direct;
        if (i) *i = r->indirect;
        if (c) *c = r->compositing;
        if (t) *t = r->taa;
        return ZR_OK;
    }
    zr_status zr_renderer_get_gbuffer(zr_renderer* r, int previous, zr_gbuffer* out)
    {
        if (!r || !out) return ZR_ERR_INVALID_ARG;
        *out = r->gbuffer[previous ? r->curr ^ 1 : r->curr];
        return ZR_OK;
    }
}
