// sky.cu -- the Sky pass: the sky-view LUT (Sky/Sky.cpp:120-147, Sky/SkyViewLUT.hlsl). Inscattering is not part of it.
//
// One thread per texel in 8x8 blocks like SKY_VIEW_LUT_THREAD_GROUP_SIZE_X/Y (Sky_Common.h:6-7); each texel marches 32 steps along its
// view ray and 8 towards the sun from each step (zr_sky.cuh). The LUT is R11G11B10F, stored as packed uint32 texels.
#include "zr_sky.cuh"
#include "zr_planes.h"

namespace zr
{
namespace
{
    __global__ void __launch_bounds__(64) k_sky_view_lut(zr_frame_constants fc, uint32_t* __restrict__ lut, uint32_t lutW, uint32_t lutH)
    {
        const uint32_t x = blockIdx.x * 8 + (threadIdx.x & 7);
        const uint32_t y = blockIdx.y * 8 + (threadIdx.x >> 3);
        if (x >= lutW || y >= lutH) return;
        lut[(size_t)y * lutW + x] = pack_r11g11b10(Sky::SkyViewTexel(fc, x, y, lutW, lutH));
    }

    bool finite(float v) { return v == v && fabsf(v) <= 3.402823466e+38f; }
}
} // namespace zr

struct zr_sky_pass
{
    uint32_t width = 0, height = 0;     // the LUT's size (DefaultRendererImpl.h:165-166 uses 256 x 128)
    struct Sized
    {
        zr::Planes planes{ "zr_sky_pass" };
        uint32_t* d_lut = nullptr;
    } sz;

    zr_status Setup() { return ZR_OK; }
    zr_status OnWindowResized(uint32_t w, uint32_t h)
    {
        Sized next;
        ZR_TRY(next.planes.Alloc(next.d_lut, (size_t)w * h));
        ZR_TRY(next.planes.Clear());
        sz = std::move(next);
        width = w; height = h;
        return ZR_OK;
    }
    zr_status Render(const zr_frame_inputs* in, cudaStream_t stream)
    {
        using namespace zr;
        if (!in)
        {
            set_error("zr_sky_pass_render: missing frame inputs");
            return ZR_ERR_INVALID_ARG;
        }
        const zr_frame_constants& fc = in->frame;
        const float consts[] = { fc.PlanetRadius, fc.AtmosphereAltitude, fc.SunDir[0], fc.SunDir[1], fc.SunDir[2], fc.SunIlluminance,
            fc.RayleighSigmaSColor[0], fc.RayleighSigmaSColor[1], fc.RayleighSigmaSColor[2], fc.RayleighSigmaSScale,
            fc.OzoneSigmaAColor[0], fc.OzoneSigmaAColor[1], fc.OzoneSigmaAColor[2], fc.OzoneSigmaAScale, fc.MieSigmaS, fc.MieSigmaA, fc.g };
        for (float v : consts)
            if (!finite(v))
            {
                set_error("zr_sky_pass_render: the atmosphere constants must be finite");
                return ZR_ERR_INVALID_ARG;
            }
        if (!(fc.PlanetRadius > 0.0f) || !(fc.AtmosphereAltitude > 0.0f))
        {
            set_error("zr_sky_pass_render: PlanetRadius (%g) and AtmosphereAltitude (%g) must be positive", fc.PlanetRadius,
                fc.AtmosphereAltitude);
            return ZR_ERR_INVALID_ARG;
        }
        const dim3 grid((width + 7) / 8, (height + 7) / 8);
        ZR_PROF("k_sky_view_lut", stream);
        k_sky_view_lut<<<grid, 64, 0, stream>>>(fc, sz.d_lut, width, height);
        ZR_LAUNCH_CHECK();
        return ZR_OK;
    }
};

extern "C"
{
    zr_status zr_sky_pass_create(uint32_t lut_w, uint32_t lut_h, zr_sky_pass** out) { return zr::CreatePass("zr_sky_pass", lut_w, lut_h, out); }
    zr_status zr_sky_pass_render(zr_sky_pass* p, const zr_frame_inputs* in, void* stream)
    {
        if (!p) return ZR_ERR_INVALID_ARG;
        return p->Render(in, (cudaStream_t)stream);
    }
    zr_status zr_sky_pass_get_output(zr_sky_pass* p, zr_image2d* out)
    {
        if (!p || !out) return ZR_ERR_INVALID_ARG;
        *out = zr_image2d{ p->sz.d_lut, p->width, p->height, p->width * 4u, 4u };
        return ZR_OK;
    }
    zr_status zr_sky_pass_describe_io(zr_sky_pass* p, zr_resource_use* uses, int* n)
    {
        if (!p || !uses || !n) return ZR_ERR_INVALID_ARG;
        uses[0] = zr_resource_use{ ZR_RES_SKY_VIEW_LUT, 1 };
        *n = 1;
        return ZR_OK;
    }
    void zr_sky_pass_destroy(zr_sky_pass* p) { delete p; }
}
