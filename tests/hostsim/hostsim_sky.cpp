// hostsim_sky.cpp -- TEST INFRASTRUCTURE. Host (g++) build of the sky header (zetaray_b200/csrc/zr_sky.cuh): the LUT texels
// k_sky_view_lut stores and the background compositing and DirectLighting write. A translation unit of its own.
#include "prelude.h"
#include "hostsim_sky_api.h"
#include "../../zetaray_b200/csrc/zr_sky.cuh"

namespace zr
{
void set_error(const char*, ...) {}
}

extern "C" void hsky_view_lut(const zr_frame_constants* fc, uint32_t lut_w, uint32_t lut_h, uint32_t* out)
{
    for (uint32_t y = 0; y < lut_h; y++)
        for (uint32_t x = 0; x < lut_w; x++)
            out[(size_t)y * lut_w + x] = zr::pack_r11g11b10(zr::Sky::SkyViewTexel(*fc, x, y, lut_w, lut_h));
}

extern "C" void hsky_background(const zr_frame_constants* fc, const uint32_t* lut, uint32_t lut_w, uint32_t lut_h, float* out)
{
    const zr::Sky::LutView view{ lut, lut_w, lut_h };
    for (uint32_t y = 0; y < fc->RenderHeight; y++)
        for (uint32_t x = 0; x < fc->RenderWidth; x++)
        {
            const float3 c = zr::Sky::Le_SkyWithSunDisk(*fc, view, x, y);
            const size_t i = (size_t)y * fc->RenderWidth + x;
            out[3 * i] = c.x; out[3 * i + 1] = c.y; out[3 * i + 2] = c.z;
        }
}
