/* sky_api.h -- entry points of libsky.so: the sky-view LUT and the sky behind geometry restated on the CPU (test infrastructure,
 * not product code).
 *
 * Sources restated: Common/Volumetric.hlsli (atmosphere), Math.hlsli:104-134 (ArcCos, SphericalToCartesian / FromCartesian),
 * Sky/SkyViewLUT.hlsl (the LUT), Common/LightSource.hlsli:158-199 (Le_Sky, Le_SkyWithSunDisk), and the two places the sky is
 * written: Compositing.hlsl:43-47 (frames that do not accumulate) and ReSTIR_DI_Temporal.hlsl:274-285 (frames that do).
 * Plain C types only, parsed by zetaray_b200/_lib.prototypes like orc_api.h. */
#ifndef SKY_API_H
#define SKY_API_H

#include "../orc_api.h"

#ifdef __cplusplus
extern "C" {
#endif

#define SKY_API __attribute__((visibility("default")))

/* zr_atan2f (include/zr_fpmath.h) over n pairs */
SKY_API void sky_atan2f(const float* y, const float* x, uint32_t n, float* out);

/* SkyViewLUT.hlsl: the lut_w x lut_h LUT as packed R11G11B10F texels (row-major) */
SKY_API void sky_view_lut(const zr_frame_constants* fc, uint32_t lut_w, uint32_t lut_h, uint32_t* out);

/* Light::Le_Sky for n directions (3 floats each) over a packed LUT; out: 3 floats each */
SKY_API void sky_le_sky(const uint32_t* lut, uint32_t lut_w, uint32_t lut_h, const float* wi, uint32_t n, float* out);

/* Light::Le_SkyWithSunDisk for every pixel of the frame: out 3 floats per pixel; sun (may be NULL) 1 where the sun disk is shown */
SKY_API void sky_background(const zr_frame_constants* fc, const uint32_t* lut, uint32_t lut_w, uint32_t lut_h, float* out,
    uint8_t* sun);

/* Compositing.hlsl:43-47 over a composited image (float4 per pixel, from orc_compositing): pixels without geometry of a frame that
 * does not accumulate become Le_SkyWithSunDisk when emissive_di is set and 0 otherwise (alpha 0) */
SKY_API void sky_composite(const zr_frame_constants* fc, const uint32_t* core, const uint32_t* lut, uint32_t lut_w, uint32_t lut_h,
    uint32_t emissive_di, float* composited);

/* ReSTIR_DI_Temporal.hlsl:274-281 in a frame with Accumulate && CameraStatic: each pixel without geometry of DirectLighting's
 * output final_img becomes before's rgb, kept only when NumFramesCameraStatic > 1, plus Le_SkyWithSunDisk; alpha is before's.
 * before and final_img are float4 per pixel; other frames and other pixels are left as they are. */
SKY_API void sky_di_accumulate(const zr_frame_constants* fc, const uint32_t* core, const uint32_t* lut, uint32_t lut_w,
    uint32_t lut_h, const float* before, float* final_img);

#ifdef __cplusplus
}
#endif

#endif
