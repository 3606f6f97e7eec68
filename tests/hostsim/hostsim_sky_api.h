/* hostsim_sky_api.h -- entry points of libhostsim_sky.so: the sky header (zetaray_b200/csrc/zr_sky.cuh) compiled for the host, so
 * tests compare it with the oracle's restatement (oracle/sky) without a GPU. Plain C types only, parsed by
 * zetaray_b200/_lib.prototypes. */
#ifndef HOSTSIM_SKY_API_H
#define HOSTSIM_SKY_API_H

#include "../../include/zr_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define HSKY_API __attribute__((visibility("default")))

/* k_sky_view_lut's texels: packed R11G11B10F, row-major */
HSKY_API void hsky_view_lut(const zr_frame_constants* fc, uint32_t lut_w, uint32_t lut_h, uint32_t* out);
/* Sky::Le_SkyWithSunDisk for every pixel of the frame (3 floats each) */
HSKY_API void hsky_background(const zr_frame_constants* fc, const uint32_t* lut, uint32_t lut_w, uint32_t lut_h, float* out);

#ifdef __cplusplus
}
#endif

#endif
