/* orc_api.h -- every entry point of the CPU oracle (liborc.so) and every struct that crosses into Python.
 *
 * Plain C types only, so that one parser (zetaray_b200/_lib.prototypes) gives tests/orc.py each function's ctypes types and a C
 * compiler can lay out the structs for the layout test. Every orc_*.cpp that defines an entry point includes this header, so a
 * definition whose types differ from its declaration does not compile.
 *
 * G-buffer and image planes are passed as their words: a core texel is 4 uint32_t, a motion/emissive or coat texel 2, a
 * colour texel 4 float. A scene is the opaque handle orc_scene_create returns. */
#ifndef ORC_API_H
#define ORC_API_H

#include "../include/zr_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_API __attribute__((visibility("default")))

/* A BSDF probe surface: BSDF::ShadingData::Init's arguments. tests/hostsim's probes take the same struct. */
typedef struct orc_surface_desc
{
    float normal[3];
    float wo[3];
    uint32_t metallic;
    float roughness;
    float baseColor[3];
    float eta_curr;
    float eta_next;
    uint32_t specTr;
    float trDepth;
    float subsurface;
    float coat_weight;
    float coat_color[3];
    float coat_roughness;
    float coat_ior;
} orc_surface_desc;

/* The planes ReSTIR PT keeps across frames: two reservoir buffers (which is current is orc_rpt_render's state[0]), the target
 * and final colour (float4 per pixel), the spatial neighbour and the two sort thread maps (uint16_t per pixel). */
typedef struct orc_rpt_buffers
{
    zr_rpt_reservoir* res[2];
    float* target;
    float* finalImg;
    uint16_t* neighbor;
    uint16_t* threadMapCtN;
    uint16_t* threadMapNtC;
} orc_rpt_buffers;

/* ---- alias table, RNG and Halton (orc_alias.cpp) ---- */
ORC_API float orc_kahan_sum(const float* data, int64_t N, int prologue);
ORC_API void orc_alias_normalize(float* w, int64_t N, int prologue);
ORC_API void orc_alias_build(float* probs, int64_t N, int prologue, void* table);
ORC_API void orc_alias_build_emissive(float* probs, int64_t N, int prologue, void* table);
ORC_API void orc_alias_sample(const void* table, int64_t N, uint64_t stream_id, int num_draws, uint32_t* out_idx, float* out_pdf);
ORC_API void orc_rng64_stream(uint64_t stream_id, int mode, uint32_t bound, int count, uint32_t* out_u, float* out_f);
ORC_API void orc_alias_sample_gpu(const void* table, uint32_t N, uint32_t seed, uint32_t num_draws, uint32_t* out_idx, float* out_pdf);
ORC_API float orc_halton(int i, int b);
ORC_API void orc_pcg3d(uint32_t x, uint32_t y, uint32_t z, uint32_t out[3]);
ORC_API void orc_pcg4d(uint32_t x, uint32_t y, uint32_t z, uint32_t w, uint32_t out[4]);
ORC_API uint32_t orc_pcg(uint32_t x);
ORC_API void orc_rng32_stream(uint32_t seed, int count, uint32_t* out_u, float* out_f);

/* ---- auto exposure and display (orc_display.cpp) ---- */
ORC_API void orc_lum_bins(const float* signal, int64_t n, const zr_auto_exposure_params* p, uint32_t* bins);
ORC_API void orc_lum_histogram(const float* signal, uint32_t W, uint32_t y0, uint32_t y1, const zr_auto_exposure_params* p, uint32_t* hist);
ORC_API void orc_exposure(const uint32_t* hist, uint32_t numPixels, const zr_auto_exposure_params* p, float dt, float* state);
ORC_API void orc_display(const uint16_t* taa, uint32_t W, uint32_t y0, uint32_t y1, const zr_display_params* p, const float* exposure,
    const uint32_t* lut, uint32_t* out);
ORC_API void orc_rgb9e5_decode(const uint32_t* v, int64_t n, float* rgb);
ORC_API void orc_srgb_oetf(const float* v, int64_t n, float* out);
ORC_API void orc_tonemap(const float* rgb, int64_t n, const zr_display_params* p, const uint32_t* lut, float* out);

/* ---- G-buffer debug views, picking and outline (orc_display_views.cpp) ---- */
ORC_API uint32_t orc_gbuffer_pick(void* scene, const zr_frame_constants* fc, uint32_t x, uint32_t y);
ORC_API void orc_display_view(const uint32_t* core, const uint32_t* me, const uint32_t* coat, uint32_t W, uint32_t y0, uint32_t y1,
    uint32_t view, float roughnessTh, float cameraNear, uint32_t* out);
ORC_API void orc_raster_world_tris(const float* tris, uint32_t n, const zr_frame_constants* fc, uint32_t y0, uint32_t y1, int count_mode,
    uint32_t bit, uint32_t* out);
ORC_API void orc_raster_pixel_tris(const float* tris, uint32_t n, uint32_t W, uint32_t H, uint32_t* out);
ORC_API void orc_pick_mask(void* scene, const zr_frame_constants* fc, const uint32_t* inst, uint32_t n, uint32_t y0, uint32_t y1,
    uint32_t* mask);
ORC_API void orc_outline(const uint32_t* mask, uint32_t W, uint32_t H, uint32_t y0, uint32_t y1, uint32_t* out);

/* ---- scene, ray queries, G-buffer, presampling and the light voxel grid (orc_gbuffer.cpp) ---- */
ORC_API void orc_set_rho_lut(const uint16_t* data);
ORC_API void* orc_scene_create(const zr_vertex* v, const uint32_t* idx, const zr_mesh_instance* inst, uint32_t numInst,
    const uint32_t* instNumTris, const zr_material* mats, const zr_emissive_tri* em, uint32_t numEm, const zr_alias_entry* alias);
ORC_API void orc_scene_destroy(void* s);
ORC_API uint32_t orc_scene_num_tris(void* s);
ORC_API void orc_scene_get_tris(void* s, float* out);
ORC_API void orc_trace_closest(void* s, const float* rays, uint32_t n, float* hits);
ORC_API void orc_trace_any(void* s, const float* rays, uint32_t n, uint32_t* flags);
ORC_API void orc_gbuffer(void* scene, const zr_frame_constants* fc, uint32_t* core, float* depthPlane, uint32_t* me, uint32_t* coat,
    uint32_t* tridiff, int nthreads);
ORC_API void orc_presample(void* scene, uint32_t frameNum, uint32_t numTotal, zr_presampled_tri* out);
ORC_API void orc_scene_set_sample_sets(void* scene, const zr_presampled_tri* sets, uint32_t numSets, uint32_t setSize);
ORC_API void orc_scene_set_lvg(void* scene, const zr_voxel_sample* lvg, const uint32_t dim[3], const float extents[3], float offset_y);
ORC_API void orc_build_lvg(void* scene, const zr_frame_constants* fc, zr_voxel_sample* out);
ORC_API void orc_estimate_power(void* scene, float* power);

/* ---- compositing, firefly filter and TAA (orc_post.cpp) ---- */
ORC_API void orc_compositing(const zr_frame_constants* fc, const uint32_t* core, const float* direct, const float* indirect, float* out);
ORC_API void orc_firefly(const zr_frame_constants* fc, const uint32_t* core, const float* in, float* out);
ORC_API void orc_taa(const zr_frame_constants* fc, const uint32_t* core, const uint32_t* motionEmissive, const float* signal,
    const uint32_t* prevOut, uint32_t* out, float blendWeight, int temporalIsValid);

/* ---- ReSTIR DI (orc_rdi.cpp) ---- */
ORC_API void orc_rdi_set_sample_pattern(const float* p);
ORC_API void orc_rdi_render(void* scene, const zr_frame_constants* fc, const uint32_t* core, const uint32_t* me, const uint32_t* coat,
    const uint32_t* pcore, const uint32_t* pcoat, const zr_direct_params* p, zr_rdi_reservoir* res0, zr_rdi_reservoir* res1,
    uint32_t* target, float* finalImg, uint32_t* state, int nthreads);
ORC_API void orc_probe_rdi_pixel(void* scene, const zr_frame_constants* fc, const uint32_t* core, const uint32_t* me, const uint32_t* coat,
    const uint32_t* pcore, const uint32_t* pcoat, const zr_rdi_reservoir* prevRes, int x, int y, uint32_t sampleSetIdx, int temporal,
    uint32_t M_max, uint32_t* out);
ORC_API void orc_probe_rdi_pairwise(void* scene, const zr_frame_constants* fc, const uint32_t* core, const uint32_t* coat,
    const zr_rdi_reservoir* res, const void* target, int x, int y, const int* nx, const int* ny, int numNeighbors, uint32_t seed,
    uint32_t* out);

/* ---- plain path tracer and ReSTIR GI (orc_rgi.cpp) ---- */
ORC_API void orc_pt_render(void* scene, const zr_frame_constants* fc, const uint32_t* core, const uint32_t* me, const uint32_t* coat,
    const zr_gi_params* p, float* finalImg, int nthreads);
ORC_API void orc_rgi_render(void* scene, const zr_frame_constants* fc, const uint32_t* core, const uint32_t* me, const uint32_t* coat,
    const uint32_t* pcore, const uint32_t* pcoat, const zr_gi_params* p, zr_rgi_reservoir* res0, zr_rgi_reservoir* res1, float* finalImg,
    uint32_t* state, int nthreads);
ORC_API void orc_probe_rgi_temporal(void* scene, const zr_frame_constants* fc, const uint32_t* core, const uint32_t* me, const uint32_t* coat,
    const uint32_t* pcore, const uint32_t* pcoat, const zr_rgi_reservoir* prevRes, const zr_rgi_reservoir* initial, int x, int y,
    uint32_t seed, uint32_t M_max, uint32_t* out);

/* ---- ReSTIR PT (orc_rpt.cpp) ---- */
ORC_API void orc_rpt_set_sample_pattern(const float* pattern512x2);
ORC_API void orc_rpt_render(void* scene, const zr_frame_constants* fc, const uint32_t* core, const uint32_t* me, const uint32_t* coat,
    const uint32_t* pcore, const uint32_t* pcoat, const zr_indirect_params* p, orc_rpt_buffers* b, uint32_t* state, int last_stage,
    int nthreads);

/* ---- SVGF (orc_svgf.cpp) ---- */
ORC_API void orc_svgf_temporal(const zr_frame_constants* fc, const uint32_t* core, const uint32_t* me, const float* color,
    const uint32_t* prevGuide, const uint32_t* histPrev, int historyValid, uint32_t* histCurr, uint32_t* cv, uint32_t* guide, int nthreads);
ORC_API void orc_svgf_atrous(uint32_t W, uint32_t H, const uint32_t* guide, const uint32_t* in, uint32_t* out, float* outF, uint32_t step,
    const float* params4, int nthreads);

/* ---- codec, BSDF and device-source probes (orc_testapi.cpp) ---- */
ORC_API void orc_oct32_roundtrip(const float* in, int n, float* out);
ORC_API uint32_t orc_pack_r11g11b10(float r, float g, float b);
ORC_API void orc_unpack_r11g11b10(uint32_t p, float* out);
ORC_API uint32_t orc_pack_snorm16x2(float x, float y);
ORC_API void orc_unpack_snorm16x2(uint32_t p, float* out);
ORC_API void orc_bsdf_sample(const orc_surface_desc* d, uint32_t seed, float* out);
ORC_API void orc_bsdf_eval_sampler(const orc_surface_desc* d, const float* wi, uint32_t lobe, uint32_t seed, float* out);
ORC_API float orc_bsdf_sampler_pdf(const orc_surface_desc* d, const float* wi, uint32_t seed);
ORC_API void orc_bsdf_sample_nodiffuse(const orc_surface_desc* d, uint32_t seed, float* out);
ORC_API float orc_bsdf_sampler_pdf_nodiffuse(const orc_surface_desc* d, const float* wi);
ORC_API void orc_bsdf_unified(const orc_surface_desc* d, const float* wi, float* out);
ORC_API void orc_probe_path_vertex(void* scene, const float* in, uint32_t seed, uint32_t* out);
ORC_API void orc_probe_emissive_and_visibility(void* scene, const float* in, uint32_t* out);
ORC_API void orc_probe_sample_light(void* scene, const float* pos3, uint32_t sampleSetIdx, uint32_t seed, int advance, uint32_t* out);
ORC_API void orc_probe_rpt_reservoir(const zr_rpt_reservoir* in, uint32_t n, uint32_t M_max, zr_rpt_reservoir* out, zr_rpt_reservoir* out2);
ORC_API void orc_probe_rpt_shift(void* scene, const float* ray6, const zr_rpt_reservoir* rec, float alpha_min, uint32_t* out);
ORC_API void orc_probe_load_pixels(void* scene, const zr_frame_constants* fc, const uint32_t* core, const uint32_t* coat, int prev, uint32_t* out);
ORC_API void orc_probe_lvg_sample(void* scene, const zr_frame_constants* fc, const float* pos3, uint32_t seed, uint32_t* out);

#ifdef __cplusplus
}
#endif

#endif
