/* hostsim_api.h -- every entry point of the host builds of the device source (libhostsim.so, libhostsim_di.so, libhostsim_io.so)
 * and every struct that crosses into Python.
 *
 * Plain C types only, so that one parser (zetaray_b200/_lib.prototypes) gives tests/hostsim's loaders each function's ctypes
 * types and a C compiler can lay out the structs for the layout test. Each hostsim*.cpp includes this header, so a definition
 * whose types differ from its declaration does not compile. The BSDF probes take the oracle's surface (orc_surface_desc). */
#ifndef HOSTSIM_API_H
#define HOSTSIM_API_H

#include "../../include/zr_abi.h"
#include "../../oracle/orc_api.h"

#ifdef __cplusplus
extern "C" {
#endif

#define HOSTSIM_API __attribute__((visibility("default")))

/* A scene resident in host memory, in the device's layouts: the flat buffers as uploaded, the BVH of zr_bvh_build_host, and
 * optionally the presampled emissive sets and the light voxel grid. */
typedef struct hostsim_scene
{
    const void* vertices;
    const uint32_t* indices;
    const void* instances;
    const void* materials;
    const void* emissives;
    const void* aliasTable;
    const void* nodes;
    const float* leafTris;
    const uint32_t* triMesh;
    const uint32_t* meshFirstTri;
    const uint16_t* rho;
    uint32_t numInstances;
    uint32_t numEmissives;
    uint32_t numTris;
    const void* sampleSets;
    uint32_t numSampleSets;
    uint32_t sampleSetSize;
    const void* lvg;
    uint32_t lvgDim[3];
    float lvgExtents[3];
    float lvgOffsetY;
} hostsim_scene;

/* ---- libhostsim.so (hostsim.cpp): traversal, BSDF, storage codecs, ray queries, ReSTIR PT and ReSTIR GI probes ---- */
/* rays: n x {origin xyz, tmin, dir xyz, tmax}; hits: n x {t, u, v, triGlobal-as-float-bits}; anyFlags (any-hit) may be null */
HOSTSIM_API int hostsim_trace(const void* nodes, const float* leafTris, const uint32_t* triMesh, const uint32_t* meshFirstTri,
    const float* rays, uint32_t n, float* hits, uint32_t* anyFlags, const uint32_t* ignoreIDs, int threads);
HOSTSIM_API int hostsim_brute(const float* worldTris, uint32_t numTris, const float* rays, uint32_t n, float* hits, int threads);
HOSTSIM_API uint64_t hostsim_validate(const void* nodes, uint32_t numNodes, const float* leafTris, uint32_t numTris, uint64_t stats[4]);
HOSTSIM_API int hostsim_trace_stats(const void* nodes, const float* leafTris, const uint32_t* triMesh, const uint32_t* meshFirstTri,
    const float* rays, uint32_t n, uint32_t* outNodes, uint32_t* outTris, int anyhit);
HOSTSIM_API void hostsim_set_rho_lut(const uint16_t* data);
HOSTSIM_API void hostsim_bsdf_sample(const orc_surface_desc* d, uint32_t seed, float* out);
HOSTSIM_API void hostsim_bsdf_sample_nodiffuse(const orc_surface_desc* d, uint32_t seed, float* out);
HOSTSIM_API void hostsim_bsdf_eval_sampler(const orc_surface_desc* d, const float* wi, uint32_t lobe, uint32_t seed, float* out);
HOSTSIM_API float hostsim_bsdf_sampler_pdf(const orc_surface_desc* d, const float* wi, uint32_t seed);
HOSTSIM_API float hostsim_bsdf_sampler_pdf_nodiffuse(const orc_surface_desc* d, const float* wi);
HOSTSIM_API void hostsim_bsdf_unified(const orc_surface_desc* d, const float* wi, float* out);
HOSTSIM_API void hostsim_oct32_roundtrip(const float* in, int n, float* out, uint32_t* enc);
HOSTSIM_API uint32_t hostsim_pack_r11g11b10(float r, float g, float b);
HOSTSIM_API void hostsim_unpack_r11g11b10(uint32_t p, float* out);
HOSTSIM_API uint32_t hostsim_pack_snorm16x2(float x, float y);
HOSTSIM_API void hostsim_unpack_snorm16x2(uint32_t p, float* out);
HOSTSIM_API uint32_t hostsim_pack_half2(float a, float b);
HOSTSIM_API void hostsim_probe_path_vertex(const hostsim_scene* hsc, const float* in, uint32_t seed, uint32_t* out);
HOSTSIM_API void hostsim_probe_emissive_and_visibility(const hostsim_scene* hsc, const float* in, uint32_t* out);
HOSTSIM_API void hostsim_probe_sample_light(const hostsim_scene* hsc, const float* pos3, uint32_t sampleSetIdx, uint32_t seed, int advance,
    uint32_t* out);
HOSTSIM_API void hostsim_probe_rpt_reservoir(const zr_rpt_reservoir* in, uint32_t n, uint32_t M_max, zr_rpt_reservoir* out,
    zr_rpt_reservoir* out2);
HOSTSIM_API void hostsim_probe_rpt_shift(const hostsim_scene* hsc, const float* ray6, const zr_rpt_reservoir* rec, float alpha_min,
    uint32_t* out);
HOSTSIM_API void hostsim_probe_load_pixels(const hostsim_scene* hsc, const zr_frame_constants* fc, const void* core, const void* coat,
    int prev, uint32_t* out);
HOSTSIM_API void hostsim_probe_lvg_sample(const hostsim_scene* hsc, const zr_frame_constants* fc, const float* pos3, uint32_t seed,
    uint32_t* out);
HOSTSIM_API void hostsim_probe_rgi_temporal(const hostsim_scene* hsc, const zr_frame_constants* fc, const void* core, const void* me,
    const void* coat, const void* pcore, const void* pcoat, const zr_rgi_reservoir* prevRes, const zr_rgi_reservoir* initial, int x, int y,
    uint32_t seed, uint32_t M_max, uint32_t* out);

/* ---- libhostsim_di.so (hostsim_di.cpp): ReSTIR DI probes (the light voxel grid fields of the scene are not read) ---- */
HOSTSIM_API void hostsim_probe_rdi_pixel(const hostsim_scene* hsc, const zr_frame_constants* fc, const void* core, const void* me,
    const void* coat, const void* pcore, const void* pcoat, const zr_rdi_reservoir* prevRes, int x, int y, uint32_t sampleSetIdx,
    int temporal, uint32_t M_max, uint32_t* out);
HOSTSIM_API void hostsim_probe_rdi_pairwise(const hostsim_scene* hsc, const zr_frame_constants* fc, const void* core, const void* coat,
    const zr_rdi_reservoir* res, const void* target, int x, int y, const int* nx, const int* ny, int numNeighbors, uint32_t seed,
    uint32_t* out);

/* ---- libhostsim_io.so (hostsim_io.cpp): ReSTIR PT per-pixel I/O and the oct32 codec ---- */
HOSTSIM_API void hostsim_probe_copy_to_next_frame(const zr_rpt_reservoir* in, uint32_t n, uint32_t M_max, zr_rpt_reservoir* out,
    zr_rpt_reservoir* ref, uint32_t* usedShortCut);
HOSTSIM_API uint64_t hostsim_oct32_round_trip(int threads, uint64_t* boundaryChanged);

#ifdef __cplusplus
}
#endif

#endif
