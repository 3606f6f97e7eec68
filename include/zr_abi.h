/*
 * zr_abi.h -- C-ABI of the H100-native ReSTIR path-tracing core (libzetaray_b200.so).
 *
 * Every entry point replaces one piece of ZetaRay's render-pass interface for the hot path
 * (G-buffer -> pre-lighting/alias table -> ReSTIR DI -> ReSTIR PT -> compositing/firefly/TAA).
 * Citations are relative to the reference tree (alipbcs/ZetaRay @ 6fd82f1e).
 *
 * Conventions
 *  - plain C, no torch / C++ types; all "d_" pointers are CUDA device pointers, "h_" host pointers
 *  - every function returns zr_status (0 = ok) and never throws; the reference aborts through
 *    Check/CheckHR (ZetaCore/Utility/Error.h:33-92) -- here the failing call returns an error
 *    code and zr_last_error() carries the message
 *  - `stream` is a cudaStream_t passed as void*; all GPU work of a call is enqueued on it and the
 *    call returns without synchronising (== recording into a CommandList,
 *    ZetaCore/Core/RenderGraph.cpp:494-518)
 *  - a pass handle is thread-compatible: concurrent calls on different handles are allowed
 *    (ZetaCore/Core/RenderGraph.cpp:541-558)
 */
#ifndef ZR_ABI_H
#define ZR_ABI_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define ZR_API __declspec(dllexport)
#else
#define ZR_API __attribute__((visibility("default")))
#endif

typedef int32_t zr_status;
enum
{
    ZR_OK = 0,
    ZR_ERR_INVALID_ARG = 1,
    ZR_ERR_CUDA = 2,
    ZR_ERR_NOT_INITIALIZED = 3,
    ZR_ERR_UNSUPPORTED = 4,
    ZR_ERR_OUT_OF_MEMORY = 5
};

/* Last error message of the calling thread ("" if none). */
ZR_API const char* zr_last_error(void);
/* Library/ABI version: (major << 16) | minor. */
/* (major << 16) | minor; additions bump the minor. 1.1 added zr_bvh_build_host, zr_renderer_set_integrator,
 * zr_renderer_get_gi_pass, zr_renderer_apply_scene_settings and zr_gi_pass_set_method; 1.2 the SVGF pass, zr_comm, the strip-sharded
 * renderer (zr_renderer_set_shard) and zr_gi_pass_set_rows / set_halo_exchange. 1.3 removed two
 * measurement and test hooks: the ReSTIR PT execution-model switch and the two-dispatch compositing entry point. 1.4 removed
 * the stage-limited ReSTIR PT render and its stage enum, which nothing called. 1.6 added the AutoExposure and Display passes,
 * zr_renderer_set_display / get_display_output and zr_comm_allreduce_u32. 1.7 added zr_comm_create_transport (zr_comm_transport). 1.8
 * added zr_svgf_pass_set_rows / set_halo_exchange, and zr_renderer_set_shard runs the SVGF stage sharded instead of refusing it. 1.9
 * added zr_scene_update_materials and zr_scene_get_tables. 1.10 added pixel picking (zr_gbuffer_pass_pick / get_pick), the Display
 * pass's G-buffer debug views (zr_display_pass_set_view) and the outline of picked instances (zr_display_pass_set_picked). 1.11
 * added the ReSTIR PT debug views (zr_indirect_pass_set_debug_view). The sky (zr_sky_pass_*, zr_direct_pass_set_sky,
 * zr_compositing_pass_set_sky, zr_renderer_set_sky) was added without a minor of its own: the version still reads 1.11, so
 * detect those entry points by symbol. */
ZR_API uint32_t zr_abi_version(void);

/* ------------------------------------------------------------------------------------------
 * Scene data layouts -- bit-identical to the reference's GPU structs
 * ------------------------------------------------------------------------------------------ */

/* Vertex: ZetaRenderPass/Common/Common.hlsli:5-11, ZetaCore/Core/Vertex.h:8-14 (28 bytes) */
typedef struct zr_vertex
{
    float pos[3];
    float uv[2];
    uint16_t normal[2];     /* octahedral, 2 x UNORM16 */
    uint16_t tangent[2];
} zr_vertex;

/* Material: ZetaCore/Core/Material.h:29-427 (8 x u32 with bit fields, 32 bytes) */
typedef struct zr_material
{
    uint32_t BaseColorFactor;
    uint32_t BaseColorTex_Subsurf_CoatWeight;
    uint32_t NormalTex_TrDepth;
    uint32_t MRTex_SpecRoughness_CoatRoughness;
    uint32_t EmissiveFactor_NormalScale;
    uint32_t EmissiveStrength_IOR;
    uint32_t EmissiveTex_AlphaCutoff_CoatIOR;
    uint32_t CoatColor_Flags;
} zr_material;

/* RT::MeshInstance: ZetaCore/RayTracing/RtCommon.h:47-64 (64 bytes) */
typedef struct zr_mesh_instance
{
    uint32_t BaseVtxOffset;
    uint32_t BaseIdxOffset;
    uint16_t Rotation[4];       /* unorm4 quaternion */
    uint16_t Scale[3];          /* half3 */
    uint16_t MatIdx;
    uint32_t BaseEmissiveTriOffset;
    float Translation[3];
    uint16_t PrevRotation[4];
    uint16_t PrevScale[3];
    uint16_t dTranslation[3];   /* half3 */
    uint16_t BaseColorTex;
    uint16_t AlphaFactor_Cutoff;
} zr_mesh_instance;

/* RT::EmissiveTriangle: RtCommon.h:66-114 (ENCODE_EMISSIVE_POS 1, EMISSIVE_UV_HALF 1; 48 bytes) */
typedef struct zr_emissive_tri
{
    float Vtx0[3];
    uint16_t V0V1[2];           /* oct-encoded unit edge, UNORM16 */
    uint16_t V0V2[2];
    uint16_t EdgeLengths[2];    /* half2 */
    uint32_t ID;
    uint32_t PackedA;           /* [0,24) emissive factor RGB8, bit 24 id-patched, bit 25 double sided */
    uint32_t PackedB;           /* [0,16) texture, [16,32) strength (half) */
    uint16_t UV0[2];
    uint16_t UV1[2];
    uint16_t UV2[2];
} zr_emissive_tri;

/* RT::EmissiveLumenAliasTableEntry: RtCommon.h:302-310 (16 bytes) */
typedef struct zr_alias_entry
{
    float CachedP_Orig;
    float CachedP_Alias;
    float P_Curr;
    uint32_t Alias;
} zr_alias_entry;

/* cbFrameConstants: ZetaRenderPass/Common/FrameConstants.h:10-78 (same field order and offsets;
 * matrices are the reference's row_major float3x4 / float4x4). The *DescHeapOffset fields are
 * kept for layout compatibility and ignored. */
typedef struct zr_frame_constants
{
    float CurrView[3][4];
    float PrevView[3][4];
    float CurrViewInv[3][4];
    float PrevViewInv[3][4];
    float CurrViewProj[4][4];
    float PrevViewProj[4][4];

    float CameraPos[3];
    float CameraNear;

    float AspectRatio;
    float PixelSpreadAngle;
    float TanHalfFOV;
    float dt;

    uint32_t FrameNum;
    uint32_t CurrGBufferDescHeapOffset;
    uint32_t PrevGBufferDescHeapOffset;
    uint32_t BaseColorMapsDescHeapOffset;

    uint32_t NormalMapsDescHeapOffset;
    uint32_t MetallicRoughnessMapsDescHeapOffset;
    uint32_t EmissiveMapsDescHeapOffset;
    uint32_t EnvMapDescHeapOffset;

    uint32_t RenderWidth;
    uint32_t RenderHeight;
    uint32_t DisplayWidth;
    uint32_t DisplayHeight;

    float CurrCameraJitter[2];
    float PrevCameraJitter[2];

    float PlanetRadius;
    float SunCosAngularRadius;
    float SunSinAngularRadius;
    float pad;

    float SunDir[3];
    float SunIlluminance;

    float RayleighSigmaSColor[3];
    float RayleighSigmaSScale;

    float OzoneSigmaAColor[3];
    float OzoneSigmaAScale;

    float MieSigmaS;
    float MieSigmaA;
    float AtmosphereAltitude;
    float g;

    uint32_t NumFramesCameraStatic;
    uint32_t CameraStatic;
    uint32_t Accumulate;
    uint32_t SunMoved;

    float CameraRayUVGradsScale;
    float MipBias;
    float OneDivNumEmissiveTriangles;
    uint32_t NumEmissiveTriangles;

    float FocusDepth;
    float LensRadius;
    uint32_t DoF;
    uint32_t pad2;
} zr_frame_constants;

/* ------------------------------------------------------------------------------------------
 * Per-pixel state layouts in HBM (AoS records sized for 128-bit accesses)
 * ------------------------------------------------------------------------------------------ */

/* G-buffer. The reference keeps 10 textures (ZetaRenderer/Default/DefaultRendererImpl.h:97-109);
 * here the planes every consumer reads together share one 16-byte record:
 *   core[i]   = { depth (f32 bits), normal (2 x UNORM16 oct), baseColor (RGBA8),
 *                 flags | roughness(UNORM8) << 8 | ior(UNORM8) << 16 }
 *   depth[i]  = view depth again as its own 4-byte plane, so the depth-only stencil taps
 *               (firefly, TAA dilation) do not drag the 16-byte record through HBM
 *   motion_emissive[i] = { motion (2 x SNORM16), emissive (R11G11B10_FLOAT) }
 *   coat[i]   = { coatColor.rg | ..., see GBuffers.hlsli:110-121 } (3 x u16 in a uint2)
 *   tridiff[i]= 12 halves (dpdu, dpdv, dndu, dndv), GBufferRT.hlsli:159-175; optional (may be NULL)
 * Quantisation is identical to the reference formats. */
typedef struct zr_gbuffer
{
    void* d_core;               /* uint4[w*h] */
    void* d_depth;              /* float[w*h]: copy of core.x for depth-only consumers (stencils) */
    void* d_motion_emissive;    /* uint2[w*h] */
    void* d_coat;               /* uint2[w*h] */
    void* d_tridiff;            /* 3 x uint2[w*h] or NULL */
} zr_gbuffer;

#define ZR_GBUFFER_FLAG_TRANSMISSIVE 0x01u
#define ZR_GBUFFER_FLAG_EMISSIVE     0x02u
#define ZR_GBUFFER_FLAG_INVALID      0x04u
#define ZR_GBUFFER_FLAG_TRDEPTH_GT0  0x08u
#define ZR_GBUFFER_FLAG_SUBSURFACE   0x10u
#define ZR_GBUFFER_FLAG_COATED       0x20u
#define ZR_GBUFFER_FLAG_METALLIC     0x80u

/* ReSTIR PT reservoir: the reference's 7 planes A..G (IndirectLighting.h:128-144,
 * ReSTIR_PT/Reservoir.hlsli:267-463; 62 B/px) as one 64-byte record = 4 x 128-bit. */
typedef struct zr_rpt_reservoir
{
    /* q0 */
    uint32_t meta;      /* A: byte0 = (k-2 | EMPTY=0xf) | M << 4, byte1 = lobe_{k-1} | lobe_k << 3 | lt_k << 6,
                              byte2 = lt_{k+1} | x_k_in_motion << 2 */
    float w_sum;        /* B.x */
    float W;            /* B.y */
    uint32_t L_b;       /* E: half L.b (low 16 bits) */
    /* q1 = C */
    uint32_t jacobian_or_seed_nee;
    uint32_t seed_replay;
    uint32_t ID;
    uint32_t x_k_x;
    /* q2 = D */
    uint32_t x_k_y;
    uint32_t x_k_z;
    uint32_t w_k;       /* oct32: w_k | light normal | w_sky */
    uint32_t L_rg;      /* half2 */
    /* q3 = F, G */
    float lightPdf;     /* sign bit = one-sided (Shift.hlsli:131) */
    float dwdA;
    uint32_t seed_nee;
    uint32_t meshIdx;
} zr_rpt_reservoir;

/* ReSTIR DI reservoir: A RGBA32_UINT + B RG32F (DirectLighting/Emissive/Reservoir.hlsli:134-199)
 * as one 32-byte record = 2 x 128-bit. */
typedef struct zr_rdi_reservoir
{
    uint32_t bary;          /* 2 x UNORM16 */
    uint32_t le_rg;         /* half2 */
    uint32_t le_b_meta;     /* half le.b | M(5 bits) << 16 */
    uint32_t lightIdx;
    float w_sum;
    float W;
    uint32_t pad[2];
} zr_rdi_reservoir;

typedef struct zr_image2d
{
    void* d_ptr;
    uint32_t width;
    uint32_t height;
    uint32_t pitch_bytes;
    uint32_t texel_bytes;
} zr_image2d;

/* ---- Strip-sharded frames (multi-GPU; no reference counterpart, SURVEY 8e) ---------------------------------
 * A frame is split into horizontal strips whose boundaries are multiples of 32 rows (the sort tile of
 * ReSTIR_PT_Sort.hlsl:10 and a multiple of every thread-group height), one strip per device. Every pass has
 * set_rows(y0, y1): it then computes and writes rows [y0, y1) only, while reading up to 32 rows beyond them
 * (spatial neighbours <= 15 px for ReSTIR PT, Util.hlsli:9; <= 23 px for ReSTIR DI, Resampling.hlsli:418-423;
 * 1-2 px for the stencils). The lighting passes and the SVGF pass call the halo-exchange hook at the points where rows they
 * just wrote are about to be read by other strips (after temporal resampling and after every spatial or a-trous pass); the hook
 * must make the 32 rows either side of [y0, y1) of each plane coherent across devices on `stream` (the renderer's hook:
 * zr_comm_exchange_halos, one grouped send / recv of the boundary bands with the neighbouring strips, csrc/comm.cu). */
typedef void (*zr_halo_exchange_fn)(void* user, const zr_image2d* planes, int n_planes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Scene: flat buffers named in ZetaCore/Scene/SceneRenderer.h:15-33 + the acceleration structure
 * that replaces the DXR TLAS (ZetaCore/RayTracing/RtAccelerationStructure.cpp).
 * ------------------------------------------------------------------------------------------ */
typedef struct zr_scene zr_scene;

typedef struct zr_scene_desc
{
    const zr_vertex* h_vertices;            uint32_t num_vertices;
    const uint32_t* h_indices;              uint32_t num_indices;
    const zr_mesh_instance* h_instances;    uint32_t num_instances;
    /* triangles per instance (instances index consecutive ranges of the index buffer) */
    const uint32_t* h_instance_num_tris;
    const zr_material* h_materials;         uint32_t num_materials;
    /* emissive triangles already in world space with hashed IDs (SceneCore.cpp:199-235) */
    const zr_emissive_tri* h_emissives;     uint32_t num_emissives;
} zr_scene_desc;

/* Uploads the buffers, builds the 8-wide compressed BVH on the host and uploads it. */
ZR_API zr_status zr_scene_create(const zr_scene_desc* desc, zr_scene** out);
ZR_API void zr_scene_destroy(zr_scene* scene);
/* BVH statistics for tests: {num_nodes, num_tris, max_depth, bytes}. */
ZR_API zr_status zr_scene_bvh_stats(const zr_scene* scene, uint32_t out[4]);
/* The optional BSDF features the scene's materials use: the OR over its material table as zr_scene_create or the last
 * zr_scene_update_materials left it. The lighting passes read it on every render and run kernels built without clear coat,
 * specular transmission and thin-walled transmission when none is set. */
#define ZR_MATERIAL_COAT         0x1u   /* coat weight > 0 */
#define ZR_MATERIAL_TRANSMISSION 0x2u   /* transmissive flag (bit 26 of CoatColor_Flags) */
#define ZR_MATERIAL_THIN_WALLED  0x4u   /* thin-walled flag (bit 29 of CoatColor_Flags) with subsurface weight > 0 */
ZR_API zr_status zr_scene_material_features(const zr_scene* scene, uint32_t* out);

/* Scene edit between frames (SceneCore::UpdateMaterial / UpdateEmissiveMaterial, SceneCore.cpp:436, 711-715): replaces materials
 * [first, first + count) of the scene's table. The scene's geometry, instances, BVH and its set of emissive triangles are unchanged.
 *  - Refusals (ZR_ERR_INVALID_ARG, zr_last_error names the rule) are decided on the host before any work, and leave the material
 *    table, the emissive triangles, the power estimate, the alias table and zr_scene_material_features as they were: a NULL scene or
 *    h_materials, count == 0, first + count > the number of materials; an edit that gives a material a non-zero emissive factor
 *    where it had none while an instance using it has no emissive triangles (BaseEmissiveTriOffset == 0xffffffff); and, in a scene
 *    with emissive triangles, an edit after which every instance with emissive triangles uses a material of zero emissive factor
 *    or zero strength (the light distribution cannot be normalised over zero power). A light whose factor goes to zero keeps its
 *    triangles in the emissive set, with zero power.
 *  - Ordering: the material copy waits for the frames in flight (like every host-side replacement of data a frame reads), the
 *    rest is enqueued on `stream`: the next render on `stream` sees the edited scene, and no earlier frame does.
 *  - The emissive triangles of the instances whose material's emissive factor, double-sided flag or strength changed take the new
 *    bits on the device (k_refresh_emissives: PackedA's factor, double-sided and strength bits, PackedB's strength); positions,
 *    UVs, IDs and the id-patched bit stay. When any did and zr_prelighting_render has run before, the call runs it again on
 *    `stream` (power estimate + alias build), so the next frame samples the new distribution; an edit that changes no emissive
 *    bits launches no kernel. Presampled sets and the light voxel grid are redrawn every frame and need nothing.
 *  - The material features are recomputed over the whole table; the next render picks its kernel build from them.
 *  - History is left alone, as the reference leaves it: ReSTIR DI / PT / GI reservoirs that cached the old radiance age out through
 *    their M caps. To restart accumulation, render the next frame with CameraStatic = 0 and NumFramesCameraStatic = 0
 *    (DefaultRenderer.cpp:96-102 after SceneModified), or reset a pass's temporal history.
 *  - Strip-sharded frames: every rank makes the same call with the same materials; the work is deterministic, so every rank's
 *    tables end identical. */
ZR_API zr_status zr_scene_update_materials(zr_scene* scene, uint32_t first, uint32_t count, const zr_material* h_materials,
    void* stream);
/* The scene's device material table and emissive triangles (read-only; valid until zr_scene_destroy). */
ZR_API zr_status zr_scene_get_tables(const zr_scene* scene, const zr_material** d_materials, uint32_t* num_materials,
    const zr_emissive_tri** d_emissives, uint32_t* num_emissives);

/* The BVH builder alone, on host memory (no GPU needed): world-space triangles as 9 floats {v0, e1, e2} in, 80-byte
 * nodes and the leaf-order permutation out (either may be NULL to query sizes). out_info = {num_nodes, num_tris,
 * max_depth, max_traversal_stack}; zr_scene_create refuses a tree whose max_traversal_stack exceeds the kernels' stack. */
ZR_API zr_status zr_bvh_build_host(const float* h_world_tris, uint32_t num_tris, void* h_nodes, uint32_t node_capacity,
    uint32_t* h_leaf_order, uint32_t out_info[4]);

/* Ray queries through the product traversal kernel, for parity tests against the oracle's brute
 * force (mirrors RtRayQuery::Hit::FindClosest / Visibility_Segment, Common/RayQuery.hlsli:15-144,
 * 337-406). rays: n x {origin xyz, tmin, dir xyz, tmax}; hits: n x {t, bary.x, bary.y, triGlobal(u32)}. */
ZR_API zr_status zr_scene_trace_closest(const zr_scene* scene, const float* d_rays, uint32_t n,
    float* d_hits, void* stream);
ZR_API zr_status zr_scene_trace_any(const zr_scene* scene, const float* d_rays, uint32_t n,
    uint32_t* d_hit_flags, void* stream);

/* ------------------------------------------------------------------------------------------
 * Pre-lighting: power estimate + alias table (replaces EstimateTriEmissivePower.hlsl and the CPU
 * BuildAliasTable round trip, PreLighting/PreLighting.cpp:27-158, 512-585)
 * ------------------------------------------------------------------------------------------ */

/* Math::AliasTable_Normalize + BuildAliasTable on the device. d_weights is normalised in place
 * (as the reference does to its readback buffer). d_scratch: 2*n + 16 u32. Bit-exact with the CPU
 * reference for 32-byte aligned input (the production case, SURVEY 8a-1). */
ZR_API zr_status zr_alias_table_build(float* d_weights, uint32_t n, zr_alias_entry* d_table,
    uint32_t* d_scratch, void* stream);
/* Light::AliasTableSample::get (Common/LightSource.hlsli:72-97) for `num_draws` consecutive draws
 * of one RNG stream seeded RNG::Init(seed). */
ZR_API zr_status zr_alias_table_sample(const zr_alias_entry* d_table, uint32_t n, uint32_t seed,
    uint32_t num_draws, uint32_t* d_out_idx, float* d_out_pdf, void* stream);
/* EstimateTriEmissivePower (PreLighting/EstimateTriEmissivePower.hlsl:30-79): d_power[n]. */
ZR_API zr_status zr_estimate_emissive_power(const zr_scene* scene, float* d_power, void* stream);
/* Convenience used by the pre-lighting node: power estimate + alias build into the scene's own
 * alias table (frame-1 protocol, ZetaRenderer/Default/PathTracer.cpp:195-240). */
ZR_API zr_status zr_prelighting_render(zr_scene* scene, void* stream);

/* ---- Presampled emissive sets (PreLighting/PresampleEmissives.hlsl:19-44; SURVEY a-5) ----
 * num_sets x set_size power-proportional light samples drawn once per frame; every thread group of the lighting passes
 * then picks ONE set and samples it uniformly, so a group's light fetches stay inside set_size records instead of
 * scattering over the emissive buffer. The reference enables 128 x 512 when the scene has >= 13107 emissive triangles
 * (ZetaRenderer/Default/DefaultRendererImpl.h:37-41, DefaultRenderer.cpp:362) and compiles the *_WPS shader variants;
 * here the host makes the same decision with zr_scene_set_presampling and the kernels branch on it. */
typedef struct zr_presampled_tri       /* RT::PresampledEmissiveTriangle, ZetaCore/RayTracing/RtCommon.h:312-322 (40 bytes) */
{
    float pos[3];
    uint32_t normal;        /* octahedral, 2 x UNORM16 */
    float pdf;
    uint32_t ID;
    uint32_t idx;
    uint32_t bary;          /* 2 x UNORM16 */
    uint16_t le[3];         /* half3 */
    uint16_t twoSided;
} zr_presampled_tri;
#define ZR_PRESAMPLING_MIN_EMISSIVES 13107u
#define ZR_PRESAMPLING_NUM_SETS 128u
#define ZR_PRESAMPLING_SET_SIZE 512u
ZR_API zr_status zr_scene_set_presampling(zr_scene* scene, uint32_t num_sets, uint32_t set_size);  /* 0, 0 = off (default) */
ZR_API zr_status zr_presample_emissives(zr_scene* scene, uint32_t frame_num, void* stream);       /* once per frame, before lighting */
ZR_API zr_status zr_scene_get_sample_sets(zr_scene* scene, void** d_sets, uint32_t* num_sets, uint32_t* set_size);

/* ---- Light voxel grid (PreLighting/BuildLightVoxelGrid.hlsl:56-162, Common/LightVoxelGrid.hlsli; SURVEY a-6) ----
 * A camera-centred grid of grid_dim voxels (half-extents `extents`, view space, y shifted by offset_y); every frame each
 * voxel keeps 64 light samples chosen by RIS over 6 alias-table candidates with target Lum(Le) / d^2. ReSTIR GI then
 * takes its NEE light sample after the first indirect vertex from the voxel around the shading point (ReSTIR_GI_LVG
 * variant, ReSTIR_GI_NEE.hlsli:123-193) and falls back to the presampled set outside the grid, so it needs presampling
 * on (DefaultRenderer.cpp:363). The reference's defaults are 32 x 8 x 40 voxels of (0.6, 0.45, 0.6). */
typedef struct zr_voxel_sample         /* RT::VoxelSample, ZetaCore/RayTracing/RtCommon.h:324-332 (32 bytes) */
{
    float pos[3];
    uint32_t normal;        /* octahedral, 2 x UNORM16 */
    float pdf;
    uint32_t ID;
    uint16_t le[3];         /* half3 */
    uint16_t twoSided;
} zr_voxel_sample;
#define ZR_LVG_SAMPLES_PER_VOXEL 64u
ZR_API zr_status zr_scene_set_light_voxel_grid(zr_scene* scene, const uint32_t grid_dim[3], const float extents[3], float offset_y);
ZR_API zr_status zr_build_light_voxel_grid(zr_scene* scene, const zr_frame_constants* frame, void* stream);   /* once per frame */
ZR_API zr_status zr_scene_get_light_voxel_grid(zr_scene* scene, void** d_samples, uint32_t* num_samples);
ZR_API zr_status zr_scene_get_alias_table(const zr_scene* scene, const zr_alias_entry** d_table, uint32_t* n);

/* ------------------------------------------------------------------------------------------
 * Frame inputs shared by the passes (== the global resources a pass looks up by name)
 * ------------------------------------------------------------------------------------------ */
typedef struct zr_frame_inputs
{
    zr_frame_constants frame;
    zr_gbuffer curr;
    zr_gbuffer prev;
    const zr_scene* scene;
} zr_frame_inputs;

ZR_API zr_status zr_gbuffer_alloc(uint32_t width, uint32_t height, int with_tridiff, zr_gbuffer* out);
ZR_API void zr_gbuffer_free(zr_gbuffer* g);

/* Render-graph node metadata (Core/RenderGraph.h:81-105): ids are zr_resource_id below. */
typedef enum zr_resource_id
{
    ZR_RES_GBUFFER_CURR = 1, ZR_RES_GBUFFER_PREV, ZR_RES_SCENE_BVH, ZR_RES_ALIAS_TABLE,
    ZR_RES_DI_FINAL, ZR_RES_INDIRECT_FINAL, ZR_RES_COMPOSITED, ZR_RES_TAA_OUT, ZR_RES_SKY_VIEW_LUT
} zr_resource_id;
typedef struct zr_resource_use { uint32_t id; uint32_t write; } zr_resource_use;

/* ---- Pass lifetime ----
 * zr_*_pass_create / _resize take a non-zero width and height. A resize is all-or-nothing: the pass allocates and clears a
 * complete new set of planes and frees the old ones only when that succeeded, so while it runs both sets are allocated, and on
 * failure the pass is exactly as it was (same size, same planes, same history). A successful resize drops the temporal history
 * and forgets what described the old size: set_rows returns to the whole frame, the cost map and the schedule costs are unset.
 * A halo-exchange hook stays. A failed device allocation returns ZR_ERR_OUT_OF_MEMORY (ZR_ERR_CUDA for other CUDA errors),
 * with zr_last_error naming the pass and the bytes asked for. */

/* ---- GBufferRT (GBuffer/GBufferRT.h, GBufferRT.cpp:99-160) ---- */
typedef struct zr_gbuffer_pass zr_gbuffer_pass;
ZR_API zr_status zr_gbuffer_pass_create(zr_gbuffer_pass** out);
ZR_API zr_status zr_gbuffer_pass_render(zr_gbuffer_pass* p, const zr_frame_inputs* in, void* stream);
ZR_API zr_status zr_gbuffer_pass_set_rows(zr_gbuffer_pass* p, uint32_t y0, uint32_t y1);
ZR_API zr_status zr_gbuffer_pass_describe_io(zr_gbuffer_pass* p, zr_resource_use* uses, int* n);
ZR_API void zr_gbuffer_pass_destroy(zr_gbuffer_pass* p);
/* Pixel picking (DefaultRenderer::Pick -> GBufferRT::PickPixel, DefaultRenderer.cpp:558-568; GBufferRT_Inline.hlsl:241-242). A pick
 * is one-shot: the next zr_gbuffer_pass_render writes into the pass's pick word the index of the instance under pixel (x, y) (its
 * position in zr_scene_desc.h_instances), or 0xffffffff when the primary ray misses, (x, y) lies outside the frame or row y
 * outside the rows this pass renders; later renders leave the word alone. The word holds 0xffffffff from create on. Copy it to
 * the host after that render on its stream (Display.cpp:210-229, ReadbackPickIdx). */
ZR_API zr_status zr_gbuffer_pass_pick(zr_gbuffer_pass* p, uint32_t x, uint32_t y);
ZR_API zr_status zr_gbuffer_pass_get_pick(zr_gbuffer_pass* p, zr_image2d* out);        /* 1 x 1 uint32, device */

/* ---- DirectLighting (ReSTIR DI, DirectLighting/Emissive/DirectLighting.h:36-57) ---- */
typedef struct zr_direct_pass zr_direct_pass;
typedef struct zr_direct_params
{
    uint32_t temporal_resample;     /* CB_RDI_FLAGS::TEMPORAL_RESAMPLE */
    uint32_t spatial_resample;
    uint32_t stochastic_spatial;
    uint32_t extra_disocclusion_sampling;
    uint32_t M_max;                 /* default 20, DirectLighting.h:95 */
    float alpha_min;                /* default 0.05^2 */
} zr_direct_params;
typedef enum zr_direct_output { ZR_DIRECT_FINAL = 0, ZR_DIRECT_RESERVOIR_CURR, ZR_DIRECT_TARGET } zr_direct_output;
ZR_API zr_status zr_direct_pass_create(uint32_t width, uint32_t height, zr_direct_pass** out);
ZR_API zr_status zr_direct_pass_resize(zr_direct_pass* p, uint32_t width, uint32_t height);
ZR_API zr_status zr_direct_pass_reset_temporal(zr_direct_pass* p);
ZR_API zr_status zr_direct_pass_default_params(zr_direct_params* out);
ZR_API zr_status zr_direct_pass_set_params(zr_direct_pass* p, const zr_direct_params* params);
ZR_API zr_status zr_direct_pass_render(zr_direct_pass* p, const zr_frame_inputs* in, void* stream);
ZR_API zr_status zr_direct_pass_set_rows(zr_direct_pass* p, uint32_t y0, uint32_t y1);
ZR_API zr_status zr_direct_pass_set_halo_exchange(zr_direct_pass* p, zr_halo_exchange_fn fn, void* user);
/* Cost feedback (optional). set_cost_map: d_cycles[ceil(H/32)][ceil(W/32)] (uint64, device, row-major) accumulates the SM
 * cycles each 32x32-pixel tile costs while set. set_schedule_costs: the pass then launches only the thread blocks that
 * touch its rows, most expensive tile first (csrc/zr_schedule.h); h_tile_cost == NULL restores plain order. Strip
 * boundaries are chosen from the same numbers (zetaray_b200/sharding.py). Results do not depend on either call. */
ZR_API zr_status zr_direct_pass_set_cost_map(zr_direct_pass* p, void* d_cycles);
ZR_API zr_status zr_direct_pass_set_schedule_costs(zr_direct_pass* p, const double* h_tile_cost, uint32_t tiles_x, uint32_t tiles_y);
ZR_API zr_status zr_direct_pass_get_output(zr_direct_pass* p, zr_direct_output id, zr_image2d* out);
ZR_API zr_status zr_direct_pass_describe_io(zr_direct_pass* p, zr_resource_use* uses, int* n);
/* The sky in accumulating frames (ReSTIR_DI_Temporal.hlsl:274-285): with a LUT set (zr_sky_pass_get_output), each render with
 * Accumulate && CameraStatic copies FINAL's rows before it runs and afterwards sets every pixel without geometry to that copy
 * (kept only when NumFramesCameraStatic > 1) plus Le_SkyWithSunDisk, so Compositing's division by the frame count averages the
 * sky like any other pixel. Other frames leave those pixels at 0, as without a LUT. The copy is allocated only while a LUT is set.
 * lut == NULL turns it off; an image that is not a non-empty unpadded 4-byte-texel plane is refused. The pass does not own the LUT. */
ZR_API zr_status zr_direct_pass_set_sky(zr_direct_pass* p, const zr_image2d* lut);
ZR_API void zr_direct_pass_destroy(zr_direct_pass* p);

/* ---- IndirectLighting (ReSTIR PT, IndirectLighting/IndirectLighting.h:72-108) ---- */
typedef struct zr_indirect_pass zr_indirect_pass;
typedef struct zr_indirect_params
{
    uint32_t max_non_tr_bounces;    /* default 3, IndirectLighting.h:231-244 */
    uint32_t max_glossy_tr_bounces; /* default 4 */
    uint32_t russian_roulette;      /* default 1 */
    uint32_t temporal_resample;     /* default 1 */
    uint32_t num_spatial_passes;    /* default 1 */
    uint32_t M_max_temporal;        /* default 10 */
    uint32_t M_max_spatial;         /* default 8 */
    uint32_t boiling_suppression;   /* default 1 */
    uint32_t sort_temporal;         /* default 1 */
    uint32_t sort_spatial;          /* default 1 */
    float alpha_min;                /* default 0.175^2 */
} zr_indirect_params;
typedef enum zr_indirect_output
{
    ZR_INDIRECT_FINAL = 0, ZR_INDIRECT_RESERVOIR_CURR, ZR_INDIRECT_RESERVOIR_PREV, ZR_INDIRECT_TARGET,
    ZR_INDIRECT_NEIGHBOR, ZR_INDIRECT_THREADMAP_NTC = 6
} zr_indirect_output;
ZR_API zr_status zr_indirect_pass_create(uint32_t width, uint32_t height, zr_indirect_pass** out);
ZR_API zr_status zr_indirect_pass_resize(zr_indirect_pass* p, uint32_t width, uint32_t height);
ZR_API zr_status zr_indirect_pass_reset_temporal(zr_indirect_pass* p);
ZR_API zr_status zr_indirect_pass_default_params(zr_indirect_params* out);
ZR_API zr_status zr_indirect_pass_set_params(zr_indirect_pass* p, const zr_indirect_params* params);
ZR_API zr_status zr_indirect_pass_render(zr_indirect_pass* p, const zr_frame_inputs* in, void* stream);
ZR_API zr_status zr_indirect_pass_get_output(zr_indirect_pass* p, zr_indirect_output id, zr_image2d* out);
ZR_API zr_status zr_indirect_pass_describe_io(zr_indirect_pass* p, zr_resource_use* uses, int* n);
/* multi-GPU: rows [y0, y1) this rank owns; halo rows are read from the (all-gathered) planes */
ZR_API zr_status zr_indirect_pass_set_rows(zr_indirect_pass* p, uint32_t y0, uint32_t y1);
ZR_API zr_status zr_indirect_pass_set_halo_exchange(zr_indirect_pass* p, zr_halo_exchange_fn fn, void* user);
ZR_API zr_status zr_indirect_pass_set_cost_map(zr_indirect_pass* p, void* d_cycles);
ZR_API zr_status zr_indirect_pass_set_schedule_costs(zr_indirect_pass* p, const double* h_tile_cost, uint32_t tiles_x, uint32_t tiles_y);
ZR_API void zr_indirect_pass_destroy(zr_indirect_pass* p);
/* ReSTIR PT debug views (RPT_DEBUG_VIEW, IndirectLighting_Common.h:58-67, same order; IndirectLighting::DebugViewCallback,
 * IndirectLighting.cpp:1233, 1543-1549). A view other than NONE replaces the indirect output (ZR_INDIRECT_FINAL) by
 * RPT_Util::DebugColor (ReSTIR_PT/Util.hlsli:69-139) of the reconnection in the reservoir that produces it: the reconnection vertex's
 * index k, its case, whether there is one, the BSDF lobe before or after x_k. The colour is written where the reference writes it --
 * the path-trace output with temporal reuse off (ReSTIR_PT_PathTrace.hlsl:540-556), temporal reuse's output without spatial reuse
 * (Reconnect_TtC.hlsl:386-388), else each spatial pass's output (Reconnect_StC.hlsl:348-351) -- and every other output write of those
 * stages is black while a view is on (Util.hlsli:141-160): no reusable neighbour, no temporal history, a history without a
 * reconnection. An empty reconnection is black, and so is case 3 in CONNECTION_LOBE_K. Accumulation, invalid and emissive pixels
 * behave as without a view, and reservoirs, target, neighbour and thread-map planes are the same bytes with and without one. Debug
 * frames launch one more kernel per write stage and hold 80 bytes per pixel more (freed when the view returns to NONE). Default
 * NONE; the view survives resize and reset_temporal. A view > CONNECTION_LOBE_K or a NULL pass is ZR_ERR_INVALID_ARG. */
typedef enum zr_rpt_debug_view
{
    ZR_RPT_DEBUG_VIEW_NONE = 0, ZR_RPT_DEBUG_VIEW_K, ZR_RPT_DEBUG_VIEW_CASE, ZR_RPT_DEBUG_VIEW_FOUND_CONNECTION,
    ZR_RPT_DEBUG_VIEW_CONNECTION_LOBE_K_MIN_1, ZR_RPT_DEBUG_VIEW_CONNECTION_LOBE_K
} zr_rpt_debug_view;
ZR_API zr_status zr_indirect_pass_set_debug_view(zr_indirect_pass* p, uint32_t view);

/* ---- IndirectLighting, INTEGRATOR::ReSTIR_GI (IndirectLighting.cpp:277-368; ReSTIR_GI shaders) ----
 * One kernel per frame: a path-traced initial candidate (second path vertex + outgoing radiance), temporal reuse with one
 * or two reprojected candidates and the reconnection Jacobian, wave-level outlier suppression. Emissive NEE only
 * (alias table, presampled sets, or the light voxel grid when it is enabled on the scene); the sun/sky variant is not
 * part of this build. */
typedef struct zr_rgi_reservoir        /* RGI_Util::Reservoir planes A/B/C (ReSTIR_GI/Reservoir.hlsli:88-131) in one 48-byte record */
{
    float pos[3]; uint32_t ID;          /* A: RGBA32F {pos, asfloat(ID)} */
    uint32_t Lo_rg, Lo_b_M;             /* B: RGBA16F {Lo, M} */
    float w_sum, W;                     /* C.xy */
    uint32_t normal;                    /* C.z: octahedral 2 x UNORM16 */
    uint32_t pad[3];
} zr_rgi_reservoir;
typedef struct zr_gi_params            /* cb_ReSTIR_GI fields the UI drives (IndirectLighting_Common.h:79-102, IndirectLighting.h:231-244) */
{
    uint32_t max_non_tr_bounces;        /* 3 */
    uint32_t max_glossy_tr_bounces;     /* 4 */
    uint32_t russian_roulette;          /* 1 */
    uint32_t stochastic_multi_bounce;   /* 1 */
    uint32_t boiling_suppression;       /* 1 */
    uint32_t M_max;                     /* 10 */
    uint32_t temporal_resample;         /* 1 */
} zr_gi_params;
typedef struct zr_gi_pass zr_gi_pass;
typedef enum zr_gi_output { ZR_GI_FINAL = 0, ZR_GI_RESERVOIR_CURR = 1, ZR_GI_RESERVOIR_PREV = 2 } zr_gi_output;
ZR_API zr_status zr_gi_pass_create(uint32_t width, uint32_t height, zr_gi_pass** out);
ZR_API zr_status zr_gi_pass_resize(zr_gi_pass* p, uint32_t width, uint32_t height);
ZR_API zr_status zr_gi_pass_reset_temporal(zr_gi_pass* p);
ZR_API zr_status zr_gi_pass_default_params(zr_gi_params* out);
ZR_API zr_status zr_gi_pass_set_params(zr_gi_pass* p, const zr_gi_params* params);
/* The integrators of IndirectLighting.h's INTEGRATOR enum. PATH_TRACING (IndirectLighting/PathTracer/PathTracer.hlsl: MIS next-event
 * estimation at every bounce, exact shadow rays, Beer's law in translucent media, no reuse -- the in-repo ground truth) and
 * ReSTIR GI run on this pass object (both read cb_ReSTIR_GI in the reference); ReSTIR PT is zr_indirect_pass. */
typedef enum zr_integrator { ZR_INTEGRATOR_PATH_TRACING = 0, ZR_INTEGRATOR_RESTIR_GI = 1, ZR_INTEGRATOR_RESTIR_PT = 2 } zr_integrator;
ZR_API zr_status zr_gi_pass_set_method(zr_gi_pass* p, zr_integrator method);     /* default RESTIR_GI; a change drops the history */
/* multi-GPU: rows [y0, y1) this rank owns; the hook runs once per frame on the reservoirs just written (next frame's temporal
 * candidates, searched up to 16 px around the reprojected pixel) */
ZR_API zr_status zr_gi_pass_set_rows(zr_gi_pass* p, uint32_t y0, uint32_t y1);
ZR_API zr_status zr_gi_pass_set_halo_exchange(zr_gi_pass* p, zr_halo_exchange_fn fn, void* user);
ZR_API zr_status zr_gi_pass_render(zr_gi_pass* p, const zr_frame_inputs* in, void* stream);
ZR_API zr_status zr_gi_pass_get_output(zr_gi_pass* p, zr_gi_output id, zr_image2d* out);
ZR_API void zr_gi_pass_destroy(zr_gi_pass* p);

/* ---- Sky (Sky/Sky.h, Sky.cpp:120-147): the sky-view LUT (Sky/SkyViewLUT.hlsl) ----
 * create(lut_w, lut_h): a lut_w x lut_h LUT (the renderer's is 256 x 128, DefaultRendererImpl.h:165-166). render reads only
 * in->frame: the sun (SunDir, SunIlluminance) and the atmosphere (PlanetRadius, AtmosphereAltitude, Rayleigh / Mie / ozone
 * coefficients, g), and refuses non-finite values or a PlanetRadius or AtmosphereAltitude <= 0. Each texel is the sun's light
 * scattered once towards a viewer 0.2 km above the ground (Volumetric.hlsli EstimateLs, 32 steps; 8 towards the sun), at
 * longitude 2 pi x / lut_w and latitude pi/2 +- 2 pi (y / lut_h - 1/2)^2. get_output (GetOutput(SKY_VIEW_LUT)): R11G11B10F texels
 * as uint32, pitch = 4 * lut_w. No sizes beyond the create; inscattering is not part of this pass. */
typedef struct zr_sky_pass zr_sky_pass;
ZR_API zr_status zr_sky_pass_create(uint32_t lut_w, uint32_t lut_h, zr_sky_pass** out);
ZR_API zr_status zr_sky_pass_render(zr_sky_pass* p, const zr_frame_inputs* in, void* stream);
ZR_API zr_status zr_sky_pass_get_output(zr_sky_pass* p, zr_image2d* out);
ZR_API zr_status zr_sky_pass_describe_io(zr_sky_pass* p, zr_resource_use* uses, int* n);
ZR_API void zr_sky_pass_destroy(zr_sky_pass* p);

/* ---- Compositing + FireflyFilter (Compositing/Compositing.cpp:83-145) ---- */
typedef struct zr_compositing_pass zr_compositing_pass;
typedef struct zr_compositing_params { uint32_t emissive_di; uint32_t indirect; uint32_t firefly_filter; } zr_compositing_params;
ZR_API zr_status zr_compositing_pass_create(uint32_t width, uint32_t height, zr_compositing_pass** out);
ZR_API zr_status zr_compositing_pass_resize(zr_compositing_pass* p, uint32_t width, uint32_t height);
ZR_API zr_status zr_compositing_pass_set_params(zr_compositing_pass* p, const zr_compositing_params* params);
/* d_direct / d_indirect: float4[w*h] (outputs of the lighting passes) or NULL */
ZR_API zr_status zr_compositing_pass_render(zr_compositing_pass* p, const zr_frame_inputs* in,
    const void* d_direct, const void* d_indirect, void* stream);
ZR_API zr_status zr_compositing_pass_set_rows(zr_compositing_pass* p, uint32_t y0, uint32_t y1);
ZR_API zr_status zr_compositing_pass_get_output(zr_compositing_pass* p, zr_image2d* out);
/* The sky behind geometry in frames that do not accumulate (Compositing.hlsl:43-47): with a LUT set, pixels without geometry show
 * Light::Le_SkyWithSunDisk (LightSource.hlsli:178-199) when emissive_di is on and 0 when it is off; NULL returns to 0 everywhere.
 * Accumulating frames take the sky from DirectLighting's output (zr_direct_pass_set_sky). Refuses what zr_direct_pass_set_sky
 * refuses; the pass does not own the LUT. */
ZR_API zr_status zr_compositing_pass_set_sky(zr_compositing_pass* p, const zr_image2d* lut);
ZR_API void zr_compositing_pass_destroy(zr_compositing_pass* p);

/* ------------------------------------------------------------------------------------------
 * SVGF denoiser (no reference counterpart: ZetaRay ships none; BASELINE.json north_star / config 3).
 * Temporal accumulation of colour + luminance moments -> variance, then `num_passes` a-trous wavelet passes (step 1, 2, 4, ...)
 * with depth / normal / variance-guided luminance edge stops; the algorithm is defined by oracle/orc_svgf.cpp.
 * d_signal: RGBA32F image (the Compositing output); output: RGBA32F, alpha = filtered variance. Slots between Compositing and TAA.
 * ------------------------------------------------------------------------------------------ */
typedef struct zr_svgf_pass zr_svgf_pass;
typedef struct zr_svgf_params
{
    float sigma_z;          /* relative depth tolerance per unit step (0.02) */
    float k_n;              /* normal falloff: weight = max(0, 1 - k_n (1 - n.n')) (16) */
    float sigma_l;          /* luminance tolerance in standard deviations (4) */
    uint32_t radius;        /* 2 = 5x5 B3-spline taps, 1 = 3x3 binomial taps */
    uint32_t num_passes;    /* 1..5 */
} zr_svgf_params;
typedef enum zr_svgf_output
{
    ZR_SVGF_DENOISED = 0,       /* RGBA32F, pitch = width */
    ZR_SVGF_ACCUMULATED = 1,    /* 4 x half {rgb, variance} after the temporal stage (overwritten by the second a-trous pass) */
    ZR_SVGF_GUIDE = 2,          /* {f32 view depth, oct32 normal} */
    ZR_SVGF_HISTORY = 3         /* {half4 colour | half m1, m2, N, 0}: next frame's history */
} zr_svgf_output;
ZR_API zr_status zr_svgf_pass_create(uint32_t width, uint32_t height, zr_svgf_pass** out);
ZR_API zr_status zr_svgf_pass_resize(zr_svgf_pass* p, uint32_t width, uint32_t height);
ZR_API zr_status zr_svgf_pass_reset_temporal(zr_svgf_pass* p);
ZR_API zr_status zr_svgf_pass_default_params(zr_svgf_params* out);
ZR_API zr_status zr_svgf_pass_set_params(zr_svgf_pass* p, const zr_svgf_params* params);
/* multi-GPU: rows [y0, y1) this rank owns. The hook runs num_passes + 1 times per render: after the temporal stage on colour +
 * variance, guide and history (the first a-trous pass reads colour + variance `radius` rows beyond the strip, every pass reads the
 * guide up to 32 rows beyond, next frame's reprojection reads guide and history), after every a-trous pass k but the last on the
 * colour + variance plane it wrote (pass k + 1 reads it radius * 2^(k+1) <= 32 rows beyond), and after the last one on the denoised
 * output (TAA reads it one row beyond). The internal planes it receives are padded: pitch_bytes >= width * texel_bytes. */
ZR_API zr_status zr_svgf_pass_set_rows(zr_svgf_pass* p, uint32_t y0, uint32_t y1);
ZR_API zr_status zr_svgf_pass_set_halo_exchange(zr_svgf_pass* p, zr_halo_exchange_fn fn, void* user);
ZR_API zr_status zr_svgf_pass_render(zr_svgf_pass* p, const zr_frame_inputs* in, const void* d_signal, void* stream);
ZR_API zr_status zr_svgf_pass_get_output(zr_svgf_pass* p, zr_svgf_output id, zr_image2d* out);     /* internal planes: pitch_bytes > width * texel */
ZR_API void zr_svgf_pass_destroy(zr_svgf_pass* p);

/* ---- TAA (TAA/TAA.cpp:87-123) ---- */
typedef struct zr_taa_pass zr_taa_pass;
ZR_API zr_status zr_taa_pass_create(uint32_t width, uint32_t height, zr_taa_pass** out);
ZR_API zr_status zr_taa_pass_resize(zr_taa_pass* p, uint32_t width, uint32_t height);
ZR_API zr_status zr_taa_pass_set_rows(zr_taa_pass* p, uint32_t y0, uint32_t y1);
ZR_API zr_status zr_taa_pass_set_blend_weight(zr_taa_pass* p, float w);  /* default 0.1, TAA.h:72 */
/* d_signal: float4[w*h]; output RGBA16F (half4, 8 B/px) */
ZR_API zr_status zr_taa_pass_render(zr_taa_pass* p, const zr_frame_inputs* in, const void* d_signal, void* stream);
ZR_API zr_status zr_taa_pass_get_output(zr_taa_pass* p, zr_image2d* out);
ZR_API void zr_taa_pass_destroy(zr_taa_pass* p);

/* ---- AutoExposure (AutoExposure/AutoExposure.h, AutoExposure.cpp:100-140) ----
 * A 256-bin luminance histogram of the signal TAA reads (k_lum_histogram, rows set by set_rows), then one block turns it into
 * a temporally adapted exposure (k_exposure): output {exposure, adapted luminance} as one float2, {0, 0} after create / resize /
 * reset (the reference's INIT_TO_ZERO texture). Adaptation reads the frame's dt in seconds: render rejects a non-finite or
 * negative dt, and dt == 0 on the first frame after create / resize / reset (the exposure would be infinite); later frames with
 * dt == 0 keep the adapted luminance. */
typedef struct zr_auto_exposure_pass zr_auto_exposure_pass;
typedef struct zr_auto_exposure_params
{
    float min_lum;          /* 5e-3, AutoExposure.h:73-80; >= 0 */
    float max_lum;          /* 4; > min_lum */
    float lum_map_exp;      /* 0.5; > 0 */
    float adaptation_rate;  /* 1 */
} zr_auto_exposure_params;
/* Called between the histogram and the exposure kernel on the 256 device bins: it must leave there the sum of every rank's bins
 * (strip-sharded frames: every rank then derives the same exposure). The renderer's hook is zr_comm_allreduce_u32. */
typedef void (*zr_reduce_u32_fn)(void* user, uint32_t* d_values, uint32_t n, void* stream);
ZR_API zr_status zr_auto_exposure_pass_create(uint32_t width, uint32_t height, zr_auto_exposure_pass** out);
ZR_API zr_status zr_auto_exposure_pass_resize(zr_auto_exposure_pass* p, uint32_t width, uint32_t height);
ZR_API zr_status zr_auto_exposure_pass_reset_temporal(zr_auto_exposure_pass* p);
ZR_API zr_status zr_auto_exposure_pass_default_params(zr_auto_exposure_params* out);
ZR_API zr_status zr_auto_exposure_pass_set_params(zr_auto_exposure_pass* p, const zr_auto_exposure_params* params);
/* d_signal: float4[w*h], the image TAA reads (Compositing or SVGF output) */
ZR_API zr_status zr_auto_exposure_pass_render(zr_auto_exposure_pass* p, const zr_frame_inputs* in, const void* d_signal, void* stream);
ZR_API zr_status zr_auto_exposure_pass_set_rows(zr_auto_exposure_pass* p, uint32_t y0, uint32_t y1);
ZR_API zr_status zr_auto_exposure_pass_set_reduce(zr_auto_exposure_pass* p, zr_reduce_u32_fn fn, void* user);   /* fn NULL: none */
ZR_API zr_status zr_auto_exposure_pass_get_output(zr_auto_exposure_pass* p, zr_image2d* out);     /* 1 x 1 float2 */
ZR_API void zr_auto_exposure_pass_destroy(zr_auto_exposure_pass* p);

/* ---- Display (Display/Display.h, Display.hlsl default view, Tonemap.hlsli) ----
 * TAA output x exposure -> tone mapper -> saturate -> sRGB OETF -> RGBA8 (alpha 255), the reference's R8G8B8A8_UNORM_SRGB back
 * buffer. Render size must equal display size. NEUTRAL is Tony McMapface: the caller supplies its 48^3 LUT in the packed
 * R9G9B9E5_SHAREDEXP form (x fastest, as tony_mc_mapface.dds stores it) with set_lut; rendering NEUTRAL without it is
 * ZR_ERR_INVALID_ARG. */
typedef enum zr_tonemapper
{
    ZR_TONEMAPPER_NONE = 0, ZR_TONEMAPPER_NEUTRAL = 1, ZR_TONEMAPPER_AGX_DEFAULT = 2, ZR_TONEMAPPER_AGX_GOLDEN = 3,
    ZR_TONEMAPPER_AGX_PUNCHY = 4, ZR_TONEMAPPER_AGX_CUSTOM = 5
} zr_tonemapper;
typedef struct zr_display_params
{
    uint32_t tonemapper;    /* zr_tonemapper, default NEUTRAL (Display.cpp:70-74) */
    uint32_t auto_exposure; /* 1: multiply by the exposure first */
    float saturation;       /* 1: NEUTRAL's desaturation lerp and AGX_CUSTOM */
    float agx_exp;          /* 1: AGX_CUSTOM's exponent */
} zr_display_params;
typedef struct zr_display_pass zr_display_pass;
ZR_API zr_status zr_display_pass_create(uint32_t width, uint32_t height, zr_display_pass** out);
ZR_API zr_status zr_display_pass_resize(zr_display_pass* p, uint32_t width, uint32_t height);
ZR_API zr_status zr_display_pass_default_params(zr_display_params* out);
ZR_API zr_status zr_display_pass_set_params(zr_display_pass* p, const zr_display_params* params);
ZR_API zr_status zr_display_pass_set_lut(zr_display_pass* p, const uint32_t* h_rgb9e5, uint32_t dim);     /* dim must be 48 */
/* d_signal: the TAA output (half4[w*h]); d_exposure: the auto-exposure output (float2), may be NULL with auto_exposure off */
ZR_API zr_status zr_display_pass_render(zr_display_pass* p, const zr_frame_inputs* in, const void* d_signal, const void* d_exposure,
    void* stream);
ZR_API zr_status zr_display_pass_set_rows(zr_display_pass* p, uint32_t y0, uint32_t y1);
ZR_API zr_status zr_display_pass_get_output(zr_display_pass* p, zr_image2d* out);      /* RGBA8, 4 B/px */
ZR_API void zr_display_pass_destroy(zr_display_pass* p);
/* Debug views (DisplayOption, Display_Common.h:6-19, same order; Display.hlsl:53-170). A view other than DEFAULT shows one
 * channel of the current G-buffer in place of the tone-mapped signal: render then reads no signal, exposure or LUT (d_signal and
 * d_exposure may be NULL) and writes (0, 0, 0, 0) where the primary ray missed. ROUGHNESS_TH marks roughness >= roughness_th.
 * Default DEFAULT, 1.0 (Display.cpp:73); a view > DEPTH or a non-finite threshold is ZR_ERR_INVALID_ARG. */
typedef enum zr_display_view
{
    ZR_DISPLAY_VIEW_DEFAULT = 0, ZR_DISPLAY_VIEW_BASE_COLOR, ZR_DISPLAY_VIEW_NORMAL, ZR_DISPLAY_VIEW_METALNESS_ROUGHNESS,
    ZR_DISPLAY_VIEW_COAT_WEIGHT, ZR_DISPLAY_VIEW_COAT_COLOR, ZR_DISPLAY_VIEW_ROUGHNESS_TH, ZR_DISPLAY_VIEW_EMISSIVE,
    ZR_DISPLAY_VIEW_TRANSMISSION, ZR_DISPLAY_VIEW_DEPTH
} zr_display_view;
ZR_API zr_status zr_display_pass_set_view(zr_display_pass* p, uint32_t view, float roughness_th);
/* Outline of picked instances (SetPickedInstance / GetPickedInstances; Display.cpp:293-400, DrawPicked.hlsl, Sobel.hlsl). Each
 * frame with picks, render rasterises picked instance k into bit k of a mask (placed by its TRS, clipped at CameraNear, no culling
 * and no depth test) and draws the mask's Sobel outline over the image. h_instances holds instance indices as in
 * zr_gbuffer_pass_pick; n == 0 clears the picks. More than ZR_DISPLAY_MAX_PICKED, or NULL with n > 0, is ZR_ERR_INVALID_ARG; render
 * refuses, before it launches anything, an index that is not in the frame's scene. Picks and the view survive a resize. */
#define ZR_DISPLAY_MAX_PICKED 32u
ZR_API zr_status zr_display_pass_set_picked(zr_display_pass* p, const uint32_t* h_instances, uint32_t n);

/* ---- host <-> device helpers so callers need no CUDA runtime of their own ---- */
ZR_API zr_status zr_device_malloc(void** d_ptr, size_t bytes);
ZR_API void zr_device_free(void* d_ptr);
ZR_API zr_status zr_memcpy_h2d(void* d_dst, const void* h_src, size_t bytes, void* stream);
ZR_API zr_status zr_memcpy_d2h(void* h_dst, const void* d_src, size_t bytes, void* stream);
ZR_API zr_status zr_memset_d(void* d_dst, int value, size_t bytes, void* stream);
ZR_API zr_status zr_stream_synchronize(void* stream);
/* per-kernel device timing for the roofline report: while enabled every launch is bracketed by CUDA events on
 * its stream; collect() synchronises and returns "name:calls:total_ms;..." */
ZR_API zr_status zr_profile_enable(int on);
ZR_API zr_status zr_profile_collect(char* buf, size_t buf_size);
/* number of kernels this library launched since load (for bench.py's gpu_launches) */
ZR_API uint64_t zr_kernel_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Strip-sharded frames across GPUs (SURVEY 8e; the reference is single-GPU). One process per GPU; zr_comm carries the halo bands
 * between neighbouring strips with grouped NCCL send / recv issued from C++ on the producing stream (csrc/comm.cu).
 * Rank 0 calls zr_comm_unique_id and distributes the 256 bytes (any out-of-band channel: torch.distributed broadcast, MPI, a file);
 * every rank then calls zr_comm_create with the same bytes. A host without NCCL creates its zr_comm from its own transport instead
 * (zr_comm_create_transport); either kind drives zr_renderer_set_shard.
 * ------------------------------------------------------------------------------------------ */
typedef struct zr_comm zr_comm;
ZR_API zr_status zr_comm_unique_id(void* out256);
ZR_API zr_status zr_comm_create(const void* id256, int rank, int world, zr_comm** out);
/* A caller-supplied transport: each callback has the contract of the zr_comm_* entry point of the same name (arguments already
 * checked, world > 1) and returns ZR_OK or an error, which zr_renderer_render then returns. The callbacks run on the calling thread,
 * inside zr_renderer_render or a pass's render, and must leave the bands in place in stream order. The struct is copied; dlopen is
 * never involved. */
typedef struct zr_comm_transport {
    zr_status (*exchange_halos)(void* user, int which_comm, const uint32_t* bounds, uint32_t halo_rows,
                                const zr_image2d* planes, int n_planes, void* stream);
    zr_status (*gather_rows)(void* user, const uint32_t* bounds, const zr_image2d* plane, int root, void* stream);
    zr_status (*allreduce_u32)(void* user, int which_comm, uint32_t* d_values, uint32_t n, void* stream);
} zr_comm_transport;
ZR_API zr_status zr_comm_create_transport(const zr_comm_transport* t, void* user, int rank, int world, zr_comm** out);
ZR_API void zr_comm_destroy(zr_comm* c);
ZR_API zr_status zr_comm_rank(zr_comm* c, int* rank, int* world);
ZR_API zr_status zr_comm_stats(zr_comm* c, uint64_t* bytes_sent, uint64_t* calls);
/* bounds[world + 1]: strip q owns rows [bounds[q], bounds[q + 1]); which_comm: 0 = main stream, 1 = second stream */
ZR_API zr_status zr_comm_exchange_halos(zr_comm* c, int which_comm, const uint32_t* bounds, uint32_t halo_rows, const zr_image2d* planes,
    int n_planes, void* stream);
ZR_API zr_status zr_comm_gather_rows(zr_comm* c, const uint32_t* bounds, const zr_image2d* plane, int root, void* stream);
/* In-place sum of n uint32 values over every rank (one ncclAllReduce on which_comm) */
ZR_API zr_status zr_comm_allreduce_u32(zr_comm* c, int which_comm, uint32_t* d_values, uint32_t n, void* stream);

/* ---- The frame (ZetaRenderer/Default: DefaultRenderer.cpp:304-520, PathTracer.cpp:149-563) ----
 * Owns the double-buffered G-buffers and one object of every pass and runs a frame in the reference's order:
 * (frame 1: emissive power + alias table) -> presampling if enabled -> GBufferRT -> DirectLighting || IndirectLighting
 * -> Compositing + firefly filter -> TAA. When two_streams != 0, GBufferRT and IndirectLighting run on an internal stream of the
 * greatest priority and DirectLighting on an internal second stream of the least (the two lighting passes are independent
 * render-graph nodes in the reference); both join the caller's stream before Compositing. Parameters are set on the pass handles. */
typedef struct zr_renderer zr_renderer;
typedef struct zr_renderer_desc { uint32_t width, height; int with_tridiff; int two_streams; } zr_renderer_desc;
ZR_API zr_status zr_renderer_create(const zr_renderer_desc* desc, zr_scene* scene, zr_renderer** out);
ZR_API zr_status zr_renderer_render(zr_renderer* r, const zr_frame_constants* frame, void* stream);
/* optional SVGF stage between Compositing and TAA (BASELINE config 3); *out_pass (may be NULL) receives the pass for set_params */
ZR_API zr_status zr_renderer_set_denoiser(zr_renderer* r, int enable, zr_svgf_pass** out_pass);
/* Strip-sharded frame: this renderer computes rows [bounds[rank], bounds[rank + 1]) only (bounds: multiples of 32 except the last;
 * any integrator, with or without the SVGF stage); halo bands move through `comm` at the exchange points of a frame (ReSTIR PT: four,
 * ReSTIR GI: three, path tracer: two; the SVGF stage adds num_passes + 1), the finished image is gathered on rank 0
 * (gather_output != 0). A denoiser enabled later follows the current strip. comm == NULL returns to the whole frame. History must be
 * complete when the cut happens: render the warm-up frames unsharded on every rank. */
ZR_API zr_status zr_renderer_set_shard(zr_renderer* r, zr_comm* comm, const uint32_t* bounds, int gather_output);
ZR_API zr_status zr_renderer_get_output(zr_renderer* r, zr_image2d* out);      /* TAA output, RGBA16F */
/* Optional post-processing (ZetaRenderer/Default/PostProcessor.cpp): enable != 0 creates an AutoExposure pass that reads the TAA
 * input and a Display pass on the TAA output (their defaults; NEUTRAL needs zr_display_pass_set_lut on *out_display before the
 * next frame); 0 removes both. Sharded frames histogram each strip and all-reduce the bins on the main communicator, and
 * gather the display image on rank 0 along with the TAA image. out_ae / out_display may be NULL. */
ZR_API zr_status zr_renderer_set_display(zr_renderer* r, int enable, zr_auto_exposure_pass** out_ae, zr_display_pass** out_display);
ZR_API zr_status zr_renderer_get_display_output(zr_renderer* r, zr_image2d* out);      /* RGBA8; ZR_ERR_NOT_INITIALIZED when disabled */
/* The sky (Sky::Render, PathTracer.cpp:165-185, 343-362): enable != 0 creates a 256 x 128 sky pass whose LUT every frame recomputes
 * on DirectLighting's stream before DirectLighting, and hands that LUT to zr_direct_pass_set_sky and zr_compositing_pass_set_sky, so
 * pixels without geometry show the sky and the sun disk. Strip-sharded, every rank computes the whole LUT. 0 detaches the LUT and
 * frees the pass and the DirectLighting copy it needed; frames are then those of a renderer that never enabled it. *out_pass (may
 * be NULL) is the pass, or NULL when the sky is off. Off by default. */
ZR_API zr_status zr_renderer_set_sky(zr_renderer* r, int enable, zr_sky_pass** out_pass);
ZR_API zr_status zr_renderer_get_passes(zr_renderer* r, zr_gbuffer_pass** gbuffer, zr_direct_pass** direct,
    zr_indirect_pass** indirect, zr_compositing_pass** compositing, zr_taa_pass** taa);
ZR_API zr_status zr_renderer_get_gbuffer(zr_renderer* r, int previous, zr_gbuffer* out);
/* IndirectLighting::SetMethod(INTEGRATOR) as DefaultRenderer.cpp:243 calls it; values follow IndirectLighting.h's enum
 * (zr_integrator, declared with the GI pass above). PATH_TRACING and ReSTIR GI share one pass object, created on first use. */
ZR_API zr_status zr_renderer_set_integrator(zr_renderer* r, zr_integrator method);
ZR_API zr_status zr_renderer_get_gi_pass(zr_renderer* r, zr_gi_pass** gi);
/* RenderSettings::LightPresampling / UseLVG as DefaultRenderer::Update derives them from the scene
 * (DefaultRenderer.cpp:361-363, 439-478; DefaultRendererImpl.h:37-43): presampled sets 128 x 512 iff the scene has
 * >= 13107 emissive triangles, the 32 x 8 x 40 light voxel grid only if requested AND presampling is on.
 * out_applied (may be NULL) = {presampling, lvg} as decided. */
ZR_API zr_status zr_renderer_apply_scene_settings(zr_renderer* r, int use_lvg, uint32_t out_applied[2]);
ZR_API void zr_renderer_destroy(zr_renderer* r);

#ifdef __cplusplus
}
#endif

#endif /* ZR_ABI_H */
