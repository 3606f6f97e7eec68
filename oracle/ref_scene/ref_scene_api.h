/* ref_scene_api.h -- the entry points of oracle/_ref/libref_scene.so (ref_scene_wrap.cpp around the reference's scene-data
 * constructors and layouts). Plain C types only: tests/orc.py binds each function's ctypes types from these prototypes, and the
 * wrapper includes this header, so a definition whose types differ from its declaration does not compile. */
#ifndef REF_SCENE_API_H
#define REF_SCENE_API_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define REF_API __attribute__((visibility("default")))

/* out: sizeof Material, RT::MeshInstance, RT::EmissiveTriangle, Core::Vertex; returns 4 */
REF_API int ref_scene_sizes(int* out);
REF_API void ref_material(const float* p, uint32_t flags, void* out32);
REF_API void ref_emissive_triangle(const float* v, const float* uv, uint32_t factorRGB8, uint32_t tex, uint16_t strengthHalfBits,
    uint32_t triIdx, int doubleSided, void* out48);
REF_API uint32_t ref_oct32(float x, float y, float z);
REF_API void ref_oct32_decode(uint32_t enc, float* out3);
REF_API uint16_t ref_half(float f);
REF_API uint32_t ref_rgb8(float r, float g, float b);
REF_API void ref_instance_rotation_scale(const float* q4, const float* s3, uint16_t* outRot4, uint16_t* outScale3);
/* byte offset of a field of cbFrameConstants, -1 if unknown; "" -> sizeof */
REF_API int ref_frame_constants_offset(const char* field);
REF_API int ref_struct_offset(const char* strct, const char* field);

#ifdef __cplusplus
}
#endif

#endif
