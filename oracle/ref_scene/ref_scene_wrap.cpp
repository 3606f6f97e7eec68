// TEST INFRASTRUCTURE. C entry points around the REFERENCE's own scene-data constructors, compiled from the reference tree where it
// lies (oracle/ref_scene/build.sh -> oracle/_ref/libref_scene.so). They pin this repository's scene-ingest packers
// (zetaray_b200/scene.py) -- the flat-buffer formats on the caller's side of the drop-in boundary (SURVEY A.6 / A.8):
//   ZetaCore/Core/Material.h           Material ctor + setters (32 B)
//   ZetaCore/RayTracing/RtCommon.h     RT::EmissiveTriangle ctor / StoreVertices (48 B), RT::MeshInstance field types
//   ZetaCore/Math/OctahedralVector.h   oct32
//   ZetaCore/Math/Vector.h             half, half3, unorm4
//   ZetaCore/Math/Color.h              Float3ToRGB8
//   ZetaRenderPass/Common/FrameConstants.h   cbFrameConstants (field offsets: the per-frame constant block the passes receive)
//   the RT::MeshInstance / EmissiveTriangle / Material field offsets
// Nothing here is product code and no reference source is copied.
#include "ref_scene_api.h"
#include "ZetaCore/RayTracing/RtCommon.h"
#include "ZetaCore/Core/Vertex.h"
#include "ZetaRenderPass/Common/FrameConstants.h"
#include <cstddef>
#include <cstring>

using namespace ZetaRay;
using namespace ZetaRay::Math;

extern "C"
{
    int ref_scene_sizes(int* out)
    {
        out[0] = (int)sizeof(Material); out[1] = (int)sizeof(RT::MeshInstance); out[2] = (int)sizeof(RT::EmissiveTriangle);
        out[3] = (int)sizeof(Core::Vertex);
        return 4;
    }

    // p: base rgba, metallic, roughness, ior, transmission, emissive rgb, emissive strength, coat weight, coat rgb, coat roughness,
    //    coat ior, subsurface, transmission depth (19 floats); flags: bit0 double sided, bit1 thin walled
    void ref_material(const float* p, uint32_t flags, void* out32)
    {
        Material m;
        m.SetBaseColorFactor(float4(p[0], p[1], p[2], p[3]));
        m.SetMetallic(p[4]);
        m.SetSpecularRoughness(p[5]);
        m.SetSpecularIOR(p[6]);
        m.SetTransmission(p[7]);
        m.SetEmissiveFactor(float3(p[8], p[9], p[10]));
        m.SetEmissiveStrength(p[11]);
        m.SetCoatWeight(p[12]);
        m.SetCoatColor(float3(p[13], p[14], p[15]));
        m.SetCoatRoughness(p[16]);
        m.SetCoatIOR(p[17]);
        m.SetSubsurface(p[18]);
        m.SetTransmissionDepth(p[19]);
        m.SetDoubleSided((flags & 1) != 0);
        m.SetThinWalled((flags & 2) != 0);
        memcpy(out32, &m, sizeof(m));
    }

    // v: 9 floats (three vertices), uv: 6 floats
    void ref_emissive_triangle(const float* v, const float* uv, uint32_t factorRGB8, uint32_t tex, uint16_t strengthHalfBits,
        uint32_t triIdx, int doubleSided, void* out48)
    {
        RT::EmissiveTriangle t(float3(v[0], v[1], v[2]), float3(v[3], v[4], v[5]), float3(v[6], v[7], v[8]),
            float2(uv[0], uv[1]), float2(uv[2], uv[3]), float2(uv[4], uv[5]), factorRGB8, tex, half::asfloat16(strengthHalfBits),
            triIdx, doubleSided != 0);
        memcpy(out48, &t, sizeof(t));
    }

    uint32_t ref_oct32(float x, float y, float z)
    {
        oct32 o(x, y, z);
        uint32_t r;
        memcpy(&r, &o.v, 4);
        return r;
    }
    void ref_oct32_decode(uint32_t enc, float* out3)
    {
        oct32 o;
        memcpy(&o.v, &enc, 4);
        float3 d = o.decode();
        out3[0] = d.x; out3[1] = d.y; out3[2] = d.z;
    }
    uint16_t ref_half(float f) { return half(f).x; }
    uint32_t ref_rgb8(float r, float g, float b) { return Float3ToRGB8(float3(r, g, b)); }
    // quaternion (normalised floats in [-1, 1]) -> the unorm4 RT::MeshInstance::Rotation stores; scale -> half3
    void ref_instance_rotation_scale(const float* q4, const float* s3, uint16_t* outRot4, uint16_t* outScale3)
    {
        float4a q(q4[0], q4[1], q4[2], q4[3]);
        unorm4 u = unorm4::FromNormalized(q);       // RtAccelerationStructure.cpp:345 (maps [-1, 1] -> [0, 1] itself)
        memcpy(outRot4, &u, 8);
        half3 h(float3(s3[0], s3[1], s3[2]));
        memcpy(outScale3, &h, 6);
    }

    // byte offset of a field of cbFrameConstants (Common/FrameConstants.h), -1 if unknown; "" -> sizeof
    int ref_frame_constants_offset(const char* field)
    {
        if (!field[0]) return (int)sizeof(cbFrameConstants);
        if (!strcmp(field, "CurrView")) return (int)offsetof(cbFrameConstants, CurrView);
        if (!strcmp(field, "PrevView")) return (int)offsetof(cbFrameConstants, PrevView);
        if (!strcmp(field, "CurrViewInv")) return (int)offsetof(cbFrameConstants, CurrViewInv);
        if (!strcmp(field, "PrevViewInv")) return (int)offsetof(cbFrameConstants, PrevViewInv);
        if (!strcmp(field, "CurrViewProj")) return (int)offsetof(cbFrameConstants, CurrViewProj);
        if (!strcmp(field, "PrevViewProj")) return (int)offsetof(cbFrameConstants, PrevViewProj);
        if (!strcmp(field, "CameraPos")) return (int)offsetof(cbFrameConstants, CameraPos);
        if (!strcmp(field, "CameraNear")) return (int)offsetof(cbFrameConstants, CameraNear);
        if (!strcmp(field, "AspectRatio")) return (int)offsetof(cbFrameConstants, AspectRatio);
        if (!strcmp(field, "PixelSpreadAngle")) return (int)offsetof(cbFrameConstants, PixelSpreadAngle);
        if (!strcmp(field, "TanHalfFOV")) return (int)offsetof(cbFrameConstants, TanHalfFOV);
        if (!strcmp(field, "dt")) return (int)offsetof(cbFrameConstants, dt);
        if (!strcmp(field, "FrameNum")) return (int)offsetof(cbFrameConstants, FrameNum);
        if (!strcmp(field, "CurrGBufferDescHeapOffset")) return (int)offsetof(cbFrameConstants, CurrGBufferDescHeapOffset);
        if (!strcmp(field, "PrevGBufferDescHeapOffset")) return (int)offsetof(cbFrameConstants, PrevGBufferDescHeapOffset);
        if (!strcmp(field, "BaseColorMapsDescHeapOffset")) return (int)offsetof(cbFrameConstants, BaseColorMapsDescHeapOffset);
        if (!strcmp(field, "NormalMapsDescHeapOffset")) return (int)offsetof(cbFrameConstants, NormalMapsDescHeapOffset);
        if (!strcmp(field, "MetallicRoughnessMapsDescHeapOffset")) return (int)offsetof(cbFrameConstants, MetallicRoughnessMapsDescHeapOffset);
        if (!strcmp(field, "EmissiveMapsDescHeapOffset")) return (int)offsetof(cbFrameConstants, EmissiveMapsDescHeapOffset);
        if (!strcmp(field, "EnvMapDescHeapOffset")) return (int)offsetof(cbFrameConstants, EnvMapDescHeapOffset);
        if (!strcmp(field, "RenderWidth")) return (int)offsetof(cbFrameConstants, RenderWidth);
        if (!strcmp(field, "RenderHeight")) return (int)offsetof(cbFrameConstants, RenderHeight);
        if (!strcmp(field, "DisplayWidth")) return (int)offsetof(cbFrameConstants, DisplayWidth);
        if (!strcmp(field, "DisplayHeight")) return (int)offsetof(cbFrameConstants, DisplayHeight);
        if (!strcmp(field, "CurrCameraJitter")) return (int)offsetof(cbFrameConstants, CurrCameraJitter);
        if (!strcmp(field, "PrevCameraJitter")) return (int)offsetof(cbFrameConstants, PrevCameraJitter);
        if (!strcmp(field, "PlanetRadius")) return (int)offsetof(cbFrameConstants, PlanetRadius);
        if (!strcmp(field, "SunCosAngularRadius")) return (int)offsetof(cbFrameConstants, SunCosAngularRadius);
        if (!strcmp(field, "SunSinAngularRadius")) return (int)offsetof(cbFrameConstants, SunSinAngularRadius);
        if (!strcmp(field, "pad")) return (int)offsetof(cbFrameConstants, pad);
        if (!strcmp(field, "SunDir")) return (int)offsetof(cbFrameConstants, SunDir);
        if (!strcmp(field, "SunIlluminance")) return (int)offsetof(cbFrameConstants, SunIlluminance);
        if (!strcmp(field, "RayleighSigmaSColor")) return (int)offsetof(cbFrameConstants, RayleighSigmaSColor);
        if (!strcmp(field, "RayleighSigmaSScale")) return (int)offsetof(cbFrameConstants, RayleighSigmaSScale);
        if (!strcmp(field, "OzoneSigmaAColor")) return (int)offsetof(cbFrameConstants, OzoneSigmaAColor);
        if (!strcmp(field, "OzoneSigmaAScale")) return (int)offsetof(cbFrameConstants, OzoneSigmaAScale);
        if (!strcmp(field, "MieSigmaS")) return (int)offsetof(cbFrameConstants, MieSigmaS);
        if (!strcmp(field, "MieSigmaA")) return (int)offsetof(cbFrameConstants, MieSigmaA);
        if (!strcmp(field, "AtmosphereAltitude")) return (int)offsetof(cbFrameConstants, AtmosphereAltitude);
        if (!strcmp(field, "g")) return (int)offsetof(cbFrameConstants, g);
        if (!strcmp(field, "NumFramesCameraStatic")) return (int)offsetof(cbFrameConstants, NumFramesCameraStatic);
        if (!strcmp(field, "CameraStatic")) return (int)offsetof(cbFrameConstants, CameraStatic);
        if (!strcmp(field, "Accumulate")) return (int)offsetof(cbFrameConstants, Accumulate);
        if (!strcmp(field, "SunMoved")) return (int)offsetof(cbFrameConstants, SunMoved);
        if (!strcmp(field, "CameraRayUVGradsScale")) return (int)offsetof(cbFrameConstants, CameraRayUVGradsScale);
        if (!strcmp(field, "MipBias")) return (int)offsetof(cbFrameConstants, MipBias);
        if (!strcmp(field, "OneDivNumEmissiveTriangles")) return (int)offsetof(cbFrameConstants, OneDivNumEmissiveTriangles);
        if (!strcmp(field, "NumEmissiveTriangles")) return (int)offsetof(cbFrameConstants, NumEmissiveTriangles);
        if (!strcmp(field, "FocusDepth")) return (int)offsetof(cbFrameConstants, FocusDepth);
        if (!strcmp(field, "LensRadius")) return (int)offsetof(cbFrameConstants, LensRadius);
        if (!strcmp(field, "DoF")) return (int)offsetof(cbFrameConstants, DoF);
        if (!strcmp(field, "pad2")) return (int)offsetof(cbFrameConstants, pad2);
        return -1;
    }
    int ref_struct_offset(const char* strct, const char* field)
    {
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "BaseVtxOffset")) return (int)offsetof(RT::MeshInstance, BaseVtxOffset);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "BaseIdxOffset")) return (int)offsetof(RT::MeshInstance, BaseIdxOffset);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "Rotation")) return (int)offsetof(RT::MeshInstance, Rotation);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "Scale")) return (int)offsetof(RT::MeshInstance, Scale);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "MatIdx")) return (int)offsetof(RT::MeshInstance, MatIdx);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "BaseEmissiveTriOffset")) return (int)offsetof(RT::MeshInstance, BaseEmissiveTriOffset);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "Translation")) return (int)offsetof(RT::MeshInstance, Translation);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "PrevRotation")) return (int)offsetof(RT::MeshInstance, PrevRotation);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "PrevScale")) return (int)offsetof(RT::MeshInstance, PrevScale);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "dTranslation")) return (int)offsetof(RT::MeshInstance, dTranslation);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "BaseColorTex")) return (int)offsetof(RT::MeshInstance, BaseColorTex);
        if (!strcmp(strct, "MeshInstance") && !strcmp(field, "AlphaFactor_Cutoff")) return (int)offsetof(RT::MeshInstance, AlphaFactor_Cutoff);
        if (!strcmp(strct, "EmissiveTriangle") && !strcmp(field, "Vtx0")) return (int)offsetof(RT::EmissiveTriangle, Vtx0);
        if (!strcmp(strct, "EmissiveTriangle") && !strcmp(field, "V0V1")) return (int)offsetof(RT::EmissiveTriangle, V0V1);
        if (!strcmp(strct, "EmissiveTriangle") && !strcmp(field, "V0V2")) return (int)offsetof(RT::EmissiveTriangle, V0V2);
        if (!strcmp(strct, "EmissiveTriangle") && !strcmp(field, "EdgeLengths")) return (int)offsetof(RT::EmissiveTriangle, EdgeLengths);
        if (!strcmp(strct, "EmissiveTriangle") && !strcmp(field, "ID")) return (int)offsetof(RT::EmissiveTriangle, ID);
        if (!strcmp(strct, "EmissiveTriangle") && !strcmp(field, "PackedA")) return (int)offsetof(RT::EmissiveTriangle, PackedA);
        if (!strcmp(strct, "EmissiveTriangle") && !strcmp(field, "PackedB")) return (int)offsetof(RT::EmissiveTriangle, PackedB);
        if (!strcmp(strct, "EmissiveTriangle") && !strcmp(field, "UV0")) return (int)offsetof(RT::EmissiveTriangle, UV0);
        if (!strcmp(strct, "EmissiveTriangle") && !strcmp(field, "UV1")) return (int)offsetof(RT::EmissiveTriangle, UV1);
        if (!strcmp(strct, "EmissiveTriangle") && !strcmp(field, "UV2")) return (int)offsetof(RT::EmissiveTriangle, UV2);
        if (!strcmp(strct, "Material") && !strcmp(field, "BaseColorFactor")) return (int)offsetof(Material, BaseColorFactor);
        if (!strcmp(strct, "Material") && !strcmp(field, "BaseColorTex_Subsurf_CoatWeight")) return (int)offsetof(Material, BaseColorTex_Subsurf_CoatWeight);
        if (!strcmp(strct, "Material") && !strcmp(field, "NormalTex_TrDepth")) return (int)offsetof(Material, NormalTex_TrDepth);
        if (!strcmp(strct, "Material") && !strcmp(field, "MRTex_SpecRoughness_CoatRoughness")) return (int)offsetof(Material, MRTex_SpecRoughness_CoatRoughness);
        if (!strcmp(strct, "Material") && !strcmp(field, "EmissiveFactor_NormalScale")) return (int)offsetof(Material, EmissiveFactor_NormalScale);
        if (!strcmp(strct, "Material") && !strcmp(field, "EmissiveStrength_IOR")) return (int)offsetof(Material, EmissiveStrength_IOR);
        if (!strcmp(strct, "Material") && !strcmp(field, "EmissiveTex_AlphaCutoff_CoatIOR")) return (int)offsetof(Material, EmissiveTex_AlphaCutoff_CoatIOR);
        if (!strcmp(strct, "Material") && !strcmp(field, "CoatColor_Flags")) return (int)offsetof(Material, CoatColor_Flags);
        return -1;
    }
}
