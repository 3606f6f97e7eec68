// zr_pixel.cuh -- per-pixel reconstruction from the packed G-buffer, shared by the lighting passes.
// Every reference kernel starts with the same ~60 lines (e.g. ReSTIR_PT_PathTrace.hlsl:441-524,
// ReSTIR_DI_Temporal.hlsl:289-360): flags, depth -> world position (pinhole or thin lens), normal,
// base colour / IOR / coat -> BSDF::ShadingData. Here that is one 128-bit load + this function.
#pragma once
#include "zr_rt.cuh"

namespace zr
{
struct GFlags { bool metallic, transmissive, emissive, invalid, trDepthGt0, subsurface, coated; };

ZR_D GFlags DecodeFlags(uint32_t v)
{
    GFlags r;
    r.transmissive = (v & 0x1) != 0;
    r.emissive = (v & (1 << 1)) != 0;
    r.invalid = (v & (1 << 2)) != 0;
    r.trDepthGt0 = (v & (1 << 3)) != 0;
    r.subsurface = (v & (1 << 4)) != 0;
    r.coated = (v & (1 << 5)) != 0;
    r.metallic = (v & (1 << 7)) != 0;
    return r;
}

ZR_D float DecodeIOR(float e) { return mad(e, 2.5f - 1.0f, 1.0f); }

struct FrameView
{
    zr_frame_constants fc;
    const uint4* core; const float* depth; const uint2* me; const uint2* coat;     // current
    const uint4* pcore; const uint2* pcoat;                                         // previous
    uint32_t W, H;
};

// Checks the lighting passes share before a render, then the FrameView over the frame's G-buffers: scene and current G-buffer
// present, a frame of the pass's size, emissive triangles with their alias table, the presampled light sets when enabled.
// `pass` ("zr_direct_pass", ...) prefixes the error messages.
inline zr_status LightingFrame(const char* pass, const zr_frame_inputs* in, uint32_t width, uint32_t height, FrameView& f)
{
    if (!in || !in->scene || !in->curr.d_core || !in->curr.d_motion_emissive || !in->curr.d_coat)
    {
        set_error("%s_render: missing scene or G-buffer", pass);
        return ZR_ERR_INVALID_ARG;
    }
    const zr_status st = check_frame_size(pass, in->frame, width, height);
    if (st != ZR_OK) return st;
    if (in->scene->dev.numEmissives == 0 || !in->scene->aliasBuilt)
    {
        // PathTracer.cpp:274-284: the emissive variants only run when the scene has emissive triangles
        set_error("%s_render: needs emissive triangles and zr_prelighting_render first (the sun/sky variants are not part of this build)", pass);
        return ZR_ERR_UNSUPPORTED;
    }
    if (in->scene->dev.sampleSetSize && !in->scene->samplesValid)
    {
        set_error("%s_render: presampling is enabled but zr_presample_emissives has not run", pass);
        return ZR_ERR_NOT_INITIALIZED;
    }
    f.fc = in->frame;
    f.core = (const uint4*)in->curr.d_core; f.depth = (const float*)in->curr.d_depth;
    f.me = (const uint2*)in->curr.d_motion_emissive; f.coat = (const uint2*)in->curr.d_coat;
    f.pcore = (const uint4*)in->prev.d_core; f.pcoat = (const uint2*)in->prev.d_coat;
    f.W = width; f.H = height;
    return ZR_OK;
}

// accounts the cycles a block took to the tile of its first pixel
ZR_D void AccountCost(unsigned long long* costMap, uint32_t W, uint32_t H, uint32_t x, uint32_t y, long long t0)
{
    if (costMap && threadIdx.x == 0 && x < W && y < H)
        atomicAdd(&costMap[(size_t)(y >> 5) * ((W + 31) >> 5) + (x >> 5)], (unsigned long long)(clock64() - t0));
}

template<class SD>
struct PixelT
{
    GFlags flags; float roughness; float z; float3 pos, normal, origin; float2 lensSample;
    SD surface; float eta_next;
    float coatRoughness, coatIor;   // raw coat parameters (ShadingData keeps alpha / relative eta)
};
using Pixel = PixelT<BSDF::ShadingData>;

ZR_D float3 row3(const float m[3][4], int r) { return f3(m[r][0], m[r][1], m[r][2]); }

ZR_D GFlags FlagsAt(const uint4* __restrict__ core, uint32_t W, int x, int y, float* roughness = nullptr)
{
    const uint32_t w = __ldg(&core[(size_t)y * W + x].w);
    if (roughness) *roughness = (float)((w >> 8) & 0xff) / 255.0f;
    return DecodeFlags(w & 0xff);
}

// prev == false: current camera / jitter / frame number; true: previous frame's. SD: the surface type of the calling kernel
// (BSDF::ShadingDataT<scene material features>)
template<class SD = BSDF::ShadingData>
ZR_D PixelT<SD> LoadPixel(const FrameView& f, const SceneDev& sc, const uint4* __restrict__ core, const uint2* __restrict__ coat,
    int px, int py, bool prev, int coatX, int coatY)
{
    const zr_frame_constants& fc = f.fc;
    PixelT<SD> p;
    const uint4 c = ld128(&core[(size_t)py * f.W + px]);
    p.flags = DecodeFlags(c.w & 0xff);
    p.roughness = (float)((c.w >> 8) & 0xff) / 255.0f;
    p.z = asfloat(c.x);
    p.lensSample = f2(0, 0);
    p.origin = prev ? f3(fc.PrevViewInv[0][3], fc.PrevViewInv[1][3], fc.PrevViewInv[2][3]) : f3(fc.CameraPos[0], fc.CameraPos[1], fc.CameraPos[2]);
    if (fc.DoF)
    {
        const uint3 h = RNG::PCG3d(make_uint3((uint32_t)px, (uint32_t)py, (uint32_t)px));
        RNG rngDoF = RNG::Init(h.z, h.y, prev ? fc.FrameNum - 1 : fc.FrameNum);
        p.lensSample = Sampling::UniformSampleDiskConcentric(rngDoF.Uniform2D());
        p.lensSample = p.lensSample * fc.LensRadius;
    }
    const float2 renderDim = f2((float)f.W, (float)f.H);
    const float2 jitter = prev ? f2(fc.PrevCameraJitter[0], fc.PrevCameraJitter[1]) : f2(fc.CurrCameraJitter[0], fc.CurrCameraJitter[1]);
    const float3 bx = prev ? row3(fc.PrevView, 0) : row3(fc.CurrView, 0);
    const float3 by = prev ? row3(fc.PrevView, 1) : row3(fc.CurrView, 1);
    const float3 bz = prev ? row3(fc.PrevView, 2) : row3(fc.CurrView, 2);
    p.pos = Math::WorldPosFromScreenSpace2(f2((float)px, (float)py), renderDim, p.z, fc.TanHalfFOV, fc.AspectRatio, jitter,
        bx, by, bz, fc.DoF != 0, p.lensSample, fc.FocusDepth, p.origin);
    p.normal = Math::DecodeUnitVector(Math::DecodeUNorm2(c.y));
    const float3 baseColor = f3((float)(c.z & 0xff) / 255.0f, (float)((c.z >> 8) & 0xff) / 255.0f, (float)((c.z >> 16) & 0xff) / 255.0f);
    const float baseW = p.flags.subsurface ? (float)(c.z >> 24) / 255.0f : 0.0f;
    p.eta_next = BSDF::DEFAULT_ETA_MAT;
    if (p.flags.transmissive)
        p.eta_next = DecodeIOR((float)((c.w >> 16) & 0xff) / 255.0f);
    float coat_weight = 0; float3 coat_color = f3(0.0f); float coat_roughness = 0; float coat_ior = BSDF::DEFAULT_ETA_COAT;
    if (p.flags.coated)
    {
        const uint2 cc = __ldg(&coat[(size_t)coatY * f.W + coatX]);
        const uint32_t px_ = cc.x & 0xffff, py_ = cc.x >> 16, pz_ = cc.y & 0xffff;
        coat_weight = Math::UNorm8ToFloat((py_ >> 8) & 0xff);
        coat_roughness = Math::UNorm8ToFloat(pz_ & 0xff);
        coat_color = Math::UnpackRGB8(px_ | ((py_ & 0xff) << 16));
        coat_ior = DecodeIOR(Math::UNorm8ToFloat(pz_ >> 8));
    }
    p.coatRoughness = coat_roughness; p.coatIor = coat_ior;
    const float3 wo = normalize(p.origin - p.pos);
    p.surface = SD::Init(p.normal, wo, p.flags.metallic, p.roughness, baseColor, BSDF::ETA_AIR, p.eta_next,
        p.flags.transmissive, p.flags.trDepthGt0 ? 1.0f : 0.0f, to_half(baseW), coat_weight, coat_color, coat_roughness,
        coat_ior, sc.rho);
    return p;
}

ZR_D void WriteOutputColor(const zr_frame_constants& fc, float4* __restrict__ finalImg, size_t idx, float3 li)
{
    li = isnan3(li) ? f3(0) : li;
    if (fc.Accumulate && fc.CameraStatic && fc.NumFramesCameraStatic > 1)
    {
        const float4 prev = finalImg[idx];
        finalImg[idx] = f4(prev.x + li.x, prev.y + li.y, prev.z + li.z, prev.w);
    }
    else
        finalImg[idx] = f4(li.x, li.y, li.z, 0.0f);
}
} // namespace zr
