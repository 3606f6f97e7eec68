// zr_common.cuh -- device math library of the ReSTIR core.
//
// CUDA counterparts of ZetaRenderPass/Common/Math.hlsli, Sampling.hlsli and the DXGI storage
// formats the reference relies on. Numeric contract (DESIGN.md "numerics"): IEEE ops only, HLSL
// mad/dot/cross/lerp as explicit fmaf chains, compiled with -fmad=false so nothing else is fused;
// transcendentals from include/zr_fpmath.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/zr_abi.h"
#include "../../include/zr_fpmath.h"

#define ZR_D __device__ __forceinline__
// Call-graph shaping: the lighting kernels inline into megabytes of SASS if everything is forced inline, which
// thrashes the instruction cache (ncu: ~80% of stall cycles "no instruction"). ZR_Fn functions become real calls
// when ZR_NI_LEVEL >= n. Inlining does not change results (no fused contraction, no fast math).
#ifndef ZR_NI_LEVEL
#define ZR_NI_LEVEL 0
#endif
#define ZR_NI static __device__ __noinline__
// Register budget of the lighting kernels: ZR_MAXREGS caps registers/thread through __launch_bounds__'s
// min-blocks argument (0 = let ptxas take what it wants).
#ifndef ZR_MAXREGS
#define ZR_MAXREGS 0
#endif
#if ZR_MAXREGS > 0
#define ZR_LB(threads) __launch_bounds__(threads, 65536 / ((threads) * ZR_MAXREGS))
#else
#define ZR_LB(threads) __launch_bounds__(threads)
#endif
#if ZR_NI_LEVEL >= 1
#define ZR_F1 ZR_NI
#else
#define ZR_F1 ZR_D
#endif
#if ZR_NI_LEVEL >= 2
#define ZR_F2 ZR_NI
#else
#define ZR_F2 ZR_D
#endif
#if ZR_NI_LEVEL >= 3
#define ZR_F3 ZR_NI
#else
#define ZR_F3 ZR_D
#endif

namespace zr
{
constexpr float PI = 3.141592654f;
constexpr float TWO_PI = 6.283185307f;
constexpr float PI_OVER_2 = 1.570796327f;
constexpr float PI_OVER_4 = 0.7853981635f;
constexpr float ONE_OVER_PI = 0.318309886f;
constexpr float ONE_OVER_2_PI = 0.159154943f;
constexpr float FLT_MAX_ = 3.402823466e+38f;
constexpr float FLT16_MAX = 65504.0f;

// ---------------------------------------------------------------------------------------------
// host-side error plumbing
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
zr_status cuda_fail(cudaError_t e, const char* what);
void count_launch(uint64_t n = 1);
#define ZR_CUDA(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return zr::cuda_fail(e__, #expr); } while (0)
// Host-side clears (reset / resize / alloc) run on the legacy default stream, which is NOT ordered against the
// cudaStreamNonBlocking streams the frames are recorded on: wait for whatever may still use the buffers before the
// memsets (ZR_CLEAR_BEGIN) and for the memsets themselves before returning (ZR_CLEAR_END), so that a Render enqueued
// right after the call can neither be overwritten by a late memset nor overwrite an early one. These are rare host calls.
#define ZR_CLEAR_BEGIN() ZR_CUDA(cudaDeviceSynchronize())
#define ZR_CLEAR_END() ZR_CUDA(cudaStreamSynchronize(cudaStreamLegacy))
void prof_before(const char* name, cudaStream_t stream);
void prof_after();
#define ZR_PROF(name, stream) zr::prof_before(name, (cudaStream_t)(stream))
#define ZR_LAUNCH_CHECK() do { zr::count_launch(); zr::prof_after(); cudaError_t e__ = cudaGetLastError(); if (e__ != cudaSuccess) return zr::cuda_fail(e__, "kernel launch"); } while (0)

// ---------------------------------------------------------------------------------------------
// vectors
// ---------------------------------------------------------------------------------------------
ZR_D float3 f3(float x, float y, float z) { return make_float3(x, y, z); }
ZR_D float3 f3(float s) { return make_float3(s, s, s); }
ZR_D float2 f2(float x, float y) { return make_float2(x, y); }
ZR_D float4 f4(float x, float y, float z, float w) { return make_float4(x, y, z, w); }

ZR_D float3 operator+(float3 a, float3 b) { return f3(a.x + b.x, a.y + b.y, a.z + b.z); }
ZR_D float3 operator-(float3 a, float3 b) { return f3(a.x - b.x, a.y - b.y, a.z - b.z); }
ZR_D float3 operator*(float3 a, float3 b) { return f3(a.x * b.x, a.y * b.y, a.z * b.z); }
ZR_D float3 operator/(float3 a, float3 b) { return f3(a.x / b.x, a.y / b.y, a.z / b.z); }
ZR_D float3 operator*(float3 a, float s) { return f3(a.x * s, a.y * s, a.z * s); }
ZR_D float3 operator*(float s, float3 a) { return f3(s * a.x, s * a.y, s * a.z); }
ZR_D float3 operator/(float3 a, float s) { return f3(a.x / s, a.y / s, a.z / s); }
ZR_D float3 operator/(float s, float3 a) { return f3(s / a.x, s / a.y, s / a.z); }
ZR_D float3 operator+(float3 a, float s) { return f3(a.x + s, a.y + s, a.z + s); }
ZR_D float3 operator-(float3 a, float s) { return f3(a.x - s, a.y - s, a.z - s); }
ZR_D float3 operator-(float s, float3 a) { return f3(s - a.x, s - a.y, s - a.z); }
ZR_D float3 operator-(float3 a) { return f3(-a.x, -a.y, -a.z); }
ZR_D float3& operator+=(float3& a, float3 b) { a = a + b; return a; }
ZR_D float3& operator*=(float3& a, float3 b) { a = a * b; return a; }
ZR_D float3& operator*=(float3& a, float s) { a = a * s; return a; }
ZR_D float3& operator/=(float3& a, float s) { a = a / s; return a; }
ZR_D float2 operator+(float2 a, float2 b) { return f2(a.x + b.x, a.y + b.y); }
ZR_D float2 operator-(float2 a, float2 b) { return f2(a.x - b.x, a.y - b.y); }
ZR_D float2 operator*(float2 a, float2 b) { return f2(a.x * b.x, a.y * b.y); }
ZR_D float2 operator*(float2 a, float s) { return f2(a.x * s, a.y * s); }
ZR_D float2 operator/(float2 a, float2 b) { return f2(a.x / b.x, a.y / b.y); }
ZR_D float2 operator/(float2 a, float s) { return f2(a.x / s, a.y / s); }
ZR_D float2 operator+(float2 a, float s) { return f2(a.x + s, a.y + s); }
ZR_D float2 operator-(float2 a, float s) { return f2(a.x - s, a.y - s); }

ZR_D float asfloat(uint32_t u) { return __uint_as_float(u); }
ZR_D uint32_t asuint(float f) { return __float_as_uint(f); }

// ---- the numeric contract ----
ZR_D float mad(float a, float b, float c) { return fmaf(a, b, c); }
ZR_D float3 mad(float3 a, float3 b, float3 c) { return f3(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y), fmaf(a.z, b.z, c.z)); }
ZR_D float3 mad(float a, float3 b, float3 c) { return f3(fmaf(a, b.x, c.x), fmaf(a, b.y, c.y), fmaf(a, b.z, c.z)); }
ZR_D float3 mad(float3 a, float b, float3 c) { return f3(fmaf(a.x, b, c.x), fmaf(a.y, b, c.y), fmaf(a.z, b, c.z)); }
ZR_D float3 mad(float3 a, float b, float c) { return f3(fmaf(a.x, b, c), fmaf(a.y, b, c), fmaf(a.z, b, c)); }
ZR_D float dot(float3 a, float3 b) { return fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)); }
ZR_D float dot(float2 a, float2 b) { return fmaf(a.y, b.y, a.x * b.x); }
ZR_D float dot(float4 a, float4 b) { return fmaf(a.w, b.w, fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x))); }
ZR_D float3 cross(float3 a, float3 b)
{
    return f3(fmaf(a.y, b.z, -(a.z * b.y)), fmaf(a.z, b.x, -(a.x * b.z)), fmaf(a.x, b.y, -(a.y * b.x)));
}
ZR_D float length(float3 v) { return sqrtf(dot(v, v)); }
ZR_D float rsqrt_(float x) { return 1.0f / sqrtf(x); }
ZR_D float3 normalize(float3 v) { return v * rsqrt_(dot(v, v)); }
ZR_D float4 normalize(float4 v) { float r = rsqrt_(dot(v, v)); return f4(v.x * r, v.y * r, v.z * r, v.w * r); }
ZR_D float saturate(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }
ZR_D float3 saturate(float3 v) { return f3(saturate(v.x), saturate(v.y), saturate(v.z)); }
ZR_D float2 saturate(float2 v) { return f2(saturate(v.x), saturate(v.y)); }
ZR_D float lerp(float a, float b, float t) { return fmaf(t, b - a, a); }
ZR_D float3 abs3(float3 v) { return f3(fabsf(v.x), fabsf(v.y), fabsf(v.z)); }
ZR_D float3 max3(float3 a, float3 b) { return f3(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z)); }
ZR_D float3 max3(float3 a, float s) { return f3(fmaxf(a.x, s), fmaxf(a.y, s), fmaxf(a.z, s)); }
ZR_D float3 sqrt3(float3 a) { return f3(sqrtf(a.x), sqrtf(a.y), sqrtf(a.z)); }
ZR_D float3 reflect(float3 i, float3 n) { return i - (2.0f * dot(n, i)) * n; }
ZR_D float3 refract(float3 i, float3 n, float eta)
{
    float ndoti = dot(n, i);
    float k = 1.0f - eta * eta * (1.0f - ndoti * ndoti);
    if (k < 0.0f)
        return f3(0.0f);
    return eta * i - (eta * ndoti + sqrtf(k)) * n;
}
ZR_D bool isnan3(float3 v) { return (v.x != v.x) || (v.y != v.y) || (v.z != v.z); }
ZR_D bool isinf1(float x) { return fabsf(x) == asfloat(0x7f800000u); }
ZR_D bool isinf3(float3 v) { return isinf1(v.x) || isinf1(v.y) || isinf1(v.z); }

namespace Math
{
    ZR_D float NextFloat32(float f)
    {
        if (f == -0.0f) f = 0.0f;
        uint32_t u = asuint(f);
        u = f >= 0 ? u + 1 : u - 1;
        return asfloat(u);
    }
    ZR_D float PrevFloat32(float f)
    {
        if (f == 0.0f) f = -0.0f;
        uint32_t u = asuint(f);
        u = f > 0 ? u - 1 : u + 1;
        return asfloat(u);
    }
    ZR_D float Lerp(float v0, float v1, float t) { return mad(t, v1, mad(-t, v0, v0)); }
    ZR_D float3 Lerp(float3 v0, float3 v1, float t) { return mad(t, v1, mad(-t, v0, v0)); }
    ZR_D float Sanitize(float x) { return (x != x) || isinf1(x) ? 0.0f : x; }
    ZR_D float3 Sanitize(float3 v) { return isnan3(v) || isinf3(v) ? f3(0.0f) : v; }
    ZR_D float ArcCos(float x)
    {
        float xAbs = fabsf(x);
        float res = mad(-0.0206453f, xAbs, 0.0764532f);
        res = mad(res, xAbs, -0.21271f);
        res = mad(res, xAbs, 1.57075f);
        res *= sqrtf(1.0f - xAbs);
        return x >= 0 ? res : PI - res;
    }
    ZR_D float SignNotZero(float x) { return asfloat(0x3f800000u | (0x80000000u & asuint(x))); }
    ZR_D float2 NDCFromUV(float2 uv) { float2 ndc = uv * 2.0f - 1.0f; ndc.y = -ndc.y; return ndc; }
    ZR_D float2 UVFromNDC(float2 ndc) { return ndc * f2(0.5f, -0.5f) + 0.5f; }
    ZR_D float Luminance(float3 c) { return dot(f3(0.2126f, 0.7152f, 0.0722f), c); }

    ZR_D float3 mul3x4(const float m[3][4], float3 v)
    {
        float4 p = f4(v.x, v.y, v.z, 1.0f);
        return f3(dot(f4(m[0][0], m[0][1], m[0][2], m[0][3]), p),
                  dot(f4(m[1][0], m[1][1], m[1][2], m[1][3]), p),
                  dot(f4(m[2][0], m[2][1], m[2][2], m[2][3]), p));
    }
    ZR_D float3 WorldPosFromScreenSpace(float2 pos_ss, float2 renderDim, float z_view, float tanHalfFOV,
        float aspectRatio, const float viewInv[3][4], float2 jitter)
    {
        float2 uv = (pos_ss + 0.5f + jitter) / renderDim;
        float2 ndc = NDCFromUV(uv);
        float3 dir_v = f3(ndc.x * aspectRatio * tanHalfFOV * z_view, ndc.y * tanHalfFOV * z_view, z_view);
        return mul3x4(viewInv, dir_v);
    }
    ZR_D float3 WorldPosFromUV(float2 uv, float2 renderDim, float z_view, float tanHalfFOV,
        float aspectRatio, const float viewInv[3][4], float2 jitter)
    {
        float2 ndc = NDCFromUV(uv) + jitter / renderDim;
        float3 dir_v = f3(ndc.x * aspectRatio * tanHalfFOV * z_view, ndc.y * tanHalfFOV * z_view, z_view);
        return mul3x4(viewInv, dir_v);
    }
    ZR_D float3 WorldPosFromScreenSpace2(float2 pos_ss, float2 renderDim, float z_view, float tanHalfFOV,
        float aspectRatio, float2 jitter, float3 viewBasisX, float3 viewBasisY, float3 viewBasisZ,
        bool thinLens, float2 lensSample, float focusDepth, float3& origin)
    {
        float2 uv = (pos_ss + 0.5f + jitter) / renderDim;
        float2 ndc = NDCFromUV(uv);
        float3 dir_w;
        if (!thinLens)
        {
            float3 dir_v = f3(ndc.x * aspectRatio * tanHalfFOV * z_view, ndc.y * tanHalfFOV * z_view, z_view);
            dir_w = mad(dir_v.x, viewBasisX, mad(dir_v.y, viewBasisY, dir_v.z * viewBasisZ));
        }
        else
        {
            float3 dir_v = f3(ndc.x * aspectRatio * tanHalfFOV, ndc.y * tanHalfFOV, 1);
            float3 focalPoint = focusDepth * dir_v;
            dir_v = focalPoint - f3(lensSample.x, lensSample.y, 0);
            dir_w = mad(dir_v.x, viewBasisX, mad(dir_v.y, viewBasisY, dir_v.z * viewBasisZ));
            dir_w = normalize(dir_w);
            dir_w *= z_view;
            origin += mad(lensSample.x, viewBasisX, lensSample.y * viewBasisY);
        }
        return origin + dir_w;
    }

    struct CoordinateSystem
    {
        float3 b1, b2;
        static ZR_D CoordinateSystem Build(float3 n)
        {
            const float s = SignNotZero(n.z);
            const float a = -1.0f / (s + n.z);
            const float b = n.x * n.y * a;
            CoordinateSystem ret;
            ret.b1 = f3(mad(n.x * a, n.x * s, 1.0f), s * b, -s * n.x);
            ret.b2 = f3(b, mad(n.y * a, n.y, s), -n.y);
            return ret;
        }
    };

    struct TriDifferentials
    {
        float3 dpdu, dpdv, dndu, dndv;
        static ZR_D TriDifferentials Compute(float3 p0, float3 p1, float3 p2, float3 n0, float3 n1, float3 n2,
            float2 uv0, float2 uv1, float2 uv2)
        {
            TriDifferentials ret;
            float2 duv10 = uv1 - uv0;
            float2 duv20 = uv2 - uv0;
            float det = duv10.x * duv20.y - duv10.y * duv20.x;
            float invdet = 1.0f / det;
            if (fabsf(det) < 1e-7f)
            {
                float3 normal = normalize(cross(p1 - p0, p2 - p0));
                CoordinateSystem onb = CoordinateSystem::Build(normal);
                ret.dpdu = onb.b1;
                ret.dpdv = onb.b2;
                ret.dndu = f3(0);
                ret.dndv = f3(0);
                return ret;
            }
            float3 dp10 = p1 - p0;
            float3 dp20 = p2 - p0;
            ret.dpdu = (duv20.y * dp10 - duv10.y * dp20) * invdet;
            ret.dpdv = (-duv20.x * dp10 + duv10.x * dp20) * invdet;
            float3 dn10 = n1 - n0;
            float3 dn20 = n2 - n0;
            ret.dndu = (duv20.y * dn10 - duv10.y * dn20) * invdet;
            ret.dndv = (-duv20.x * dn10 + duv10.x * dn20) * invdet;
            return ret;
        }
    };

    ZR_D float3 RotateVector(float3 v, float4 q)
    {
        float3 imaginary = f3(q.x, q.y, q.z);
        float real = q.w;
        float3 t = cross(2.0f * imaginary, v);
        return v + real * t + cross(imaginary, t);
    }
    ZR_D float3 TransformTRS(float3 pos, float3 translation, float4 rotation, float3 scale)
    {
        float3 transformed = pos * scale;
        transformed = RotateVector(transformed, rotation);
        transformed += translation;
        return transformed;
    }
    ZR_D float3 InverseTransformTRS(float3 pos, float3 translation, float4 rotation, float3 scale)
    {
        float3 transformed = pos - translation;
        float4 q_conjugate = f4(-rotation.x, -rotation.y, -rotation.z, rotation.w);
        transformed = RotateVector(transformed, q_conjugate);
        transformed *= 1.0f / scale;
        return transformed;
    }

    ZR_D uint32_t FloatToUNorm8(float f) { f = saturate(f); return (uint32_t)mad(f, 255.0f, 0.5f); }
    ZR_D float UNorm8ToFloat(uint32_t u) { return (float)u / 255.0f; }
    ZR_D uint32_t FloatToUNorm16(float f) { f = saturate(f); return (uint32_t)(uint16_t)mad(f, 65535.0f, 0.5f); }
    ZR_D float UNorm16ToFloat(uint32_t u) { return (float)u / 65535.0f; }
    ZR_D float4 DecodeNormalized4(const uint16_t u[4])
    {
        float4 d = f4((float)u[0] / 65535.0f, (float)u[1] / 65535.0f, (float)u[2] / 65535.0f, (float)u[3] / 65535.0f);
        return f4(mad(d.x, 2.0f, -1.0f), mad(d.y, 2.0f, -1.0f), mad(d.z, 2.0f, -1.0f), mad(d.w, 2.0f, -1.0f));
    }
    ZR_D float2 EncodeUnitVector(float3 n)
    {
        float s = fabsf(n.x) + fabsf(n.y) + fabsf(n.z);
        float2 p = f2(n.x / s, n.y / s);
        float2 encoded = (n.z <= 0.0f) ?
            f2((1.0f - fabsf(p.y)) * SignNotZero(p.x), (1.0f - fabsf(p.x)) * SignNotZero(p.y)) : p;
        return f2(mad(encoded.x, 0.5f, 0.5f), mad(encoded.y, 0.5f, 0.5f));
    }
    ZR_D float3 DecodeUnitVector(float2 u)
    {
        u = f2(mad(u.x, 2.0f, -1.0f), mad(u.y, 2.0f, -1.0f));
        float3 n = f3(u.x, u.y, 1.0f - fabsf(u.x) - fabsf(u.y));
        float t = saturate(-n.z);
        n.x += n.x >= 0.0f ? -t : t;
        n.y += n.y >= 0.0f ? -t : t;
        return normalize(n);
    }
    ZR_D uint32_t EncodeUNorm2(float2 u)
    {
        u = saturate(u);
        uint32_t x = (uint32_t)(uint16_t)mad(u.x, 65535.0f, 0.5f);
        uint32_t y = (uint32_t)(uint16_t)mad(u.y, 65535.0f, 0.5f);
        return x | (y << 16);
    }
    ZR_D float2 DecodeUNorm2(uint32_t e) { return f2((float)(e & 0xffff) / 65535.0f, (float)(e >> 16) / 65535.0f); }
    ZR_D uint32_t EncodeOct32u(float3 n) { return EncodeUNorm2(EncodeUnitVector(n)); }
    ZR_D float3 DecodeOct32(uint32_t e) { return DecodeUnitVector(DecodeUNorm2(e)); }
    ZR_D float3 UnpackRGB8(uint32_t rgb)
    {
        return f3((float)(rgb & 0xff) / 255.0f, (float)((rgb >> 8) & 0xff) / 255.0f, (float)((rgb >> 16) & 0xff) / 255.0f);
    }
    ZR_D uint32_t Float3ToRGB8(float3 v)
    {
        v = saturate(v);
        uint32_t x = (uint32_t)mad(v.x, 255.0f, 0.5f), y = (uint32_t)mad(v.y, 255.0f, 0.5f), z = (uint32_t)mad(v.z, 255.0f, 0.5f);
        return x | (y << 8) | (z << 16);
    }
}

// ---- storage formats ----
ZR_D uint32_t pack_half2(float a, float b) { return (uint32_t)zr_f32_to_f16(a) | ((uint32_t)zr_f32_to_f16(b) << 16); }
ZR_D float half_lo(uint32_t p) { return zr_f16_to_f32((uint16_t)(p & 0xffff)); }
ZR_D float half_hi(uint32_t p) { return zr_f16_to_f32((uint16_t)(p >> 16)); }
ZR_D float to_half(float f) { return zr_f16_to_f32(zr_f32_to_f16(f)); }
ZR_D uint32_t snorm16_enc(float f)
{
    if (f != f) f = 0.0f;
    f = fminf(fmaxf(f, -1.0f), 1.0f);
    f = f * 32767.0f;
    int i = (int)(f >= 0 ? f + 0.5f : f - 0.5f);
    return (uint32_t)(uint16_t)(int16_t)i;
}
ZR_D uint32_t pack_snorm16x2(float2 v) { return snorm16_enc(v.x) | (snorm16_enc(v.y) << 16); }
ZR_D float snorm16_dec(uint32_t u) { int16_t i = (int16_t)(uint16_t)u; return fmaxf((float)i / 32767.0f, -1.0f); }
ZR_D float2 unpack_snorm16x2(uint32_t p) { return f2(snorm16_dec(p & 0xffff), snorm16_dec(p >> 16)); }
ZR_D uint32_t f32_to_ufloat(float f, int mbits)
{
    if (f != f) return ((0x1fu << mbits) | 1u);
    if (f <= 0.0f) return 0;
    uint32_t u = asuint(f);
    int e = (int)(u >> 23) - 127 + 15;
    uint32_t m = u & 0x7fffffu;
    if (e >= 31) return (0x1eu << mbits) | ((1u << mbits) - 1u);
    if (e <= 0)
    {
        if (e < -mbits) return 0;
        m = (m | 0x800000u) >> (1 - e);
        return m >> (23 - mbits);
    }
    return ((uint32_t)e << mbits) | (m >> (23 - mbits));
}
ZR_D float ufloat_to_f32(uint32_t v, int mbits)
{
    uint32_t e = v >> mbits;
    uint32_t m = v & ((1u << mbits) - 1u);
    if (e == 0)
    {
        if (m == 0) return 0.0f;
        return (float)m * (1.0f / (float)(1u << mbits)) * 6.103515625e-05f;
    }
    if (e == 31) return m ? asfloat(0x7fc00000u) : asfloat(0x7f800000u);
    return asfloat(((e + 112u) << 23) | (m << (23 - mbits)));
}
ZR_D uint32_t pack_r11g11b10(float3 c)
{
    return f32_to_ufloat(c.x, 6) | (f32_to_ufloat(c.y, 6) << 11) | (f32_to_ufloat(c.z, 5) << 22);
}
ZR_D float3 unpack_r11g11b10(uint32_t p)
{
    return f3(ufloat_to_f32(p & 0x7ff, 6), ufloat_to_f32((p >> 11) & 0x7ff, 6), ufloat_to_f32(p >> 22, 5));
}

// ---- RNG (Sampling.hlsli:12-159) ----
struct RNG
{
    uint32_t State;
    static ZR_D uint32_t PCG(uint32_t x)
    {
        uint32_t state = x * 747796405u + 2891336453u;
        uint32_t word = ((state >> ((state >> 28u) + 4u)) ^ state) * 277803737u;
        return (word >> 22u) ^ word;
    }
    static ZR_D uint3 PCG3d(uint3 v)
    {
        v.x = v.x * 1664525u + 1013904223u; v.y = v.y * 1664525u + 1013904223u; v.z = v.z * 1664525u + 1013904223u;
        v.x += v.y * v.z; v.y += v.z * v.x; v.z += v.x * v.y;
        v.x ^= v.x >> 16u; v.y ^= v.y >> 16u; v.z ^= v.z >> 16u;
        v.x += v.y * v.z; v.y += v.z * v.x; v.z += v.x * v.y;
        return v;
    }
    static ZR_D uint4 PCG4d(uint4 v)
    {
        v.x = v.x * 1664525u + 1013904223u; v.y = v.y * 1664525u + 1013904223u;
        v.z = v.z * 1664525u + 1013904223u; v.w = v.w * 1664525u + 1013904223u;
        v.x += v.y * v.w; v.y += v.z * v.x; v.z += v.x * v.y; v.w += v.y * v.z;
        v.x ^= v.x >> 16u; v.y ^= v.y >> 16u; v.z ^= v.z >> 16u; v.w ^= v.w >> 16u;
        v.x += v.y * v.w; v.y += v.z * v.x; v.z += v.x * v.y; v.w += v.y * v.z;
        return v;
    }
    static ZR_D RNG Init(uint32_t px, uint32_t py, uint32_t frame) { RNG r; r.State = PCG3d(make_uint3(px, py, frame)).x; return r; }
    static ZR_D RNG Init4(uint32_t px, uint32_t py, uint32_t frame, uint32_t idx) { RNG r; r.State = PCG4d(make_uint4(px, py, frame, idx)).x; return r; }
    static ZR_D RNG InitIdx(uint32_t idx, uint32_t frame) { RNG r; r.State = PCG(idx + PCG(frame)); return r; }
    static ZR_D RNG InitSeed(uint32_t seed) { RNG r; r.State = seed; return r; }
    ZR_D uint32_t UniformUint()
    {
        State = State * 747796405u + 2891336453u;
        uint32_t word = ((State >> ((State >> 28u) + 4u)) ^ State) * 277803737u;
        return (word >> 22u) ^ word;
    }
    ZR_D float Uniform() { return (float)(UniformUint() >> 8) * 0x1p-24f; }
    ZR_D uint32_t UniformUintBounded(uint32_t bound)
    {
        uint32_t threshold = (~bound + 1u) % bound;
        for (;;)
        {
            uint32_t r = UniformUint();
            if (r >= threshold)
                return r % bound;
        }
    }
    ZR_D uint32_t UniformUintBounded_Faster(uint32_t bound) { return (uint32_t)(Uniform() * (float)bound); }
    ZR_D float2 Uniform2D() { float a = Uniform(); float b = Uniform(); return f2(a, b); }
    ZR_D float3 Uniform3D() { float a = Uniform(); float b = Uniform(); float c = Uniform(); return f3(a, b, c); }
    ZR_D void Uniform4D() { Uniform(); Uniform(); Uniform(); Uniform(); }
};

namespace Sampling
{
    ZR_D float3 SampleCosineWeightedHemisphere(float2 u, float& pdf)
    {
        const float phi = TWO_PI * u.y;
        const float sinTheta = sqrtf(u.x);
        float s, c;
        zr_sincosf(phi, &s, &c);
        const float x = c * sinTheta;
        const float y = s * sinTheta;
        const float z = sqrtf(1.0f - u.x);
        pdf = z * ONE_OVER_PI;
        return f3(x, y, z);
    }
    ZR_D float2 UniformSampleDiskConcentric(float2 u)
    {
        float a = 2.0f * u.x - 1.0f;
        float b = 2.0f * u.y - 1.0f;
        if (a == 0 && b == 0)
            return f2(0, 0);
        float r, phi;
        if (a * a > b * b) { r = a; phi = PI_OVER_4 * (b / a); }
        else { r = b; phi = PI_OVER_2 - PI_OVER_4 * (a / b); }
        float s, c;
        zr_sincosf(phi, &s, &c);
        return f2(r * c, r * s);
    }
    ZR_D float2 UniformSampleTriangle(float2 u)
    {
        float b1, b2;
        if (u.y > u.x) { b1 = u.x * 0.5f; b2 = u.y - b1; }
        else { b2 = u.y * 0.5f; b1 = u.x - b2; }
        return f2(b1, b2);
    }
}

// Common.hlsli:127-157
ZR_D uint2 SwizzleThreadGroup(uint32_t Gidx, uint32_t Gidy, uint32_t GTx, uint32_t GTy, uint32_t groupDimX,
    uint32_t groupDimY, uint32_t dispatchDimX, uint32_t tileWidth, uint32_t log2TileWidth,
    uint32_t numGroupsInTile, uint2& swizzledGid)
{
    const uint32_t groupIDFlattened = Gidy * dispatchDimX + Gidx;
    const uint32_t tileID = groupIDFlattened / numGroupsInTile;
    const uint32_t groupIDinTileFlattened = groupIDFlattened % numGroupsInTile;
    const uint32_t numFullTiles = dispatchDimX / tileWidth;
    const uint32_t numGroupsInFullTiles = numFullTiles * numGroupsInTile;
    uint32_t gx, gy;
    if (groupIDFlattened >= numGroupsInFullTiles)
    {
        const uint32_t lastTileDimX = dispatchDimX - tileWidth * numFullTiles;
        gx = groupIDinTileFlattened % lastTileDimX;
        gy = groupIDinTileFlattened / lastTileDimX;
    }
    else
    {
        gx = groupIDinTileFlattened & (tileWidth - 1);
        gy = groupIDinTileFlattened >> log2TileWidth;
    }
    const uint32_t swizzledGidFlattened = gy * dispatchDimX + tileID * tileWidth + gx;
    swizzledGid = make_uint2(swizzledGidFlattened % dispatchDimX, swizzledGidFlattened / dispatchDimX);
    return make_uint2(swizzledGid.x * groupDimX + GTx, swizzledGid.y * groupDimY + GTy);
}

// Wave sum with the contract's fixed xor-butterfly order; inactive lanes must pass 0.
ZR_D float WaveSum32(float v)
{
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1)
        v = v + __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}
ZR_D float WaveMax32(float v)
{
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1)
        v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, off));
    return v;
}

// 128-bit streaming accesses for the per-pixel records
ZR_D uint4 ld128(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
ZR_D uint4 ld128_rw(const void* p) { return *reinterpret_cast<const uint4*>(p); }
ZR_D void st128(void* p, uint4 v) { *reinterpret_cast<uint4*>(p) = v; }
} // namespace zr
