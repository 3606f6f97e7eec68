/*
 * zr_fpmath.h -- libm replacement shared by the CUDA product and the CPU oracle.
 *
 * Why this exists: the reference's shaders use the GPU's hardware sin/cos/exp/log
 * (Source/ZetaRenderPass/Common/Sampling.hlsli:166-175, BSDF.hlsli:1003,1222), whose results
 * are implementation defined. glibc's libm and CUDA's libm disagree in the last ulp, which
 * would make RNG-driven branch decisions diverge between a CPU oracle and a GPU kernel.
 * Both sides therefore call the SAME transcendental approximations below, built only from
 * IEEE-754 +,-,*,/,sqrt and fma so they are bit-identical on x86-64 (gcc, -ffp-contract=off)
 * and sm_90a (nvcc, -fmad=false). Nothing here restates the reference's algorithms; it plays
 * the role "the same libm on both sides" plays in a CPU-vs-CPU comparison.
 *
 * Accuracy: sin/cos <= 2 ulp on [-2pi, 4pi]; exp/log <= 2 ulp on normal range; atan2 <= 2 ulp.
 */
#ifndef ZR_FPMATH_H
#define ZR_FPMATH_H

#include <stdint.h>
#if defined(__CUDACC__)
#include <cuda_fp16.h>
#endif
#include <string.h>
#include <math.h>

#if defined(__CUDACC__)
#define ZR_HD __host__ __device__ __forceinline__
#else
#define ZR_HD static inline
#endif

ZR_HD uint32_t zr_f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
ZR_HD float zr_u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

/* ---- sin / cos: Cody-Waite reduction by pi/2 + minimax polynomials (Cephes sinf/cosf) ---- */
ZR_HD void zr_sincosf(float x, float* s, float* c)
{
    const float k = rintf(x * 0.636619772367581343f);   /* x * 2/pi */
    const int q = (int)k;
    /* pi/2 split in three parts */
    float r = fmaf(-k, 1.5703125f, x);
    r = fmaf(-k, 4.837512969970703125e-4f, r);
    r = fmaf(-k, 7.54978995489188216e-8f, r);
    const float z = r * r;
    /* sin(r), |r| <= pi/4 */
    float ps = fmaf(-1.9515295891e-4f, z, 8.3321608736e-3f);
    ps = fmaf(ps, z, -1.6666654611e-1f);
    const float sr = fmaf(ps * z, r, r);
    /* cos(r) */
    float pc = fmaf(2.443315711809948e-5f, z, -1.388731625493765e-3f);
    pc = fmaf(pc, z, 4.166664568298827e-2f);
    const float cr = fmaf(pc * z, z, fmaf(-0.5f, z, 1.0f));
    float ss, cc;
    switch (q & 3)
    {
    case 0: ss = sr; cc = cr; break;
    case 1: ss = cr; cc = -sr; break;
    case 2: ss = -sr; cc = -cr; break;
    default: ss = -cr; cc = sr; break;
    }
    *s = ss;
    *c = cc;
}

ZR_HD float zr_sinf(float x) { float s, c; zr_sincosf(x, &s, &c); return s; }
ZR_HD float zr_cosf(float x) { float s, c; zr_sincosf(x, &s, &c); return c; }

/* ---- exp: x = n ln2 + r, degree-5 polynomial (Cephes expf) ---- */
ZR_HD float zr_expf(float x)
{
    if (x != x) return x;
    if (x > 88.72283905206835f) return zr_u2f(0x7f800000u);
    if (x < -87.33654475055310f) return 0.0f;   /* flush (sub)normal results to zero */
    const float n = rintf(x * 1.44269504088896341f);
    float r = fmaf(-n, 0.693359375f, x);
    r = fmaf(-n, -2.12194440e-4f, r);
    float p = fmaf(1.9875691500e-4f, r, 1.3981999507e-3f);
    p = fmaf(p, r, 8.3334519073e-3f);
    p = fmaf(p, r, 4.1665795894e-2f);
    p = fmaf(p, r, 1.6666665459e-1f);
    p = fmaf(p, r, 5.0000001201e-1f);
    const float e = fmaf(p * r, r, r) + 1.0f;
    /* scale by 2^n in two steps to stay in range */
    const int ni = (int)n;
    const int n1 = ni / 2;
    const int n2 = ni - n1;
    return (e * zr_u2f((uint32_t)(n1 + 127) << 23)) * zr_u2f((uint32_t)(n2 + 127) << 23);
}

/* ---- log: x = 2^e m, m in [sqrt(1/2), sqrt(2)), degree-8 polynomial (Cephes logf) ---- */
ZR_HD float zr_logf(float x)
{
    if (x != x) return x;
    if (x < 0.0f) return zr_u2f(0x7fc00000u);
    if (x == 0.0f) return zr_u2f(0xff800000u);
    if (x == zr_u2f(0x7f800000u)) return x;
    uint32_t u = zr_f2u(x);
    int e = 0;
    if (u < 0x00800000u)        /* subnormal: scale up by 2^23 */
    {
        x = x * 8388608.0f;
        u = zr_f2u(x);
        e = -23;
    }
    e += (int)(u >> 23) - 126;
    float m = zr_u2f((u & 0x007fffffu) | 0x3f000000u);   /* [0.5, 1) */
    if (m < 0.707106781186547524f)
    {
        e -= 1;
        m = (m + m) - 1.0f;
    }
    else
        m = m - 1.0f;
    const float z = m * m;
    float p = fmaf(7.0376836292e-2f, m, -1.1514610310e-1f);
    p = fmaf(p, m, 1.1676998740e-1f);
    p = fmaf(p, m, -1.2420140846e-1f);
    p = fmaf(p, m, 1.4249322787e-1f);
    p = fmaf(p, m, -1.6668057665e-1f);
    p = fmaf(p, m, 2.0000714765e-1f);
    p = fmaf(p, m, -2.4999993993e-1f);
    p = fmaf(p, m, 3.3333331174e-1f);
    float y = (p * m) * z;
    const float fe = (float)e;
    y = fmaf(fe, -2.12194440e-4f, y);
    y = fmaf(-0.5f, z, y);
    return fmaf(fe, 0.693359375f, m + y);
}

/* ---- atan2: octant reduction to t = min/max in [0, 1], t > tan(pi/8) folded to (num-den)/(num+den), degree-5 polynomial in t^2
   (least-squares fit on [0, tan(pi/8)]); pi/4, pi/2 and pi are added as hi + lo pairs so the final subtraction does not lose the last bits.
   IEEE special cases: signed zeros and the axes give +-0, +-pi/2 and +-pi; a NaN gives NaN. ---- */
ZR_HD float zr_atan2f(float y, float x)
{
    if (x != x || y != y) return x + y;
    const float ax = fabsf(x), ay = fabsf(y);
    const float PIO4_HI = 7.8539818525e-01f, PIO4_LO = -2.1855694e-08f;
    const float PIO2_HI = 1.5707963705e+00f, PIO2_LO = -4.3711388e-08f;
    const float PI_HI = 3.1415927410e+00f, PI_LO = -8.7422777e-08f;
    float r;
    if (ax == 0.0f && ay == 0.0f)
        r = 0.0f;
    else if (ax == ay)      /* including both infinite */
        r = PIO4_HI;
    else
    {
        const int swap = ay > ax;
        const float num = swap ? ax : ay, den = swap ? ay : ax;
        float a = num, b = den;
        float off_hi = 0.0f, off_lo = 0.0f;
        if (num > 0.41421356237f * den)
        {
            /* scaling both by 1/4 is exact and keeps num + den finite */
            const float k = den > 1e38f ? 0.25f : 1.0f;
            a = num * k - den * k;
            b = num * k + den * k;
            off_hi = PIO4_HI; off_lo = PIO4_LO;
        }
        const float t = a / b;                      /* 0 when num is finite and den infinite */
        const float t_lo = b > 3.40282347e38f ? 0.0f : fmaf(-t, b, a) / b;      /* the division's rounding error (none when b is infinite) */
        const float z = t * t;
        float p = fmaf(5.055331811e-2f, z, -8.627819270e-2f);
        p = fmaf(p, z, 1.107185036e-1f);
        p = fmaf(p, z, -1.428418159e-1f);
        p = fmaf(p, z, 1.999997795e-1f);
        p = fmaf(p, z, -3.333333433e-1f);
        r = off_hi + ((fmaf(p * z, t, t_lo) + t) + off_lo);
        if (swap) r = PIO2_HI - (r - PIO2_LO);
    }
    if (zr_f2u(x) >> 31) r = PI_HI - (r - PI_LO);
    return (zr_f2u(y) >> 31) ? -r : r;
}

ZR_HD float zr_log2f(float x) { return zr_logf(x) * 1.44269504088896341f; }
ZR_HD float zr_powf(float x, float y) { return zr_expf(y * zr_logf(x)); }

/* ---- binary16 <-> binary32, round-to-nearest-even (== F16C / __float2half_rn) ---- */
ZR_HD uint16_t zr_f32_to_f16(float f)
{
#if defined(__CUDA_ARCH__)
    /* cvt.rn.f16.f32 is the same IEEE round-to-nearest-even conversion (overflow to inf, subnormal halves); only the
       NaN payload rule below is this file's own, so NaNs take the software path */
    if (f == f)
        return __half_as_ushort(__float2half_rn(f));
#endif
    const uint32_t x = zr_f2u(f);
    const uint32_t sign = (x >> 16) & 0x8000u;
    const uint32_t ax = x & 0x7fffffffu;
    if (ax >= 0x7f800000u)          /* inf / nan */
        return (uint16_t)(sign | 0x7c00u | ((ax > 0x7f800000u) ? (0x200u | ((ax >> 13) & 0x3ffu)) : 0u));
    if (ax >= 0x477ff000u)          /* rounds to >= 65520 -> inf */
        return (uint16_t)(sign | 0x7c00u);
    if (ax < 0x33000001u)           /* rounds to zero (<= 2^-25) */
        return (uint16_t)sign;
    if (ax < 0x38800000u)           /* subnormal half */
    {
        const uint32_t exp = ax >> 23;
        const uint32_t man = (ax & 0x007fffffu) | 0x00800000u;
        const uint32_t shift = 126u - exp;           /* 14 .. 24 */
        const uint32_t rem_mask = (1u << shift) - 1u;
        const uint32_t rem = man & rem_mask;
        uint32_t h = man >> shift;
        const uint32_t halfway = 1u << (shift - 1u);
        if (rem > halfway || (rem == halfway && (h & 1u)))
            h += 1u;
        return (uint16_t)(sign | h);
    }
    uint32_t h = ((ax - 0x38000000u) >> 13);
    const uint32_t rem = ax & 0x1fffu;
    if (rem > 0x1000u || (rem == 0x1000u && (h & 1u)))
        h += 1u;
    return (uint16_t)(sign | h);
}

ZR_HD float zr_f16_to_f32(uint16_t h)
{
#if defined(__CUDA_ARCH__)
    if (((uint32_t)h & 0x7c00u) != 0x7c00u)     /* finite: the hardware conversion is exact */
        return __half2float(__ushort_as_half(h));
#endif
    const uint32_t sign = ((uint32_t)h & 0x8000u) << 16;
    const uint32_t exp = ((uint32_t)h >> 10) & 0x1fu;
    uint32_t man = (uint32_t)h & 0x3ffu;
    if (exp == 0x1fu)
        return zr_u2f(sign | 0x7f800000u | (man << 13));
    if (exp == 0)
    {
        if (man == 0)
            return zr_u2f(sign);
        /* normalise subnormal */
        int e = -1;
        do { e++; man <<= 1; } while ((man & 0x400u) == 0);
        return zr_u2f(sign | ((uint32_t)(112 - e) << 23) | ((man & 0x3ffu) << 13));
    }
    return zr_u2f(sign | ((exp + 112u) << 23) | (man << 13));
}

#endif /* ZR_FPMATH_H */
