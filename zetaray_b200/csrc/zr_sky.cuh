// zr_sky.cuh -- the atmosphere and the sky it shows: single-scattering sky-view LUT texels, the LUT lookup and the sky with its sun
// disk behind geometry. Shared by k_sky_view_lut (sky.cu), the sky branches of compositing (post.cu) and DirectLighting's
// accumulating frames (rdi.cu); tests/hostsim compiles it for the host.
//
// Restates Common/Volumetric.hlsli (densities, ray-sphere tests, EstimateTransmittance, EstimateLs, phase functions),
// Math::SphericalToCartesian / SphericalFromCartesian (Math.hlsli:115-134), Sky/SkyViewLUT.hlsl:19-54, Light::Le_Sky and
// Light::Le_SkyWithSunDisk (Common/LightSource.hlsli:158-199). Numerics (DESIGN §2): mad / dot are fmaf chains, every other
// product and sum is rounded on its own in HLSL text order, sin / cos / exp / atan2 come from zr_fpmath.h. Distances are in km.
#pragma once
#include "zr_common.cuh"

namespace zr
{
namespace Sky
{
    constexpr float ONE_OVER_4_PI = 0.079577472f;

    // ---- Volume:: (Volumetric.hlsli) ----
    ZR_D float RayleighPhaseFunction(float cosTheta) { return 0.0596831f * (1.0f + cosTheta * cosTheta); }
    ZR_D float SchlickPhaseFunction(float cosTheta, float g)
    {
        const float k = 1.55f * g - 0.55f * g * g * g;
        const float denom = 1.0f - k * cosTheta;
        return ONE_OVER_4_PI * (1.0f - k * k) / (denom * denom);
    }
    ZR_D float DensityRayleigh(float altitude) { return zr_expf(-fmaxf(0.0f, altitude / 8.0f)); }
    ZR_D float DensityMie(float altitude) { return zr_expf(-fmaxf(0.0f, altitude / 1.2f)); }
    ZR_D float DensityOzone(float altitude) { return fmaxf(0.0f, 1.0f - fabsf(altitude - 25.0f) / 15.0f); }
    ZR_D float3 AtmosphereDensity(float altitude) { return f3(DensityRayleigh(altitude), DensityMie(altitude), DensityOzone(altitude)); }
    ZR_D float Altitude(float3 pos, float planetRadius) { return length(pos) - planetRadius; }

    // the ray starts inside the sphere: the positive root
    ZR_D float IntersectRayAtmosphere(float radius, float3 rayOrigin, float3 rayDir)
    {
        const float mDotdir = dot(rayDir, rayOrigin);
        float delta = mDotdir * mDotdir - dot(rayOrigin, rayOrigin) + radius * radius;
        delta = sqrtf(delta);
        return -mDotdir + delta;
    }
    // the ray starts outside the sphere: the nearer root, a hit when it is >= 0
    ZR_D bool IntersectRayPlanet(float radius, float3 rayOrigin, float3 rayDir, float& t)
    {
        const float mDotdir = dot(rayDir, rayOrigin);
        float delta = mDotdir * mDotdir - dot(rayOrigin, rayOrigin) + radius * radius;
        if (delta < 0.0f)
        {
            t = 0.0f;
            return false;
        }
        delta = sqrtf(delta);
        t = fminf(-mDotdir - delta, -mDotdir + delta);
        return t >= 0.0f;
    }

    // optical thickness by the midpoint rule over numSteps segments
    ZR_D float3 EstimateTransmittance(float planetRadius, float3 rayOrigin, float3 rayDir, float t, float3 sigma_t_rayleigh,
        float sigma_t_mie, float3 sigma_t_ozone, int numSteps)
    {
        if (t <= 1e-5f)
            return f3(1.0f);
        const float stepSize = t / (float)numSteps;
        float3 pos = rayOrigin + 0.5f * stepSize * rayDir;
        float3 opticalThickness = f3(0.0f);
        for (int s = 0; s < numSteps; s++)
        {
            const float3 density = AtmosphereDensity(Altitude(pos, planetRadius));
            opticalThickness += density;
            pos += stepSize * rayDir;
        }
        opticalThickness = sigma_t_rayleigh * opticalThickness.x + sigma_t_mie * opticalThickness.y + sigma_t_ozone * opticalThickness.z;
        opticalThickness *= stepSize;
        return f3(zr_expf(-opticalThickness.x), zr_expf(-opticalThickness.y), zr_expf(-opticalThickness.z));
    }

    // light of the sun scattered once towards the ray origin (Rayleigh + Mie), numSteps midpoint segments
    ZR_D float3 EstimateLs(float planetRadius, float3 rayOrigin, float3 rayDir, float3 lightDir, float atmosphereHeight, float g,
        float3 sigma_s_rayleigh, float sigma_s_mie, float sigma_t_mie, float3 sigma_t_ozone, int numSteps)
    {
        float t = IntersectRayAtmosphere(planetRadius + atmosphereHeight, rayOrigin, rayDir);
        float tPlanet;
        if (IntersectRayPlanet(planetRadius, rayOrigin, rayDir, tPlanet))
            t = tPlanet;
        const float stepSize = t / (float)numSteps;
        float3 pos = rayOrigin + 0.5f * stepSize * rayDir;
        float3 opticalThickness = f3(0.0f);
        float3 LsRayleigh = f3(0.0f);
        float3 LsMie = f3(0.0f);
        for (int s = 0; s < numSteps; s++)
        {
            const float3 density = AtmosphereDensity(Altitude(pos, planetRadius));
            opticalThickness += density * stepSize;
            const float3 e = sigma_s_rayleigh * opticalThickness.x + sigma_t_mie * opticalThickness.y + sigma_t_ozone * opticalThickness.z;
            const float3 rayOriginToPosTr = f3(zr_expf(-e.x), zr_expf(-e.y), zr_expf(-e.z));
            const float posToAtmosphereDist = IntersectRayAtmosphere(planetRadius + atmosphereHeight, pos, -lightDir);
            const float3 LoTransmittance = EstimateTransmittance(planetRadius, pos, -lightDir, posToAtmosphereDist, sigma_s_rayleigh,
                sigma_t_mie, sigma_t_ozone, 8);
            LsRayleigh += rayOriginToPosTr * density.x * LoTransmittance;
            LsMie += rayOriginToPosTr * density.y * LoTransmittance;
            pos += stepSize * rayDir;
        }
        const float cosTheta = dot(lightDir, -rayDir);
        const float phaseRayleigh = RayleighPhaseFunction(cosTheta);
        const float phaseMie = SchlickPhaseFunction(cosTheta, g);
        float3 Ls = LsRayleigh * sigma_s_rayleigh * phaseRayleigh;
        Ls += LsMie * sigma_s_mie * phaseMie;
        Ls *= stepSize;
        return Ls;
    }

    // ---- Math:: (Math.hlsli:115-134); y is up, phi is measured clockwise from +x ----
    ZR_D float3 SphericalToCartesian(float r, float theta, float phi)
    {
        const float sinTheta = zr_sinf(theta);
        return f3(r * sinTheta * zr_cosf(phi), r * zr_cosf(theta), -r * sinTheta * zr_sinf(phi));
    }
    ZR_D float2 SphericalFromCartesian(float3 w)
    {
        float2 thetaPhi;
        thetaPhi.x = Math::ArcCos(w.y);
        thetaPhi.y = zr_atan2f(-w.z, w.x);
        thetaPhi.y = thetaPhi.y < 0 ? thetaPhi.y + TWO_PI : thetaPhi.y;
        return thetaPhi;
    }

    ZR_D float3 Vec3(const float v[3]) { return f3(v[0], v[1], v[2]); }

    // SkyViewLUT.hlsl main: texel (x, y) of a lutW x lutH LUT, before R11G11B10 storage. Latitude is mapped non-linearly so that more
    // texels lie near the horizon: theta = pi/2 +- 2 pi (v - 1/2)^2.
    ZR_D float3 SkyViewTexel(const zr_frame_constants& fc, uint32_t x, uint32_t y, uint32_t lutW, uint32_t lutH)
    {
        float phi = (float)x / (float)lutW;
        phi *= TWO_PI;
        const float v = (float)y / (float)lutH;
        const float s = v >= 0.5f ? 1.0f : -1.0f;
        const float a = v - 0.5f;
        const float theta = a * a * TWO_PI * s + PI_OVER_2;
        const float3 w = SphericalToCartesian(1.0f, theta, phi);
        const float3 sigma_s_rayleigh = Vec3(fc.RayleighSigmaSColor) * fc.RayleighSigmaSScale;
        const float sigma_t_mie = fc.MieSigmaA + fc.MieSigmaS;
        const float3 sigma_t_ozone = Vec3(fc.OzoneSigmaAColor) * fc.OzoneSigmaAScale;
        const float3 rayOrigin = f3(0.0f, fc.PlanetRadius + 0.2f, 0.0f);
        float3 Ls = EstimateLs(fc.PlanetRadius, rayOrigin, w, Vec3(fc.SunDir), fc.AtmosphereAltitude, fc.g, sigma_s_rayleigh,
            fc.MieSigmaS, sigma_t_mie, sigma_t_ozone, 32);
        Ls *= fc.SunIlluminance;
        return f3(fmaxf(0.0f, Ls.x), fmaxf(0.0f, Ls.y), fmaxf(0.0f, Ls.z));
    }

    // The LUT as compositing and DirectLighting read it: R11G11B10F texels, row-major, lutW x lutH
    struct LutView
    {
        const uint32_t* texels;
        uint32_t w, h;
    };

    // SampleLevel(g_samLinearWrap, uv, 0): bilinear at texel-centre mapping, wrap on both axes, float weights
    ZR_D float3 SampleLinearWrap(const LutView& lut, float2 uv)
    {
        const float tx = uv.x * (float)lut.w - 0.5f, ty = uv.y * (float)lut.h - 0.5f;
        const float fx0 = floorf(tx), fy0 = floorf(ty);
        const float fx = tx - fx0, fy = ty - fy0;
        const int W = (int)lut.w, H = (int)lut.h;
        int x0 = (int)fx0 % W, y0 = (int)fy0 % H;
        x0 = x0 < 0 ? x0 + W : x0;
        y0 = y0 < 0 ? y0 + H : y0;
        const int x1 = x0 + 1 == W ? 0 : x0 + 1, y1 = y0 + 1 == H ? 0 : y0 + 1;
        const float3 c00 = unpack_r11g11b10(__ldg(&lut.texels[(size_t)y0 * W + x0]));
        const float3 c10 = unpack_r11g11b10(__ldg(&lut.texels[(size_t)y0 * W + x1]));
        const float3 c01 = unpack_r11g11b10(__ldg(&lut.texels[(size_t)y1 * W + x0]));
        const float3 c11 = unpack_r11g11b10(__ldg(&lut.texels[(size_t)y1 * W + x1]));
        const float w00 = (1.0f - fx) * (1.0f - fy), w10 = fx * (1.0f - fy), w01 = (1.0f - fx) * fy, w11 = fx * fy;
        return c00 * w00 + c10 * w10 + c01 * w01 + c11 * w11;
    }

    // Light::Le_Sky: the LUT in direction wi, through the inverse of the latitude map
    ZR_D float3 Le_Sky(float3 wi, const LutView& lut)
    {
        const float2 thetaPhi = SphericalFromCartesian(wi);
        float2 uv = f2(thetaPhi.y * ONE_OVER_2_PI, thetaPhi.x * ONE_OVER_PI);
        const float sn = thetaPhi.x >= PI_OVER_2 ? 1.0f : -1.0f;
        uv.y = mad(0.5f, thetaPhi.x, -PI_OVER_4);
        uv.y = 0.5f + sn * sqrtf(fabsf(uv.y) * ONE_OVER_PI);
        return SampleLinearWrap(lut, uv);
    }

    // Light::Le_SkyWithSunDisk: pixel (x, y)'s pinhole camera ray (jitter included; the thin lens is not used here) shows the sun
    // disk where it is within the sun's angular radius and the disk's lower edge is above the horizon, else the sky
    ZR_D float3 Le_SkyWithSunDisk(const zr_frame_constants& fc, const LutView& lut, uint32_t x, uint32_t y)
    {
        const float2 renderDim = f2((float)fc.RenderWidth, (float)fc.RenderHeight);
        const float2 jitter = f2(fc.CurrCameraJitter[0], fc.CurrCameraJitter[1]);
        const float2 uv = (f2((float)x, (float)y) + 0.5f + jitter) / renderDim;
        const float2 ndc = Math::NDCFromUV(uv);
        const float3 dirV = f3(ndc.x * fc.AspectRatio * fc.TanHalfFOV, ndc.y * fc.TanHalfFOV, 1.0f);
        const float3 bx = f3(fc.CurrView[0][0], fc.CurrView[0][1], fc.CurrView[0][2]);
        const float3 by = f3(fc.CurrView[1][0], fc.CurrView[1][1], fc.CurrView[1][2]);
        const float3 bz = f3(fc.CurrView[2][0], fc.CurrView[2][1], fc.CurrView[2][2]);
        const float3 wc = normalize(mad(dirV.x, bx, mad(dirV.y, by, dirV.z * bz)));

        float3 rayOrigin = f3(0.0f, 1e-1f, 0.0f);
        rayOrigin.y += fc.PlanetRadius;
        float3 wTemp = wc;
        // cos(a - b) = cos a cos b + sin a sin b
        wTemp.y = wTemp.y * fc.SunCosAngularRadius + sqrtf(1.0f - wc.y * wc.y) * fc.SunSinAngularRadius;
        float t;
        const bool intersectedPlanet = IntersectRayPlanet(fc.PlanetRadius, rayOrigin, wTemp, t);
        if (dot(-wc, Vec3(fc.SunDir)) >= fc.SunCosAngularRadius && !intersectedPlanet)
            return f3(fc.SunIlluminance);
        return Le_Sky(wc, lut);
    }

    // Host: the LUT image a set_sky entry point was given, as a LutView. NULL turns the sky off (view.texels = NULL); anything but a
    // non-empty, unpadded 4-byte-texel image is refused.
    inline zr_status ViewOf(const char* fn, const zr_image2d* img, LutView& view)
    {
        view = LutView{ nullptr, 0, 0 };
        if (!img) return ZR_OK;
        if (!img->d_ptr || !img->width || !img->height || img->texel_bytes != 4 || img->pitch_bytes != img->width * 4u)
        {
            set_error("%s: the sky-view LUT must be a non-empty R11G11B10F image (4-byte texels, pitch = 4 * width)", fn);
            return ZR_ERR_INVALID_ARG;
        }
        view = LutView{ (const uint32_t*)img->d_ptr, img->width, img->height };
        return ZR_OK;
    }
}
} // namespace zr
