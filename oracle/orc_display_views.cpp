// ORACLE -- test infrastructure, not product code (see orc_math.h header).
//
// CPU restatement of the editor side of the Display and G-buffer passes:
//   pick           GBufferRT_Inline.hlsl:241-242 (hitMeshIdx under the picked pixel), the camera ray of orc_gbuffer
//   debug views    Display/Display.hlsl:53-170 (DisplayOption != DEFAULT) and the R8G8B8A8_UNORM_SRGB store
//   pick mask      Display.cpp:293-400 + DrawPicked.hlsl: the picked instance's triangles, clipped at CameraNear, projected with
//                  the inverse of the G-buffer's camera-ray mapping, pixel centres inside under the D3D top-left rule
//   outline        Sobel.hlsl:27-105, for each bit of the mask
// DESIGN 6b states the rasteriser's rules; the device kernels are csrc/display.cu and csrc/gbuffer.cu.
#include "orc_api.h"
#include "orc_scene.h"

using namespace orc;

namespace
{
    constexpr uint32_t VIEW_BASE_COLOR = 1, VIEW_NORMAL = 2, VIEW_METALNESS_ROUGHNESS = 3, VIEW_COAT_WEIGHT = 4, VIEW_COAT_COLOR = 5,
                       VIEW_ROUGHNESS_TH = 6, VIEW_EMISSIVE = 7, VIEW_TRANSMISSION = 8, VIEW_DEPTH = 9;

    float Oetf(float v) { return v <= 0.0031308f ? 12.92f * v : 1.055f * zr_powf(v, 1.0f / 2.4f) - 0.055f; }
    uint32_t Srgb8(float3 c)
    {
        c = saturate(c);
        return Math::FloatToUNorm8(Oetf(c.x)) | Math::FloatToUNorm8(Oetf(c.y)) << 8 | Math::FloatToUNorm8(Oetf(c.z)) << 16;
    }

    int ClipNear(const float3 v[3], float nearZ, float3 out[4])
    {
        int n = 0;
        for (int e = 0; e < 3; e++)
        {
            const float3 a = v[e], b = v[(e + 1) % 3];
            const bool ina = a.z >= nearZ, inb = b.z >= nearZ;
            if (ina)
                out[n++] = a;
            if (ina != inb)
            {
                // from the inside vertex: both triangles of a shared edge clip it to the same point
                const float3 p = ina ? a : b, q = ina ? b : a;
                const float t = (nearZ - p.z) / (q.z - p.z);
                out[n++] = f3(p.x + t * (q.x - p.x), p.y + t * (q.y - p.y), nearZ);
            }
        }
        return n;
    }

    float2 ProjectToPixel(float3 p, const zr_frame_constants& fc)
    {
        const float2 ndc = f2(p.x / p.z / fc.TanHalfFOV / fc.AspectRatio, p.y / p.z / fc.TanHalfFOV);
        const float2 uv = Math::UVFromNDC(ndc);
        return f2(uv.x * (float)fc.RenderWidth - fc.CurrCameraJitter[0], uv.y * (float)fc.RenderHeight - fc.CurrCameraJitter[1]);
    }

    float EdgeFn(float2 a, float2 b, float2 p)
    {
        const bool swap = b.y < a.y || (b.y == a.y && b.x < a.x);
        const float2 s = swap ? b : a, t = swap ? a : b;
        const float e = (t.x - s.x) * (p.y - s.y) - (t.y - s.y) * (p.x - s.x);
        return swap ? -e : e;
    }
    bool EdgeIn(float2 a, float2 b, float2 p)
    {
        const float e = EdgeFn(a, b, p);
        return e > 0.0f || (e == 0.0f && (b.y < a.y || (b.y == a.y && b.x > a.x)));
    }
    bool InTriangle(float2 a, float2 b, float2 c, float2 p)
    {
        const float area = EdgeFn(a, b, c);
        if (area == 0.0f)
            return false;
        if (area < 0.0f)
            std::swap(b, c);
        return EdgeIn(a, b, p) && EdgeIn(b, c, p) && EdgeIn(c, a, p);
    }

    // screen-space polygon (3 or 4 vertices) over rows [y0, y1): fn(pixel index) per covered pixel
    template<typename Fn>
    void RasterPolygon(const float2* s, int n, uint32_t W, uint32_t y0, uint32_t y1, Fn fn)
    {
        float x0 = FLT_MAX_, x1 = -FLT_MAX_, ya = FLT_MAX_, yb = -FLT_MAX_;
        for (int j = 0; j < n; j++)
        {
            x0 = fminf(x0, s[j].x); x1 = fmaxf(x1, s[j].x); ya = fminf(ya, s[j].y); yb = fmaxf(yb, s[j].y);
        }
        const float xs = fmaxf(ceilf(x0 - 0.5f), 0.0f), xe = fminf(floorf(x1 - 0.5f), (float)W - 1.0f);
        const float ys = fmaxf(ceilf(ya - 0.5f), (float)y0), ye = fminf(floorf(yb - 0.5f), (float)y1 - 1.0f);
        if (!(xs <= xe && ys <= ye))
            return;
        for (uint32_t y = (uint32_t)ys; y <= (uint32_t)ye; y++)
            for (uint32_t x = (uint32_t)xs; x <= (uint32_t)xe; x++)
            {
                const float2 p = f2((float)x + 0.5f, (float)y + 0.5f);
                if (InTriangle(s[0], s[1], s[2], p) || (n == 4 && InTriangle(s[0], s[2], s[3], p)))
                    fn((size_t)y * W + x);
            }
    }

    // a view-space triangle: clip, project, rasterise
    template<typename Fn>
    void RasterViewTri(const float3 v[3], const zr_frame_constants& fc, uint32_t y0, uint32_t y1, Fn fn)
    {
        float3 c[4];
        const int n = ClipNear(v, fc.CameraNear, c);
        if (n < 3)
            return;
        float2 s[4];
        for (int j = 0; j < n; j++)
            s[j] = ProjectToPixel(c[j], fc);
        RasterPolygon(s, n, fc.RenderWidth, y0, y1, fn);
    }
}

extern "C"
{
    // GBufferRT::PickPixel answered by one render: the instance under pixel (x, y), 0xffffffff for a miss or a pixel outside the frame
    uint32_t orc_gbuffer_pick(void* scene_, const zr_frame_constants* fc, uint32_t x, uint32_t y)
    {
        const Scene& sc = *(const Scene*)scene_;
        const uint32_t W = fc->RenderWidth, H = fc->RenderHeight;
        if (x >= W || y >= H)
            return 0xffffffffu;
        const float2 renderDim = f2((float)W, (float)H);
        const float2 jitter = f2(fc->CurrCameraJitter[0], fc->CurrCameraJitter[1]);
        const float2 uv = (f2((float)x, (float)y) + 0.5f + jitter) / renderDim;
        const float2 ndc = Math::NDCFromUV(uv);
        float3 rayDirCS = f3(ndc.x * fc->AspectRatio * fc->TanHalfFOV, ndc.y * fc->TanHalfFOV, 1);
        float3 rayOrigin = f3(fc->CameraPos[0], fc->CameraPos[1], fc->CameraPos[2]);
        const float3 bx = f3(fc->CurrView[0][0], fc->CurrView[0][1], fc->CurrView[0][2]);
        const float3 by = f3(fc->CurrView[1][0], fc->CurrView[1][1], fc->CurrView[1][2]);
        const float3 bz = f3(fc->CurrView[2][0], fc->CurrView[2][1], fc->CurrView[2][2]);
        if (fc->DoF)
        {
            const uint3 h = RNG::PCG3d(uint3{ x, y, x });
            RNG rng = RNG::Init(h.z, h.y, fc->FrameNum);
            const float2 lensSample = Sampling::UniformSampleDiskConcentric(rng.Uniform2D()) * fc->LensRadius;
            rayOrigin += mad(lensSample.x, bx, lensSample.y * by);
            const float3 focalPoint = fc->FocusDepth * rayDirCS;
            rayDirCS = focalPoint - f3(lensSample.x, lensSample.y, 0);
        }
        const float3 rayDir = normalize(mad(rayDirCS.x, bx, mad(rayDirCS.y, by, rayDirCS.z * bz)));
        const RayHit h = sc.Closest(rayOrigin, rayDir, 0.0f, FLT_MAX_);
        return h.hit ? sc.triMesh[h.tri] : 0xffffffffu;
    }

    // Display.hlsl:53-170 over rows [y0, y1) of a W-wide G-buffer (core uint4, me uint2, coat uint2) -> RGBA8
    void orc_display_view(const uint32_t* core_, const uint32_t* me_, const uint32_t* coat_, uint32_t W, uint32_t y0, uint32_t y1, uint32_t view,
        float roughnessTh, float cameraNear, uint32_t* out)
    {
        const uint4* core = (const uint4*)core_;
        const uint2* me = (const uint2*)me_;
        const uint2* coat = (const uint2*)coat_;
        for (size_t i = (size_t)y0 * W; i < (size_t)y1 * W; i++)
        {
            const uint4 c = core[i];
            const float z = asfloat(c.x);
            if (z == FLT_MAX_)
            {
                out[i] = 0u;
                continue;
            }
            const bool transmissive = c.w & 1u, emissive = (c.w >> 1) & 1u, coated = (c.w >> 5) & 1u, metallic = (c.w >> 7) & 1u;
            const float roughness = Math::UNorm8ToFloat((c.w >> 8) & 0xff);
            const float3 baseColor = Math::UnpackRGB8(c.z & 0xffffff);
            float3 d = f3(0.0f);
            if (view == VIEW_BASE_COLOR)
                d = baseColor;
            else if (view == VIEW_NORMAL)
                d = Math::DecodeUnitVector(Math::DecodeUNorm2(c.y)) * 0.5f + 0.5f;
            else if (view == VIEW_METALNESS_ROUGHNESS)
                d = f3(metallic ? 1.0f : 0.0f, roughness, 0.0f);
            else if ((view == VIEW_COAT_WEIGHT || view == VIEW_COAT_COLOR) && coated)
            {
                const uint32_t px = coat[i].x & 0xffff, py = coat[i].x >> 16;
                d = view == VIEW_COAT_WEIGHT ? f3(Math::UNorm8ToFloat((py >> 8) & 0xff)) : Math::UnpackRGB8(px | ((py & 0xff) << 16));
            }
            else if (view == VIEW_ROUGHNESS_TH)
                d = roughness >= roughnessTh ? f3(0.26f, 0.014f, 0.021f) : f3(0.0f);
            else if (view == VIEW_EMISSIVE)
                d = emissive ? unpack_r11g11b10(me[i].y) : baseColor * 0.005f;
            else if (view == VIEW_TRANSMISSION)
                d = f3(transmissive ? 1.0f : 0.0f, transmissive ? 0.0f : 1.0f, 0.0f);
            else if (view == VIEW_DEPTH)
                d = f3(cameraNear / z);
            out[i] = Srgb8(d) | 0xff000000u;
        }
    }

    // The rasteriser alone on world-space triangles (n x 9 floats), rows [y0, y1) of the frame fc describes. count_mode != 0:
    // out[pixel] += 1 per covering triangle; else out[pixel] |= bit.
    void orc_raster_world_tris(const float* tris, uint32_t n, const zr_frame_constants* fc, uint32_t y0, uint32_t y1, int count_mode,
        uint32_t bit, uint32_t* out)
    {
        for (uint32_t t = 0; t < n; t++)
        {
            float3 v[3];
            for (int j = 0; j < 3; j++)
                v[j] = Math::mul3x4(fc->CurrView, f3(tris[9 * t + 3 * j], tris[9 * t + 3 * j + 1], tris[9 * t + 3 * j + 2]));
            RasterViewTri(v, *fc, y0, y1, [&](size_t i) { if (count_mode) out[i] += 1; else out[i] |= bit; });
        }
    }

    // The coverage rule alone on pixel-space triangles (n x 6 floats) of a W x H frame: out[pixel] += 1 per covering triangle
    void orc_raster_pixel_tris(const float* tris, uint32_t n, uint32_t W, uint32_t H, uint32_t* out)
    {
        for (uint32_t t = 0; t < n; t++)
        {
            const float2 s[3] = { f2(tris[6 * t], tris[6 * t + 1]), f2(tris[6 * t + 2], tris[6 * t + 3]), f2(tris[6 * t + 4], tris[6 * t + 5]) };
            RasterPolygon(s, 3, W, 0, H, [&](size_t i) { out[i] += 1; });
        }
    }

    // k_pick_mask: picked instance k -> bit k over rows [y0, y1) of mask (W x H uint32, cleared by the caller)
    void orc_pick_mask(void* scene_, const zr_frame_constants* fc, const uint32_t* inst, uint32_t n, uint32_t y0, uint32_t y1, uint32_t* mask)
    {
        const Scene& sc = *(const Scene*)scene_;
        for (uint32_t k = 0; k < n; k++)
        {
            const uint32_t m = inst[k];
            const zr_mesh_instance& md = sc.instances[m];
            const uint32_t first = sc.meshFirstTri[m];
            const uint32_t numTris = (m + 1 < sc.numInstances ? sc.meshFirstTri[m + 1] : (uint32_t)sc.triMesh.size()) - first;
            const float4 q = normalize(Math::DecodeNormalized4(md.Rotation));
            const float3 scale = Scene::h3(md.Scale);
            const float3 translation = f3(md.Translation[0], md.Translation[1], md.Translation[2]);
            for (uint32_t prim = 0; prim < numTris; prim++)
            {
                float3 v[3];
                for (int j = 0; j < 3; j++)
                {
                    const zr_vertex& V = sc.vertices[sc.indices[prim * 3 + md.BaseIdxOffset + j] + md.BaseVtxOffset];
                    v[j] = Math::mul3x4(fc->CurrView, Math::TransformTRS(f3(V.pos[0], V.pos[1], V.pos[2]), translation, q, scale));
                }
                RasterViewTri(v, *fc, y0, y1, [&](size_t i) { mask[i] |= 1u << k; });
            }
        }
    }

    // k_outline over rows [y0, y1): out (RGBA8) takes the outline colour where some bit k of the W x H mask is in the in-frame 3 x 3
    // neighbourhood and its Sobel gradient (taps outside the frame read 0) is non-zero
    void orc_outline(const uint32_t* mask, uint32_t W, uint32_t H, uint32_t y0, uint32_t y1, uint32_t* out)
    {
        for (uint32_t y = y0; y < y1; y++)
            for (uint32_t x = 0; x < W; x++)
            {
                uint32_t m[3][3];
                uint32_t any = 0;
                for (int r = 0; r < 3; r++)
                    for (int c = 0; c < 3; c++)
                    {
                        const int xx = (int)x - 1 + c, yy = (int)y - 1 + r;
                        m[r][c] = xx >= 0 && xx < (int)W && yy >= 0 && yy < (int)H ? mask[(size_t)yy * W + xx] : 0u;
                        any |= m[r][c];
                    }
                for (uint32_t k = 0; k < 32; k++)
                {
                    if (!((any >> k) & 1u))
                        continue;
                    auto t = [&](int r, int c) { return (float)((m[r][c] >> k) & 1u); };
                    const float gx = -1.0f * t(0, 0) - 2.0f * t(1, 0) - 1.0f * t(2, 0) + 1.0f * t(0, 2) + 2.0f * t(1, 2) + 1.0f * t(2, 2);
                    const float gy = 1.0f * t(0, 0) + 2.0f * t(0, 1) + 1.0f * t(0, 2) - 1.0f * t(2, 0) - 2.0f * t(2, 1) - 1.0f * t(2, 2);
                    const float g = sqrtf(gx * gx + gy * gy);
                    if (Math::Luminance(f3(g)) > 0.0f)
                    {
                        out[(size_t)y * W + x] = Srgb8(f3(0.913098693f, 0.332451582f, 0.048171822f)) | 0xff000000u;
                        break;
                    }
                }
            }
    }
}
