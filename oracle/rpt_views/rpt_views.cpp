// ORACLE -- test infrastructure, not product code (see orc_math.h header).
//
// The ReSTIR PT debug views (rpt_views_api.h) at the reference's write points, over a frame the oracle (orc_rpt.cpp) rendered.
// The dispatch shapes, lane maps and early-out conditions are restated from the reference shaders:
//   ReSTIR_PT_PathTrace.hlsl   16x8 groups; every valid pixel takes DebugColor(r.rc) (:548), accumulating when Accumulate && CameraStatic
//   Reconnect_TtC.hlsl         16x8 groups, TtC thread map; no temporal history (:175-199), another surface (:240-270) and a history
//                              without a reconnection (:285-297) write black, the rest DebugColor(r_curr.rc) (:383-388)
//   Reconnect_StC.hlsl         8x8 groups, StC thread map; no reusable neighbour (:229-240) and a neighbour without a reconnection
//                              (:258-275) write black, the rest DebugColor(r_curr.rc) (:345-351)
// WriteOutputColor (Util.hlsli:141-160) accumulates when Accumulate && CameraStatic && NumFramesCameraStatic > 1.
#include "rpt_views_api.h"
#include "../orc_rpt.h"
#include "../orc_pixel.h"

using namespace orc;
using namespace orc::RPT;

namespace
{
    // RPT_Util::DebugColor (Util.hlsli:69-139): c is left as it is for NONE and where no branch matches
    void DebugColor(const Reconnection& rc, uint32_t option, float3& c)
    {
        if (option == ZR_RPT_DEBUG_VIEW_NONE)
            return;
        if (option == ZR_RPT_DEBUG_VIEW_K)
        {
            if (rc.Empty()) c = f3(0);
            else if (rc.k == 2) c = f3(0.1f, 0.25f, 0.88f);
            else if (rc.k == 3) c = f3(0.13f, 0.55f, 0.14f);
            else if (rc.k == 4) c = f3(0.69f, 0.45f, 0.1f);
            else if (rc.k >= 5) c = f3(0.88f, 0.08f, 0.1f);
        }
        else if (option == ZR_RPT_DEBUG_VIEW_CASE)
        {
            if (rc.Empty()) c = f3(0);
            else if (rc.IsCase1()) c = f3(0.85f, 0.096f, 0.1f);
            else if (rc.IsCase2()) c = f3(0.13f, 0.6f, 0.14f);
            else if (rc.IsCase3()) c = f3(0.1f, 0.27f, 0.888f);
        }
        else if (option == ZR_RPT_DEBUG_VIEW_FOUND_CONNECTION)
            c = !rc.Empty() ? f3(0.234f, 0.12f, 0.2134f) : f3(0);
        else if (option == ZR_RPT_DEBUG_VIEW_CONNECTION_LOBE_K_MIN_1)
        {
            if (rc.Empty()) c = f3(0);
            else if (rc.lobe_k_min_1 == BSDF::DIFFUSE_R) c = f3(0.384f, 0.12f, 0.2134f);
            else if (rc.lobe_k_min_1 == BSDF::GLOSSY_R) c = f3(0.12f, 0.4284f, 0.2134f);
            else if (rc.lobe_k_min_1 == BSDF::GLOSSY_T) c = f3(0.1134f, 0.12f, 0.634f);
            else if (rc.lobe_k_min_1 == BSDF::DIFFUSE_T) c = f3(0.25f, 0.25f, 0.25f);
            else c = f3(0.55f, 0.55f, 0.0f);
        }
        else if (option == ZR_RPT_DEBUG_VIEW_CONNECTION_LOBE_K)
        {
            if (rc.Empty() || rc.IsCase3()) c = f3(0);
            else if (rc.lobe_k == BSDF::DIFFUSE_R) c = f3(0.384f, 0.12f, 0.2134f);
            else if (rc.lobe_k == BSDF::GLOSSY_R) c = f3(0.12f, 0.284f, 0.2134f);
            else if (rc.lobe_k == BSDF::GLOSSY_T) c = f3(0.1134f, 0.12f, 0.634f);
            else if (rc.lobe_k == BSDF::DIFFUSE_T) c = f3(0.25f, 0.25f, 0.0f);
            else c = f3(0.25f, 0.25f, 0.25f);
        }
    }

    Reconnection RcOf(const zr_rpt_reservoir& rec) { return Reservoir::Load_NonReconnection(rec).rc; }

    // the pixel a dispatch lane works on: group swizzle (Common.hlsli SwizzleThreadGroup), then the sorted thread map (Util.hlsli:32-42)
    bool LanePixel(uint32_t W, uint32_t H, uint32_t Gx, uint32_t Gy, uint32_t GTx, uint32_t GTy, uint32_t gdx, uint32_t gdy, uint32_t dispX,
        uint32_t dispY, bool sorted, const uint16_t* threadMap, int& x, int& y)
    {
        uint32_t sx, sy, sgx, sgy;
        SwizzleThreadGroup(Gx, Gy, GTx, GTy, gdx, gdy, dispX, 16, 4, 16 * dispY, sx, sy, sgx, sgy);
        if (sx >= W || sy >= H) return false;
        x = (int)sx; y = (int)sy;
        if (!sorted) return true;
        const uint16_t enc = threadMap[(size_t)sy * W + sx];
        if (enc & (1u << 15)) return false;
        x += (int)(enc & 0x3f) - 31;
        y += (int)((enc >> 7) & 0x3f) - 31;
        return true;
    }

    // Reconnect_TtC.hlsl:166-265: is there a temporal history on the same surface?
    bool TemporalHistory(const Frame& f, int x, int y, int& ppx, int& ppy)
    {
        const float2 renderDim = f2((float)f.W, (float)f.H);
        const float2 motionVec = unpack_snorm16x2(f.me[(size_t)y * f.W + x].x);
        const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / renderDim;
        const float2 prevUV = currUV - motionVec;
        const float2 pp = prevUV * renderDim;
        ppx = (int)pp.x; ppy = (int)pp.y;
        if (prevUV.x < 0.0f || prevUV.y < 0.0f || prevUV.x > 1.0f || prevUV.y > 1.0f)
            return false;
        if (asfloat(f.pcore[(size_t)ppy * f.W + ppx].x) == FLT_MAX_)
            return false;
        const Pixel cur = LoadPixel(f, f.core, f.coat, x, y, false, x, y);
        const Pixel prev = LoadPixel(f, f.pcore, f.pcoat, ppx, ppy, true, x, y);
        if (!(fabsf(dot(cur.normal, prev.pos - cur.pos)) <= 1.0f * cur.z))
            return false;
        return !(prev.flags.emissive || fabsf(prev.roughness - cur.roughness) > 0.3f || prev.flags.transmissive != cur.flags.transmissive);
    }
}

extern "C"
{
    void rptv_debug_color(uint32_t view, const uint32_t* meta, const float* li, uint32_t n, float* out)
    {
        for (uint32_t i = 0; i < n; i++)
        {
            Reservoir r = Reservoir::Init();
            r.UnpackMetadata(meta[i]);
            float3 c = f3(li[3 * i], li[3 * i + 1], li[3 * i + 2]);
            DebugColor(r.rc, view, c);
            out[3 * i] = c.x; out[3 * i + 1] = c.y; out[3 * i + 2] = c.z;
        }
    }

    void rptv_write_point(void* scene, const zr_frame_constants* fc, const uint32_t* core, const uint32_t* me, const uint32_t* coat,
        const uint32_t* pcore, const uint32_t* pcoat, uint32_t stage, uint32_t view, uint32_t sorted, const zr_rpt_reservoir* res_out,
        const zr_rpt_reservoir* res_gate, const uint16_t* neighbor, const uint16_t* thread_map, const float* before, float* final_img)
    {
        Frame f;
        f.sc = (const Scene*)scene; f.fc = fc;
        f.core = (const uint4*)core; f.me = (const uint2*)me; f.coat = (const uint2*)coat;
        f.pcore = (const uint4*)pcore; f.pcoat = (const uint2*)pcoat;
        f.W = fc->RenderWidth; f.H = fc->RenderHeight;
        const uint32_t gd = stage == RPTV_STC ? 8 : 16, gdy = 8;
        const uint32_t dispX = (f.W + gd - 1) / gd, dispY = (f.H + gdy - 1) / gdy;
        const bool accumulate = fc->Accumulate && fc->CameraStatic && (stage == RPTV_PATHTRACE || fc->NumFramesCameraStatic > 1);
        for (uint32_t g = 0; g < dispX * dispY; g++)
            for (uint32_t t = 0; t < gd * gdy; t++)
            {
                int x, y;
                if (!LanePixel(f.W, f.H, g % dispX, g / dispX, t % gd, t / gd, gd, gdy, dispX, dispY, stage != RPTV_PATHTRACE && sorted,
                        thread_map, x, y))
                    continue;
                const GFlags flags = FlagsAt(f.core, f.W, x, y);
                if (flags.invalid || flags.emissive)
                    continue;
                const size_t idx = (size_t)y * f.W + x;
                bool colour = true;
                if (stage == RPTV_TTC)
                {
                    int ppx = 0, ppy = 0;
                    colour = TemporalHistory(f, x, y, ppx, ppy) && !RcOf(res_gate[(size_t)ppy * f.W + ppx]).Empty();
                }
                else if (stage == RPTV_STC)
                {
                    const uint16_t nb = neighbor[idx];
                    const int ox = nb & 0xff, oy = nb >> 8;
                    colour = ox != 0xff && !RcOf(res_gate[(size_t)(y + oy - 32) * f.W + (x + ox - 32)]).Empty();
                }
                // DebugColor over li = target * W: every non-empty reconnection of a record (k >= 2, one of the three cases) takes a
                // branch, so the colour never depends on li
                float3 c = f3(0);
                if (colour)
                    DebugColor(RcOf(res_out[idx]), view, c);
                float* o = final_img + 4 * idx;
                const float* p = before + 4 * idx;
                o[0] = accumulate ? p[0] + c.x : c.x;
                o[1] = accumulate ? p[1] + c.y : c.y;
                o[2] = accumulate ? p[2] + c.z : c.z;
            }
    }
}
