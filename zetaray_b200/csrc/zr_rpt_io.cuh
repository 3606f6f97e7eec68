// zr_rpt_io.cuh -- ReSTIR PT per-pixel I/O shared by path generation (rpt.cu) and the queued reuse passes
// (rpt_temporal.cu, rpt_spatial.cu): kernel parameter block, 128-bit record accesses, neighbour lookup, the boiling-suppression rule
// (ReSTIR_PT/Util.hlsli:58-67) and the "reservoir did not change" copy of Reconnect_StC (ReSTIR_PT_Reconnect_StC.hlsl:83-106).
#pragma once
#include "zr_rpt.cuh"
#include "zr_pixel.cuh"

namespace zr
{
struct RptParams
{
    uint32_t maxNonTrBounces, maxGlossyTrBounces, russianRoulette, M_max_temporal, M_max_spatial;
    uint32_t boilingSuppression, sortSpatial;
    float alpha_min;
    uint32_t temporalResample, resetTemporal, spatialFlag;
    uint32_t rowBegin, rowEnd;      // rows this rank owns (multi-GPU); whole image by default
    unsigned long long* costMap;    // optional: SM cycles spent per 32x32-pixel tile ((W + 31) / 32 per row)
};

namespace
{
    using namespace RPT;

    ZR_D void LoadRecord(const zr_rpt_reservoir* __restrict__ p, zr_rpt_reservoir& r)
    {
        const uint4* q = reinterpret_cast<const uint4*>(p);
        uint4 v[4] = { q[0], q[1], q[2], q[3] };
        memcpy(&r, v, 64);
    }
    ZR_D void StoreRecord(zr_rpt_reservoir* __restrict__ p, const zr_rpt_reservoir& r)
    {
        uint4 v[4];
        memcpy(v, &r, 64);
        uint4* q = reinterpret_cast<uint4*>(p);
        q[0] = v[0]; q[1] = v[1]; q[2] = v[2]; q[3] = v[3];
    }
    ZR_D uint4 LoadQ0(const zr_rpt_reservoir* __restrict__ p) { return *reinterpret_cast<const uint4*>(p); }

    ZR_D bool NeighborOf(const FrameView& f, const uint16_t* __restrict__ neighbor, int x, int y, int& nx, int& ny)
    {
        const uint16_t nb = __ldg(&neighbor[(size_t)y * f.W + x]);
        const int ox = nb & 0xff, oy = nb >> 8;
        if (ox == 0xff) return false;
        nx = ox - 32 + x; ny = oy - 32 + y;
        return true;
    }

    ZR_D void SuppressOutlier(float waveAvgExclusive, Reservoir& r)
    {
        if (r.w_sum > 50 * waveAvgExclusive)
        {
            r.M = 0; r.w_sum = 0; r.W = 0; r.rc.Clear();
        }
    }

    // Reservoir::Write(Reservoir::Load(rec)) leaves the reconnection words of a record unchanged whenever its two lossy fields
    // survive the round trip: the octahedral direction (EncodeOct32u(DecodeOct32(c)) == c for every code c whose two UNORM16
    // halves are not 0 / 0xffff -- checked for all 2^32 codes by tests/test_device_source_vs_oracle.py::test_oct32_round_trip;
    // the 131071 exceptions are aliases on the fold lines of the octahedron) and the three radiance halves (half -> float -> half
    // is the identity except for NaN payloads). Everything else is moved bit for bit by Load_Reconnection / Write.
    ZR_D bool RecordSurvivesRoundTrip(const zr_rpt_reservoir& in)
    {
        const uint32_t wx = in.w_k & 0xffff, wy = in.w_k >> 16;
        const bool interior = wx != 0 && wx != 0xffff && wy != 0 && wy != 0xffff;
        const uint32_t r = in.L_rg & 0x7fff, g = (in.L_rg >> 16) & 0x7fff, b = in.L_b & 0x7fff;
        return interior && r <= 0x7c00 && g <= 0x7c00 && b <= 0x7c00;
    }

    ZR_D void CopyToNextFrame(const zr_rpt_reservoir& in, zr_rpt_reservoir* __restrict__ outPtr, Reservoir r_curr, uint32_t M_max)
    {
        if (!r_curr.rc.Empty() && RecordSurvivesRoundTrip(in))
        {
            // same bytes as the decode + encode below, without the octahedral / half conversions
            zr_rpt_reservoir out = in;
            out.meta = r_curr.PackMeta(M_max);
            out.w_sum = Math::Sanitize(r_curr.w_sum);
            out.W = Math::Sanitize(r_curr.W);
            out.L_b = in.L_b & 0xffff;
            if (r_curr.rc.IsCase1()) { out.lightPdf = 0; out.dwdA = 0; out.seed_nee = 0; }
            else if (!r_curr.rc.IsCase2()) { out.dwdA = 0; out.seed_nee = 0; out.meshIdx = 0; }
            StoreRecord(outPtr, out);
        }
        else if (!r_curr.rc.Empty())
        {
            r_curr.Load_Reconnection(in);
            zr_rpt_reservoir out;
            r_curr.Write(out, M_max);
            StoreRecord(outPtr, out);
        }
        else
        {
            // WriteReservoirData: A.x and B of the OUTPUT record; its other bytes keep their old contents
            const uint4 old = LoadQ0(outPtr);
            const uint32_t k = r_curr.rc.k;   // EMPTY
            const uint32_t mm = r_curr.M < M_max ? r_curr.M : M_max;
            st128(outPtr, make_uint4((old.x & 0xffffff00u) | ((k | (mm << 4)) & 0xff), asuint(r_curr.w_sum), asuint(r_curr.W), old.w));
        }
    }

    // -------------------------------------------------------------------------------------------
    // shared lookups of the temporal pass (motion-vector reprojection, plane test, x_k between the two frames' instance transforms)
    // -------------------------------------------------------------------------------------------
    ZR_D bool PrevPixel(const FrameView& f, int x, int y, int& ppx, int& ppy)
    {
        const float2 renderDim = f2((float)f.W, (float)f.H);
        const float2 motionVec = unpack_snorm16x2(__ldg(&f.me[(size_t)y * f.W + x].x));
        const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / renderDim;
        const float2 prevUV = currUV - motionVec;
        const float2 pp = prevUV * renderDim;
        ppx = (int)pp.x; ppy = (int)pp.y;
        return !(prevUV.x < 0.0f || prevUV.y < 0.0f || prevUV.x > 1.0f || prevUV.y > 1.0f);
    }

    ZR_D bool PlaneHeuristic(float3 prevPos, float3 normal, float3 pos, float linearDepth, float th)
    {
        return fabsf(dot(normal, prevPos - pos)) <= th * linearDepth;
    }

    ZR_D void XkToPrev(const SceneDev& sc, Reconnection& rc)
    {
        const zr_mesh_instance md = LoadInstance(sc, rc.meshIdx);
        const float4 q_curr = normalize(Math::DecodeNormalized4(md.Rotation));
        const float3 T = f3(md.Translation[0], md.Translation[1], md.Translation[2]);
        const float3 x_local = Math::InverseTransformTRS(rc.x_k, T, q_curr, h3(md.Scale));
        const float3 prevTranslation = T - h3(md.dTranslation);
        const float4 q_prev = normalize(Math::DecodeNormalized4(md.PrevRotation));
        rc.x_k = Math::TransformTRS(x_local, prevTranslation, q_prev, h3(md.PrevScale));
    }
    ZR_D void XkToCurr(const SceneDev& sc, Reconnection& rc)
    {
        const zr_mesh_instance md = LoadInstance(sc, rc.meshIdx);
        const float3 T = f3(md.Translation[0], md.Translation[1], md.Translation[2]);
        const float3 dT = h3(md.dTranslation);
        const float3 prevTranslation = T - dT;
        const float4 q_prev = normalize(Math::DecodeNormalized4(md.PrevRotation));
        const float3 prevScale = h3(md.PrevScale), scale = h3(md.Scale);
        const float3 x_local = Math::InverseTransformTRS(rc.x_k, prevTranslation, q_prev, prevScale);
        const float4 q_curr = normalize(Math::DecodeNormalized4(md.Rotation));
        rc.x_k = Math::TransformTRS(x_local, T, q_curr, scale);
        const float4 dRot = f4(q_prev.x - q_curr.x, q_prev.y - q_curr.y, q_prev.z - q_curr.z, q_prev.w - q_curr.w);
        const float3 dScale = prevScale - scale;
        rc.x_k_in_motion = dot(dT, dT) > 0;
        rc.x_k_in_motion = rc.x_k_in_motion || dot(dRot, dRot) > 0;
        rc.x_k_in_motion = rc.x_k_in_motion || dot(dScale, dScale) > 0;
    }

    // ---- path generation helpers (k_pathtrace, rpt.cu) ----
    struct PrevHit { float alpha_lobe; float3 wi; float pdf; BSDF::LOBE lobe; };

    template<class SD>
    ZR_D void MaybeSetCase2OrCase3(int pathVertex, float3 pos, float3 normal, float t, uint32_t ID, uint32_t meshIdx,
        const SD& surface, const PrevHit& prevHit, const DirectLightingEstimate& ls, uint32_t seed_nee,
        Reconnection& rc, float alpha_min)
    {
        const float alpha_lobe_direct = BSDF::LobeAlpha(surface, ls.lobe);
        if (rc.Empty() && CanReconnect(prevHit.alpha_lobe, alpha_lobe_direct, prevHit.lobe, ls.lobe, alpha_min))
        {
            rc.SetCase2(pathVertex, pos, t, normal, ID, meshIdx, prevHit.wi, prevHit.lobe, prevHit.pdf, ls.wi, ls.lobe,
                ls.pdf_solidAngle, ls.lt, ls.pdf_light, ls.le, seed_nee, ls.dwdA);
        }
        if (rc.Empty() && (alpha_lobe_direct >= alpha_min))
        {
            rc.SetCase3(pathVertex + 1, ls.pos, ls.lt, ls.lobe, ls.ID, ls.le, ls.normal, ls.pdf_solidAngle, ls.pdf_light,
                ls.dwdA, ls.wi, ls.twoSided, seed_nee);
        }
    }

}
} // namespace zr
