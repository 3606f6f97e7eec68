// hostsim_di.cpp -- TEST INFRASTRUCTURE. Host (g++) build of the ReSTIR DI device source (zetaray_b200/csrc/zr_rdi.cuh) as a block of
// one thread, behind probe entry points mirrored by the oracle (oracle/orc_rdi.cpp). A translation unit of its own: zr_rdi.cuh and
// zr_rgi.cuh both live in the library's unnamed namespace and reuse names.
#include "prelude.h"
#include "hostsim_api.h"
#include "../../zetaray_b200/csrc/zr_rdi.cuh"

namespace zr
{
void set_error(const char*, ...) {}
}

extern "C"
{
    static zr::SceneDev dev_of(const hostsim_scene* h)
    {
        zr::SceneDev sc{};
        sc.vertices = (const zr_vertex*)h->vertices; sc.indices = h->indices; sc.instances = (const zr_mesh_instance*)h->instances;
        sc.materials = (const zr_material*)h->materials; sc.emissives = (const zr_emissive_tri*)h->emissives;
        sc.aliasTable = (const zr_alias_entry*)h->aliasTable; sc.nodes = (const uint4*)h->nodes; sc.tris = (const float4*)h->leafTris;
        sc.triMesh = h->triMesh; sc.meshFirstTri = h->meshFirstTri; sc.rho = h->rho;
        sc.numInstances = h->numInstances; sc.numEmissives = h->numEmissives; sc.numTris = h->numTris;
        sc.sampleSets = (const zr_presampled_tri*)h->sampleSets; sc.numSampleSets = h->numSampleSets; sc.sampleSetSize = h->sampleSetSize;
        return sc;
    }

    // ReSTIR DI at one pixel as k_di_temporal does it: RIS over BSDF + light candidates, then (temporal != 0) the temporal candidate
    // and its resampling. out (14 words): the 32-byte reservoir record, target (3), rng state, candidate valid, #BSDF samples
    void hostsim_probe_rdi_pixel(const hostsim_scene* hsc, const zr_frame_constants* fc, const void* core, const void* me, const void* coat,
        const void* pcore, const void* pcoat, const zr_rdi_reservoir* prevRes, int x, int y, uint32_t sampleSetIdx, int temporal, uint32_t M_max,
        uint32_t* out)
    {
        using namespace zr;
        const SceneDev sc = dev_of(hsc);
        FrameView f{};
        f.fc = *fc; f.core = (const uint4*)core; f.me = (const uint2*)me; f.coat = (const uint2*)coat; f.pcore = (const uint4*)pcore; f.pcoat = (const uint2*)pcoat;
        f.W = fc->RenderWidth; f.H = fc->RenderHeight;
        memset(out, 0, 14 * 4);
        const size_t idx = (size_t)y * f.W + x;
        const GFlags flags = FlagsAt(f.core, f.W, x, y);
        if (flags.invalid || flags.emissive) { out[13] = 0xffffffffu; return; }
        Pixel p = LoadPixel(f, sc, f.core, f.coat, x, y, false, x, y);
        RNG rng = RNG::Init((uint32_t)x, (uint32_t)y, fc->FrameNum);
        const int numBsdfSamples = (!p.surface.GlossSpecular() && p.roughness < 0.3f) ? 2 : 1;
        Reservoir r = RIS_InitialCandidates_Sync(true, sc, p.pos, p.normal, p.roughness, p.surface, sampleSetIdx, numBsdfSamples, rng);
        bool valid = false;
        if (temporal)
        {
            const float2 motionVec = unpack_snorm16x2(f.me[idx].x);
            const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / f2((float)f.W, (float)f.H);
            const float2 prevUV = currUV - motionVec;
            TemporalCandidate tc = FindTemporalCandidate(f, sc, p.pos, p.normal, p.roughness, p.surface, prevUV);
            valid = tc.valid;
            TemporalResample1_Sync(tc.valid, sc, p.pos, p.normal, p.surface, tc, prevRes, f.W, r, rng);
        }
        zr_rdi_reservoir rec;
        r.Write(rec, M_max);
        memcpy(out, &rec, 32);
        out[8] = asuint(r.target.x); out[9] = asuint(r.target.y); out[10] = asuint(r.target.z);
        out[11] = rng.State; out[12] = valid; out[13] = (uint32_t)numBsdfSamples;
    }

    // Pairwise-MIS spatial reuse (PairwiseMIS.hlsli) of the centre pixel (x, y) with neighbours (nx[i], ny[i]): the centre reservoir is
    // completed from the emissive buffer + target plane as k_di_spatial does it; neighbours enter with their own LoadPixel surface.
    // out (14 words): the resulting 32-byte record (Write with M_max 0 = no clamp), target (3), W, m_c, rng state
    void hostsim_probe_rdi_pairwise(const hostsim_scene* hsc, const zr_frame_constants* fc, const void* core, const void* coat,
        const zr_rdi_reservoir* res, const void* target, int x, int y, const int* nx, const int* ny, int numNeighbors, uint32_t seed, uint32_t* out)
    {
        using namespace zr;
        const SceneDev sc = dev_of(hsc);
        FrameView f{};
        f.fc = *fc; f.core = (const uint4*)core; f.coat = (const uint2*)coat; f.pcore = f.core; f.pcoat = f.coat;
        f.W = fc->RenderWidth; f.H = fc->RenderHeight;
        memset(out, 0, 14 * 4);
        const size_t idx = (size_t)y * f.W + x;
        const GFlags flags = FlagsAt(f.core, f.W, x, y);
        if (flags.invalid || flags.emissive) { out[13] = 0xffffffffu; return; }
        Pixel p = LoadPixel(f, sc, f.core, f.coat, x, y, false, x, y);
        Reservoir r = Reservoir::Load(res[idx]);
        if (r.lightIdx != UINT32_MAX_)
        {
            const zr_emissive_tri& tri = sc.emissives[r.lightIdx];
            r.lightID = tri.ID;
            const float3 vtx0 = Light::Vtx0(tri);
            const float3 vtx1 = Light::DecodeEmissiveTriV1(tri);
            const float3 vtx2 = Light::DecodeEmissiveTriV2(tri);
            r.lightPos = (1.0f - r.bary.x - r.bary.y) * vtx0 + r.bary.x * vtx1 + r.bary.y * vtx2;
            r.lightNormal = cross(vtx1 - vtx0, vtx2 - vtx0);
            r.lightNormal = dot(r.lightNormal, r.lightNormal) == 0 ? r.lightNormal : normalize(r.lightNormal);
            r.doubleSided = Light::IsDoubleSided(tri);
            r.target = abs3(LoadTarget((const uint2*)target, idx));
        }
        RNG rng; rng.State = seed;
        PairwiseMIS mis = PairwiseMIS::Init((uint32_t)numNeighbors, r);
        for (int i = 0; i < numNeighbors; i++)
        {
            const GFlags fi = FlagsAt(f.core, f.W, nx[i], ny[i]);
            if (fi.invalid || fi.emissive) continue;
            Pixel pi = LoadPixel(f, sc, f.core, f.coat, nx[i], ny[i], false, nx[i], ny[i]);
            const Reservoir r_i = Reservoir::Load(res[(size_t)ny[i] * f.W + nx[i]]);
            mis.Stream_Sync(true, sc, r, p.pos, p.normal, p.surface, r_i, pi.pos, pi.normal, pi.surface, rng);
        }
        mis.End(r, rng);
        zr_rdi_reservoir rec;
        mis.r_s.Write(rec, 0xffffffffu);
        memcpy(out, &rec, 32);
        out[8] = asuint(mis.r_s.target.x); out[9] = asuint(mis.r_s.target.y); out[10] = asuint(mis.r_s.target.z);
        out[11] = asuint(mis.r_s.W); out[12] = asuint(mis.m_c); out[13] = rng.State;
    }
}
