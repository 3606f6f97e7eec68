// hostsim.cpp -- TEST INFRASTRUCTURE. Compiles the product's own traversal source (zetaray_b200/csrc/zr_scene.cuh:
// Traverse<0/1>, TriHit, the node decode) for the host with g++, so that the BVH builder + traversal pair can be checked
// against brute force on scenes of the benchmark's size (10^5 - 10^6 triangles) in the CPU test tier, where no GPU exists.
// Nothing here is shipped or used by the product; the product path is the same source compiled by nvcc for sm_90a.
#include "prelude.h"
#include "hostsim_api.h"
struct ZrTraverseStats { unsigned long long nodes, tris; };
static thread_local ZrTraverseStats g_stats;
#define ZR_TRAVERSE_STATS g_stats
#include "../../zetaray_b200/csrc/zr_scene.cuh"
#include "../../zetaray_b200/csrc/zr_bsdf.cuh"
#include "../../zetaray_b200/csrc/zr_rt.cuh"
#include "../../zetaray_b200/csrc/zr_rpt.cuh"
#include "../../zetaray_b200/csrc/zr_pixel.cuh"
#include "../../zetaray_b200/csrc/zr_rgi.cuh"

namespace zr
{
void set_error(const char*, ...) {}
}

extern "C"
{
// rays: n x {origin xyz, tmin, dir xyz, tmax}; hits: n x {t, u, v, triGlobal-as-float-bits}; flags (any-hit) may be null
int hostsim_trace(const void* nodes, const float* leafTris /* 12 floats per tri, leaf order */, const uint32_t* triMesh,
    const uint32_t* meshFirstTri, const float* rays, uint32_t n, float* hits, uint32_t* anyFlags, const uint32_t* ignoreIDs, int threads)
{
    zr::SceneDev sc{};
    sc.nodes = reinterpret_cast<const uint4*>(nodes);
    sc.tris = reinterpret_cast<const float4*>(leafTris);
    sc.triMesh = triMesh;
    sc.meshFirstTri = meshFirstTri;
    std::atomic<uint32_t> next{0};
    auto work = [&]() {
        for (;;)
        {
            const uint32_t b = next.fetch_add(256);
            if (b >= n) break;
            for (uint32_t i = b; i < std::min(n, b + 256); i++)
            {
                const float* r = rays + (size_t)i * 8;
                const float3 o = make_float3(r[0], r[1], r[2]), d = make_float3(r[4], r[5], r[6]);
                if (hits)
                {
                    zr::RayHit h = zr::TraceClosest(sc, o, d, r[3], r[7]);
                    float* out = hits + (size_t)i * 4;
                    out[0] = h.hit ? h.t : zr::FLT_MAX_; out[1] = h.bary.x; out[2] = h.bary.y; out[3] = zr::asfloat(h.tri);
                }
                if (anyFlags)
                    anyFlags[i] = zr::TraceAnyExcept(sc, o, d, r[3], r[7], ignoreIDs ? ignoreIDs[i] : 0xffffffffu) ? 1u : 0u;
            }
        }
    };
    std::vector<std::thread> pool;
    for (int t = 0; t < std::max(threads, 1); t++) pool.emplace_back(work);
    for (auto& t : pool) t.join();
    return 0;
}

// brute force with the same hit rule (closest t, ties to the lowest global triangle index); worldTris 9 floats per tri
int hostsim_brute(const float* worldTris, uint32_t numTris, const float* rays, uint32_t n, float* hits, int threads)
{
    std::atomic<uint32_t> next{0};
    auto work = [&]() {
        for (;;)
        {
            const uint32_t i = next.fetch_add(1);
            if (i >= n) break;
            const float* r = rays + (size_t)i * 8;
            const float3 o = make_float3(r[0], r[1], r[2]), d = make_float3(r[4], r[5], r[6]);
            bool hit = false; float bt = r[7], bu = 0, bv = 0; uint32_t btri = 0xffffffffu;
            for (uint32_t k = 0; k < numTris; k++)
            {
                const float* w = worldTris + (size_t)k * 9;
                float t, u, v;
                if (zr::TriHit(o, d, make_float3(w[0], w[1], w[2]), make_float3(w[3], w[4], w[5]), make_float3(w[6], w[7], w[8]), r[3], r[7], t, u, v))
                    if (!hit || t < bt) { hit = true; bt = t; bu = u; bv = v; btri = k; }
            }
            float* out = hits + (size_t)i * 4;
            out[0] = hit ? bt : zr::FLT_MAX_; out[1] = bu; out[2] = bv; out[3] = zr::asfloat(btri);
        }
    };
    std::vector<std::thread> pool;
    for (int t = 0; t < std::max(threads, 1); t++) pool.emplace_back(work);
    for (auto& t : pool) t.join();
    return 0;
}
}

// Structural check of a built tree, decoding the quantised boxes exactly as Traverse does. Returns the number of
// violations: a triangle vertex outside the box of a child it hangs under, a triangle referenced != 1 times, a child
// offset out of range. stats = {nodes visited, leaves, max depth, triangles seen}
extern "C" uint64_t hostsim_validate(const void* nodes_, uint32_t numNodes, const float* leafTris, uint32_t numTris, uint64_t stats[4])
{
    const zr::BVH8Node* nodes = reinterpret_cast<const zr::BVH8Node*>(nodes_);
    std::vector<uint8_t> seen(numTris, 0);
    std::vector<uint8_t> nodeSeen(numNodes, 0);
    uint64_t bad = 0;
    stats[0] = stats[1] = stats[2] = stats[3] = 0;
    struct Item { uint32_t node; float lo[3], hi[3]; uint32_t depth; };
    std::vector<Item> stack;
    Item root; root.node = 0; root.depth = 1;
    for (int a = 0; a < 3; a++) { root.lo[a] = -INFINITY; root.hi[a] = INFINITY; }
    stack.push_back(root);
    while (!stack.empty())
    {
        Item it = stack.back(); stack.pop_back();
        if (it.node >= numNodes) { bad++; continue; }
        if (nodeSeen[it.node]++) { bad++; continue; }
        stats[0]++; stats[2] = std::max<uint64_t>(stats[2], it.depth);
        const zr::BVH8Node& n = nodes[it.node];
        const float p[3] = { n.px, n.py, n.pz };
        const uint8_t ex[3] = { n.ex, n.ey, n.ez };
        float s[3];
        for (int a = 0; a < 3; a++) s[a] = __uint_as_float((uint32_t)ex[a] << 23);
        for (int c = 0; c < 8; c++)
        {
            const uint32_t meta = n.meta[c];
            if (meta == 0) continue;
            float lo[3], hi[3];
            for (int a = 0; a < 3; a++)
            {
                lo[a] = fmaf((float)n.qlo[a][c], s[a], p[a]);
                hi[a] = fmaf((float)n.qhi[a][c], s[a], p[a]);
                // a child box must also lie inside what its ancestors promised (else a ray clipped by the ancestor could miss it)
                if (lo[a] < it.lo[a] - 0.0f || hi[a] > it.hi[a] + 0.0f) { /* allowed: quantisation grids differ; only triangles matter */ }
            }
            if (meta & 0x20u)
            {
                Item ch; ch.node = n.childBase + (meta & 0x1fu); ch.depth = it.depth + 1;
                for (int a = 0; a < 3; a++) { ch.lo[a] = std::max(lo[a], it.lo[a]); ch.hi[a] = std::min(hi[a], it.hi[a]); }
                stack.push_back(ch);
            }
            else
            {
                stats[1]++;
                const uint32_t nt = meta >> 6, first = n.triBase + (meta & 0x1fu);
                for (uint32_t k = 0; k < nt; k++)
                {
                    if (first + k >= numTris) { bad++; continue; }
                    const float* t = leafTris + (size_t)(first + k) * 12;
                    uint32_t g; memcpy(&g, &t[3], 4);
                    if (g >= numTris || seen[g]++) bad++;
                    stats[3]++;
                    for (int v = 0; v < 3; v++)
                        for (int a = 0; a < 3; a++)
                        {
                            const float x = v == 0 ? t[a] : t[a] + t[4 * v + a];
                            // inside this child's box and inside every ancestor's (the intersection carried down)
                            if (x < std::max(lo[a], it.lo[a]) || x > std::min(hi[a], it.hi[a])) bad++;
                        }
                }
            }
        }
    }
    for (uint32_t i = 0; i < numTris; i++) if (seen[i] != 1) bad++;
    return bad;
}

// node visits and triangle tests of every ray (closest hit, or any hit when anyhit != 0), single-threaded
extern "C" int hostsim_trace_stats(const void* nodes, const float* leafTris, const uint32_t* triMesh, const uint32_t* meshFirstTri,
    const float* rays, uint32_t n, uint32_t* outNodes, uint32_t* outTris, int anyhit)
{
    zr::SceneDev sc{};
    sc.nodes = reinterpret_cast<const uint4*>(nodes); sc.tris = reinterpret_cast<const float4*>(leafTris);
    sc.triMesh = triMesh; sc.meshFirstTri = meshFirstTri;
    for (uint32_t i = 0; i < n; i++)
    {
        const float* r = rays + (size_t)i * 8;
        const float3 o = make_float3(r[0], r[1], r[2]), d = make_float3(r[4], r[5], r[6]);
        g_stats.nodes = g_stats.tris = 0;
        if (anyhit) zr::TraceAnyExcept(sc, o, d, r[3], r[7], 0xffffffffu); else zr::TraceClosest(sc, o, d, r[3], r[7]);
        outNodes[i] = (uint32_t)g_stats.nodes; outTris[i] = (uint32_t)g_stats.tris;
    }
    return 0;
}

// ---- the device BSDF source (zr_bsdf.cuh) behind the same probe entry points the oracle exports (oracle/orc_testapi.cpp), so the
// CPU tier can hold the two transcriptions of Common/BSDF.hlsli + BSDFSampling.hlsli to each other bit for bit ----
extern "C"
{
    static const uint16_t* g_rho = nullptr;
    void hostsim_set_rho_lut(const uint16_t* data) { g_rho = data; }
    static zr::BSDF::ShadingData mk(const orc_surface_desc* d)
    {
        using namespace zr;
        return BSDF::ShadingData::Init(f3(d->normal[0], d->normal[1], d->normal[2]), f3(d->wo[0], d->wo[1], d->wo[2]), d->metallic != 0,
            d->roughness, f3(d->baseColor[0], d->baseColor[1], d->baseColor[2]), d->eta_curr, d->eta_next, d->specTr != 0, d->trDepth,
            d->subsurface, d->coat_weight, f3(d->coat_color[0], d->coat_color[1], d->coat_color[2]), d->coat_roughness, d->coat_ior, g_rho);
    }
    void hostsim_bsdf_sample(const orc_surface_desc* d, uint32_t seed, float* out)
    {
        using namespace zr;
        BSDF::ShadingData s = mk(d);
        RNG rng; rng.State = seed;
        BSDF::BSDFSample b = BSDF::SampleBSDF(f3(d->normal[0], d->normal[1], d->normal[2]), s, rng);
        out[0] = b.wi.x; out[1] = b.wi.y; out[2] = b.wi.z; out[3] = (float)b.lobe; out[4] = b.pdf;
        out[5] = b.bsdfOverPdf.x; out[6] = b.bsdfOverPdf.y; out[7] = b.bsdfOverPdf.z; out[8] = b.f.x; out[9] = b.f.y; out[10] = b.f.z;
        out[11] = asfloat(rng.State);
    }
    void hostsim_bsdf_sample_nodiffuse(const orc_surface_desc* d, uint32_t seed, float* out)
    {
        using namespace zr;
        BSDF::ShadingData s = mk(d);
        RNG rng; rng.State = seed;
        BSDF::BSDFSample b = BSDF::SampleBSDF_NoDiffuse(f3(d->normal[0], d->normal[1], d->normal[2]), s, rng);
        out[0] = b.wi.x; out[1] = b.wi.y; out[2] = b.wi.z; out[3] = (float)b.lobe; out[4] = b.pdf;
        out[5] = b.bsdfOverPdf.x; out[6] = b.bsdfOverPdf.y; out[7] = b.bsdfOverPdf.z; out[8] = b.f.x; out[9] = b.f.y; out[10] = b.f.z;
        out[11] = asfloat(rng.State);
    }
    void hostsim_bsdf_eval_sampler(const orc_surface_desc* d, const float* wi, uint32_t lobe, uint32_t seed, float* out)
    {
        using namespace zr;
        BSDF::ShadingData s = mk(d);
        RNG rng; rng.State = seed;
        BSDF::BSDFSamplerEval e = BSDF::EvalBSDFSampler(f3(d->normal[0], d->normal[1], d->normal[2]), s, f3(wi[0], wi[1], wi[2]), (BSDF::LOBE)lobe, rng);
        out[0] = e.pdf; out[1] = e.bsdfOverPdf.x; out[2] = e.bsdfOverPdf.y; out[3] = e.bsdfOverPdf.z; out[4] = e.f.x; out[5] = e.f.y; out[6] = e.f.z;
        out[7] = asfloat(rng.State);
    }
    float hostsim_bsdf_sampler_pdf(const orc_surface_desc* d, const float* wi, uint32_t seed)
    {
        using namespace zr;
        BSDF::ShadingData s = mk(d);
        RNG rng; rng.State = seed;
        return BSDF::BSDFSamplerPdf(f3(d->normal[0], d->normal[1], d->normal[2]), s, f3(wi[0], wi[1], wi[2]), rng);
    }
    float hostsim_bsdf_sampler_pdf_nodiffuse(const orc_surface_desc* d, const float* wi)
    {
        using namespace zr;
        BSDF::ShadingData s = mk(d);
        return BSDF::BSDFSamplerPdf_NoDiffuse(f3(d->normal[0], d->normal[1], d->normal[2]), s, f3(wi[0], wi[1], wi[2]));
    }
    void hostsim_bsdf_unified(const orc_surface_desc* d, const float* wi, float* out)
    {
        using namespace zr;
        BSDF::ShadingData s = mk(d);
        s.SetWi(f3(wi[0], wi[1], wi[2]), f3(d->normal[0], d->normal[1], d->normal[2]));
        float3 f = BSDF::Unified(s).f;
        out[0] = f.x; out[1] = f.y; out[2] = f.z;
    }
}

// ---- device storage codecs (zr_common.cuh) behind the oracle's probe names ----
extern "C"
{
    void hostsim_oct32_roundtrip(const float* in, int n, float* out, uint32_t* enc)
    {
        for (int i = 0; i < n; i++)
        {
            const uint32_t e = zr::Math::EncodeOct32u(zr::f3(in[3 * i], in[3 * i + 1], in[3 * i + 2]));
            const float3 d = zr::Math::DecodeOct32(e);
            out[3 * i] = d.x; out[3 * i + 1] = d.y; out[3 * i + 2] = d.z;
            if (enc) enc[i] = e;
        }
    }
    uint32_t hostsim_pack_r11g11b10(float r, float g, float b) { return zr::pack_r11g11b10(zr::f3(r, g, b)); }
    void hostsim_unpack_r11g11b10(uint32_t p, float* out) { float3 c = zr::unpack_r11g11b10(p); out[0] = c.x; out[1] = c.y; out[2] = c.z; }
    uint32_t hostsim_pack_snorm16x2(float x, float y) { return zr::pack_snorm16x2(zr::f2(x, y)); }
    void hostsim_unpack_snorm16x2(uint32_t p, float* out) { float2 c = zr::unpack_snorm16x2(p); out[0] = c.x; out[1] = c.y; }
    uint32_t hostsim_pack_half2(float a, float b) { return zr::pack_half2(a, b); }
}

// ---- ray-query / material / light-sampling device source (zr_rt.cuh) on a host-resident scene ----
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
        sc.lvg = (const zr_voxel_sample*)h->lvg;
        for (int i = 0; i < 3; i++) { sc.lvgDim[i] = h->lvgDim[i]; sc.lvgExtents[i] = h->lvgExtents[i]; }
        sc.lvgOffsetY = h->lvgOffsetY;
        return sc;
    }
    void hostsim_probe_path_vertex(const hostsim_scene* hsc, const float* in, uint32_t seed, uint32_t* out)
    {
        using namespace zr;
        const SceneDev sc = dev_of(hsc);
        const float3 pos = f3(in[0], in[1], in[2]), normal = f3(in[3], in[4], in[5]), wi = f3(in[6], in[7], in[8]);
        const bool transmissive = in[9] != 0;
        memset(out, 0, 24 * 4);
        Hit h = FindClosest(sc, pos, normal, wi, transmissive);
        out[0] = h.hit; out[1] = asuint(h.t); out[2] = asuint(h.uv.x); out[3] = asuint(h.uv.y);
        out[4] = asuint(h.normal.x); out[5] = asuint(h.normal.y); out[6] = asuint(h.normal.z); out[7] = h.ID; out[8] = h.meshIdx; out[9] = h.matIdx;
        if (!h.hit) return;
        BSDF::ShadingData surface = BSDF::ShadingData::InitEmpty(); float eta;
        const bool ok = GetMaterialData(sc, -wi, BSDF::ETA_AIR, h, surface, eta);
        out[10] = ok; out[11] = asuint(eta);
        if (!ok) return;
        RNG rng; rng.State = seed;
        BSDF::BSDFSample b = BSDF::SampleBSDF(h.normal, surface, rng);
        out[12] = asuint(b.wi.x); out[13] = asuint(b.wi.y); out[14] = asuint(b.wi.z); out[15] = (uint32_t)b.lobe; out[16] = asuint(b.pdf);
        out[17] = asuint(b.bsdfOverPdf.x); out[18] = asuint(b.bsdfOverPdf.y); out[19] = asuint(b.bsdfOverPdf.z);
        surface.SetWi(b.wi, h.normal);
        const float3 f = BSDF::Unified(surface).f;
        out[20] = asuint(f.x); out[21] = asuint(f.y); out[22] = asuint(f.z); out[23] = rng.State;
    }
    void hostsim_probe_emissive_and_visibility(const hostsim_scene* hsc, const float* in, uint32_t* out)
    {
        using namespace zr;
        const SceneDev sc = dev_of(hsc);
        const float3 pos = f3(in[0], in[1], in[2]), normal = f3(in[3], in[4], in[5]), wi = f3(in[6], in[7], in[8]);
        const bool transmissive = in[9] != 0;
        memset(out, 0, 12 * 4);
        HitEmissive h = FindClosestEmissive(sc, pos, normal, wi, transmissive);
        out[0] = h.hit; out[1] = asuint(h.t); out[2] = h.geoIdx; out[3] = h.primIdx; out[4] = h.emissiveTriIdx;
        out[5] = asuint(h.bary.x); out[6] = asuint(h.bary.y); out[7] = asuint(h.lightPos.x); out[8] = asuint(h.lightPos.y); out[9] = asuint(h.lightPos.z);
        if (!h.hit) return;
        const uint32_t id = RNG::PCG3d(make_uint3(h.geoIdx, 0u, h.primIdx)).x;
        out[10] = Visibility_Segment(sc, pos, wi, h.t, normal, id, transmissive);
        out[11] = Visibility_Segment_Precise(sc, pos, wi, h.t, normal, id, transmissive);
    }
    void hostsim_probe_sample_light(const hostsim_scene* hsc, const float* pos3, uint32_t sampleSetIdx, uint32_t seed, int advance, uint32_t* out)
    {
        using namespace zr;
        const SceneDev sc = dev_of(hsc);
        RNG rng; rng.State = seed;
        Light::LightSample ls = Light::SampleLight(sc, f3(pos3[0], pos3[1], pos3[2]), sampleSetIdx, rng, advance != 0);
        out[0] = asuint(ls.pos.x); out[1] = asuint(ls.pos.y); out[2] = asuint(ls.pos.z);
        out[3] = asuint(ls.normal.x); out[4] = asuint(ls.normal.y); out[5] = asuint(ls.normal.z);
        out[6] = asuint(ls.le.x); out[7] = asuint(ls.le.y); out[8] = asuint(ls.le.z);
        out[9] = asuint(ls.bary.x); out[10] = asuint(ls.bary.y); out[11] = asuint(ls.pdf); out[12] = ls.idx; out[13] = ls.ID; out[14] = ls.twoSided;
        out[15] = rng.State;
    }
}

// ---- ReSTIR PT reservoir record codec (zr_rpt.cuh RPT::Reservoir) ----
extern "C" void hostsim_probe_rpt_reservoir(const zr_rpt_reservoir* in, uint32_t n, uint32_t M_max, zr_rpt_reservoir* out, zr_rpt_reservoir* out2)
{
    for (uint32_t i = 0; i < n; i++)
    {
        zr::RPT::Reservoir r = zr::RPT::Reservoir::Load(in[i]);
        memset(&out[i], 0, sizeof(out[i]));
        r.Write(out[i], M_max);
        out2[i] = in[i];
        r.WriteReservoirData(out2[i], M_max);
    }
}

// ---- the hybrid shift (zr_rpt.cuh Replay_kGt2_Sync / Shift2_Sync as a block of one thread) ----
extern "C" void hostsim_probe_rpt_shift(const hostsim_scene* hsc, const float* ray6, const zr_rpt_reservoir* rec, float alpha_min, uint32_t* out)
{
    using namespace zr;
    const SceneDev sc = dev_of(hsc);
    memset(out, 0, 8 * 4);
    const float3 o = f3(ray6[0], ray6[1], ray6[2]), d = f3(ray6[3], ray6[4], ray6[5]);
    Hit h = FindClosest(sc, o, d, d, false);
    if (!h.hit) return;
    BSDF::ShadingData surface = BSDF::ShadingData::InitEmpty(); float eta;
    if (!GetMaterialData(sc, -d, BSDF::ETA_AIR, h, surface, eta)) return;
    const float3 pos = mad(h.t, d, RTU::OffsetRayRTG(o, d));
    RPT::Reservoir r = RPT::Reservoir::Load(*rec);
    if (r.rc.Empty()) return;
    out[0] = 1; out[6] = r.rc.k;
    RPT::OffsetPathContext ctx = RPT::OffsetPathContext::Init();
    if (r.rc.k > 2)
    {
        ctx = RPT::Replay_kGt2_Sync(true, sc, pos, h.normal, eta, surface, r.rc, alpha_min).Quantize();
        out[7] = asuint(ctx.throughput.x);
    }
    RPT::OffsetPath shift = RPT::Shift2_Sync(true, sc, pos, h.normal, eta, surface, r.rc, &ctx, alpha_min);
    out[1] = asuint(shift.target.x); out[2] = asuint(shift.target.y); out[3] = asuint(shift.target.z);
    out[4] = asuint(shift.partialJacobian); out[5] = shift.surfKMin1Tramsmissive;
}

// ---- LoadPixel (zr_pixel.cuh) over a whole host-resident G-buffer ----
extern "C" void hostsim_probe_load_pixels(const hostsim_scene* hsc, const zr_frame_constants* fc, const void* core, const void* coat, int prev, uint32_t* out)
{
    using namespace zr;
    const SceneDev sc = dev_of(hsc);
    FrameView f{};
    f.fc = *fc; f.core = (const uint4*)core; f.coat = (const uint2*)coat; f.pcore = f.core; f.pcoat = f.coat;
    f.W = fc->RenderWidth; f.H = fc->RenderHeight;
    for (uint32_t y = 0; y < f.H; y++)
        for (uint32_t x = 0; x < f.W; x++)
        {
            uint32_t* o = out + ((size_t)y * f.W + x) * 16;
            memset(o, 0, 64);
            const GFlags fl = FlagsAt(f.core, f.W, (int)x, (int)y);
            if (fl.invalid) { o[0] = 0xffffffffu; continue; }
            Pixel p = LoadPixel(f, sc, f.core, f.coat, (int)x, (int)y, prev != 0, (int)x, (int)y);
            o[0] = (p.flags.transmissive) | (p.flags.emissive << 1) | (p.flags.trDepthGt0 << 3) | (p.flags.subsurface << 4) | (p.flags.coated << 5) | (p.flags.metallic << 7);
            o[1] = asuint(p.roughness); o[2] = asuint(p.z);
            o[3] = asuint(p.pos.x); o[4] = asuint(p.pos.y); o[5] = asuint(p.pos.z);
            o[6] = asuint(p.normal.x); o[7] = asuint(p.normal.y); o[8] = asuint(p.normal.z);
            o[9] = asuint(p.origin.x); o[10] = asuint(p.origin.y); o[11] = asuint(p.origin.z);
            o[12] = asuint(p.eta_next);
            RNG rng; rng.State = x * 7919u + y * 104729u + 1u;
            BSDF::BSDFSample b = BSDF::SampleBSDF(p.normal, p.surface, rng);
            o[13] = asuint(b.wi.x); o[14] = asuint(b.pdf); o[15] = asuint(b.bsdfOverPdf.x);
        }
}

extern "C" void hostsim_probe_lvg_sample(const hostsim_scene* hsc, const zr_frame_constants* fc, const float* pos3, uint32_t seed, uint32_t* out)
{
    using namespace zr;
    const SceneDev sc = dev_of(hsc);
    memset(out, 0, 13 * 4);
    RNG rng; rng.State = seed;
    LVG::VoxelLight v;
    const bool ok = LVG::Sample(sc, f3(pos3[0], pos3[1], pos3[2]), f3(sc.lvgExtents[0], sc.lvgExtents[1], sc.lvgExtents[2]), sc.lvgOffsetY,
        fc->CurrView, v, rng);
    out[0] = ok; out[12] = rng.State;
    if (!ok) return;
    out[1] = asuint(v.pos.x); out[2] = asuint(v.pos.y); out[3] = asuint(v.pos.z);
    out[4] = asuint(v.normal.x); out[5] = asuint(v.normal.y); out[6] = asuint(v.normal.z);
    out[7] = asuint(v.le.x); out[8] = asuint(v.le.y); out[9] = asuint(v.le.z);
    out[10] = asuint(v.pdf); out[11] = v.ID;
}

// ---- ReSTIR GI temporal reuse (zr_rgi.cuh) at one pixel, from a given initial reservoir record ----
extern "C" void hostsim_probe_rgi_temporal(const hostsim_scene* hsc, const zr_frame_constants* fc, const void* core, const void* me, const void* coat,
    const void* pcore, const void* pcoat, const zr_rgi_reservoir* prevRes, const zr_rgi_reservoir* initial, int x, int y, uint32_t seed, uint32_t M_max,
    uint32_t* out)
{
    using namespace zr;
    const SceneDev sc = dev_of(hsc);
    FrameView f{};
    f.fc = *fc; f.core = (const uint4*)core; f.me = (const uint2*)me; f.coat = (const uint2*)coat; f.pcore = (const uint4*)pcore; f.pcoat = (const uint2*)pcoat;
    f.W = fc->RenderWidth; f.H = fc->RenderHeight;
    memset(out, 0, 17 * 4);
    const size_t idx = (size_t)y * f.W + x;
    float roughness = 0;
    const GFlags flags = FlagsAt(f.core, f.W, x, y, &roughness);
    if (flags.invalid || flags.emissive) return;
    Pixel p = LoadPixel(f, sc, f.core, f.coat, x, y, false, x, y);
    const uint4 g = ld128(&f.core[idx]);
    const float3 baseColor = f3((float)(g.z & 0xff) / 255.0f, (float)((g.z >> 8) & 0xff) / 255.0f, (float)((g.z >> 16) & 0xff) / 255.0f);
    const float3 wo = normalize(p.origin - p.pos);
    BSDF::ShadingData surface0 = BSDF::ShadingData::Init(p.normal, wo, flags.metallic, roughness, baseColor, BSDF::ETA_AIR, p.eta_next, flags.transmissive,
        0.0f, 0.0f, 0.0f, f3(0.0f), 0.0f, BSDF::DEFAULT_ETA_COAT, sc.rho);
    GIReservoir r = GIReservoir::Init();
    r.pos = f3(initial->pos[0], initial->pos[1], initial->pos[2]); r.ID = initial->ID;
    r.Lo = f3(zr_f16_to_f32((uint16_t)(initial->Lo_rg & 0xffff)), zr_f16_to_f32((uint16_t)(initial->Lo_rg >> 16)), zr_f16_to_f32((uint16_t)(initial->Lo_b_M & 0xffff)));
    r.M = (float)(uint16_t)zr_f16_to_f32((uint16_t)(initial->Lo_b_M >> 16));
    r.w_sum = initial->w_sum; r.W = initial->W; r.normal = Math::DecodeOct32(initial->normal);
    if (r.ID != UINT32_MAX_)
    {
        float3 wi = r.pos - p.pos;
        const float t = length(wi);
        wi = wi / fmaxf(t, 1e-6f);
        surface0.SetWi(wi, p.normal);
        r.target_z = r.Lo * BSDF::Unified(surface0).f;
    }
    RNG rng; rng.State = seed;
    const float2 renderDim = f2((float)f.W, (float)f.H);
    const float2 motionVec = unpack_snorm16x2(f.me[idx].x);
    const float2 currUV = f2((float)x + 0.5f, (float)y + 0.5f) / renderDim;
    const float2 prevUV = currUV - motionVec;
    TemporalSampleData data[2]; bool valid[2];
    FindTemporalCandidate(f, sc, x, y, p.pos, p.normal, p.z, roughness, surface0.specTr, prevUV, rng, data, valid);
    if (valid[1] && roughness > 0.05f)
        TemporalResample2(f, sc, prevRes, p.pos, p.normal, surface0, data, r, rng);
    else if (valid[0])
        TemporalResample1(f, sc, prevRes, p.pos, p.normal, surface0, data[0], r, rng);
    zr_rgi_reservoir rec;
    WriteReservoir(rec, r, (float)M_max);
    memcpy(out, &rec, 48);
    out[12] = asuint(r.target_z.x); out[13] = asuint(r.target_z.y); out[14] = asuint(r.target_z.z);
    out[15] = rng.State; out[16] = (valid[0] ? 1u : 0u) + (valid[1] ? 1u : 0u);
}
