// ORACLE -- test infrastructure, not product code (see orc_math.h header).
// Small C entry points so the CPU-only tests can probe codecs and the BSDF restatement directly.
#include "orc_api.h"
#include "orc_scene.h"
#include "orc_rpt.h"
#include "orc_pixel.h"

using namespace orc;

extern "C"
{
    // n unit vectors -> oct32 -> unit vectors (Math::EncodeOct32 / DecodeOct32, Math.hlsli:636-676)
    void orc_oct32_roundtrip(const float* in, int n, float* out)
    {
        for (int i = 0; i < n; i++)
        {
            float3 d = Math::DecodeOct32(Math::EncodeOct32u(f3(in[3 * i], in[3 * i + 1], in[3 * i + 2])));
            out[3 * i] = d.x; out[3 * i + 1] = d.y; out[3 * i + 2] = d.z;
        }
    }
    uint32_t orc_pack_r11g11b10(float r, float g, float b) { return pack_r11g11b10(f3(r, g, b)); }
    void orc_unpack_r11g11b10(uint32_t p, float* out) { float3 c = unpack_r11g11b10(p); out[0] = c.x; out[1] = c.y; out[2] = c.z; }
    uint32_t orc_pack_snorm16x2(float x, float y) { return pack_snorm16x2(f2(x, y)); }
    void orc_unpack_snorm16x2(uint32_t p, float* out) { float2 c = unpack_snorm16x2(p); out[0] = c.x; out[1] = c.y; }

    static BSDF::ShadingData mk(const orc_surface_desc* d)
    {
        return BSDF::ShadingData::Init(f3(d->normal[0], d->normal[1], d->normal[2]), f3(d->wo[0], d->wo[1], d->wo[2]), d->metallic != 0,
            d->roughness, f3(d->baseColor[0], d->baseColor[1], d->baseColor[2]), d->eta_curr, d->eta_next, d->specTr != 0, d->trDepth,
            d->subsurface, d->coat_weight, f3(d->coat_color[0], d->coat_color[1], d->coat_color[2]), d->coat_roughness, d->coat_ior);
    }
    // out: wi(3), lobe, pdf, bsdfOverPdf(3), f(3), rngStateAfter
    void orc_bsdf_sample(const orc_surface_desc* d, uint32_t seed, float* out)
    {
        BSDF::ShadingData s = mk(d);
        RNG rng = RNG::InitSeed(seed);
        BSDF::BSDFSample b = BSDF::SampleBSDF(f3(d->normal[0], d->normal[1], d->normal[2]), s, rng);
        out[0] = b.wi.x; out[1] = b.wi.y; out[2] = b.wi.z; out[3] = (float)b.lobe; out[4] = b.pdf;
        out[5] = b.bsdfOverPdf.x; out[6] = b.bsdfOverPdf.y; out[7] = b.bsdfOverPdf.z; out[8] = b.f.x; out[9] = b.f.y; out[10] = b.f.z;
        out[11] = asfloat(rng.State);
    }
    // out: pdf, bsdfOverPdf(3), f(3), rngStateAfter
    void orc_bsdf_eval_sampler(const orc_surface_desc* d, const float* wi, uint32_t lobe, uint32_t seed, float* out)
    {
        BSDF::ShadingData s = mk(d);
        RNG rng = RNG::InitSeed(seed);
        BSDF::BSDFSamplerEval e = BSDF::EvalBSDFSampler(f3(d->normal[0], d->normal[1], d->normal[2]), s, f3(wi[0], wi[1], wi[2]), (BSDF::LOBE)lobe, rng);
        out[0] = e.pdf; out[1] = e.bsdfOverPdf.x; out[2] = e.bsdfOverPdf.y; out[3] = e.bsdfOverPdf.z; out[4] = e.f.x; out[5] = e.f.y; out[6] = e.f.z;
        out[7] = asfloat(rng.State);
    }
    float orc_bsdf_sampler_pdf(const orc_surface_desc* d, const float* wi, uint32_t seed)
    {
        BSDF::ShadingData s = mk(d);
        RNG rng = RNG::InitSeed(seed);
        return BSDF::BSDFSamplerPdf(f3(d->normal[0], d->normal[1], d->normal[2]), s, f3(wi[0], wi[1], wi[2]), rng);
    }
    void orc_bsdf_sample_nodiffuse(const orc_surface_desc* d, uint32_t seed, float* out)
    {
        BSDF::ShadingData s = mk(d);
        RNG rng = RNG::InitSeed(seed);
        BSDF::BSDFSample b = BSDF::SampleBSDF_NoDiffuse(f3(d->normal[0], d->normal[1], d->normal[2]), s, rng);
        out[0] = b.wi.x; out[1] = b.wi.y; out[2] = b.wi.z; out[3] = (float)b.lobe; out[4] = b.pdf;
        out[5] = b.bsdfOverPdf.x; out[6] = b.bsdfOverPdf.y; out[7] = b.bsdfOverPdf.z; out[8] = b.f.x; out[9] = b.f.y; out[10] = b.f.z;
        out[11] = asfloat(rng.State);
    }
    float orc_bsdf_sampler_pdf_nodiffuse(const orc_surface_desc* d, const float* wi)
    {
        BSDF::ShadingData s = mk(d);
        return BSDF::BSDFSamplerPdf_NoDiffuse(f3(d->normal[0], d->normal[1], d->normal[2]), s, f3(wi[0], wi[1], wi[2]));
    }
    // f(wi) * |cos| as BSDF::Unified returns it
    void orc_bsdf_unified(const orc_surface_desc* d, const float* wi, float* out)
    {
        BSDF::ShadingData s = mk(d);
        s.SetWi(f3(wi[0], wi[1], wi[2]), f3(d->normal[0], d->normal[1], d->normal[2]));
        float3 f = BSDF::Unified(s).f;
        out[0] = f.x; out[1] = f.y; out[2] = f.z;
    }

    // ---- ray-query / material / light-sampling probes on a scene (mirrored by tests/hostsim for the device source) ----
    // in: pos(3) normal(3) wi(3) transmissive; out: 24 words
    void orc_probe_path_vertex(void* scene_, const float* in, uint32_t seed, uint32_t* out)
    {
        const Scene& sc = *(const Scene*)scene_;
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
        RNG rng = RNG::InitSeed(seed);
        BSDF::BSDFSample b = BSDF::SampleBSDF(h.normal, surface, rng);
        out[12] = asuint(b.wi.x); out[13] = asuint(b.wi.y); out[14] = asuint(b.wi.z); out[15] = (uint32_t)b.lobe; out[16] = asuint(b.pdf);
        out[17] = asuint(b.bsdfOverPdf.x); out[18] = asuint(b.bsdfOverPdf.y); out[19] = asuint(b.bsdfOverPdf.z);
        surface.SetWi(b.wi, h.normal);
        const float3 f = BSDF::Unified(surface).f;
        out[20] = asuint(f.x); out[21] = asuint(f.y); out[22] = asuint(f.z); out[23] = rng.State;
    }
    // in: as above; out: 12 words {hit, t, geoIdx, primIdx, emissiveTriIdx, bary(2), lightPos(3), visApprox, visPrecise} -- the two
    // visibility queries go from pos along wi to the hit distance, target = the hit triangle's ID
    void orc_probe_emissive_and_visibility(void* scene_, const float* in, uint32_t* out)
    {
        const Scene& sc = *(const Scene*)scene_;
        const float3 pos = f3(in[0], in[1], in[2]), normal = f3(in[3], in[4], in[5]), wi = f3(in[6], in[7], in[8]);
        const bool transmissive = in[9] != 0;
        memset(out, 0, 12 * 4);
        HitEmissive h = FindClosestEmissive(sc, pos, normal, wi, transmissive);
        out[0] = h.hit; out[1] = asuint(h.t); out[2] = h.geoIdx; out[3] = h.primIdx; out[4] = h.emissiveTriIdx;
        out[5] = asuint(h.bary.x); out[6] = asuint(h.bary.y); out[7] = asuint(h.lightPos.x); out[8] = asuint(h.lightPos.y); out[9] = asuint(h.lightPos.z);
        if (!h.hit) return;
        const uint32_t id = RNG::PCG3d(uint3{ h.geoIdx, 0u, h.primIdx }).x;
        out[10] = Visibility_Segment(sc, pos, wi, h.t, normal, id, transmissive);
        out[11] = Visibility_Segment_Precise(sc, pos, wi, h.t, normal, id, transmissive);
    }
    // out: 14 words {pos(3), normal(3), le(3), bary(2)->2, pdf, idx, ID, twoSided -> 15?}
    void orc_probe_sample_light(void* scene_, const float* pos3, uint32_t sampleSetIdx, uint32_t seed, int advance, uint32_t* out)
    {
        const Scene& sc = *(const Scene*)scene_;
        RNG rng = RNG::InitSeed(seed);
        Light::LightSample ls = Light::SampleLight(sc, f3(pos3[0], pos3[1], pos3[2]), sampleSetIdx, rng, advance != 0);
        out[0] = asuint(ls.pos.x); out[1] = asuint(ls.pos.y); out[2] = asuint(ls.pos.z);
        out[3] = asuint(ls.normal.x); out[4] = asuint(ls.normal.y); out[5] = asuint(ls.normal.z);
        out[6] = asuint(ls.le.x); out[7] = asuint(ls.le.y); out[8] = asuint(ls.le.z);
        out[9] = asuint(ls.bary.x); out[10] = asuint(ls.bary.y); out[11] = asuint(ls.pdf); out[12] = ls.idx; out[13] = ls.ID; out[14] = ls.twoSided;
        out[15] = rng.State;
    }

    // ReSTIR PT reservoir record: Load -> Write(M_max) -> out, and Load -> WriteReservoirData(M_max) over a copy of the input -> out2
    void orc_probe_rpt_reservoir(const zr_rpt_reservoir* in, uint32_t n, uint32_t M_max, zr_rpt_reservoir* out, zr_rpt_reservoir* out2)
    {
        for (uint32_t i = 0; i < n; i++)
        {
            RPT::Reservoir r = RPT::Reservoir::Load(in[i]);
            memset(&out[i], 0, sizeof(out[i]));
            r.Write(out[i], M_max);
            out2[i] = in[i];
            r.WriteReservoirData(out2[i], M_max);
        }
    }

    // The hybrid shift of ReSTIR PT (Shift.hlsli: random replay for k > 2, then reconnection) applied to a path held in a
    // 64-byte reservoir record, from a NEW primary vertex: the first hit of the camera ray (origin, dir).
    // out (8 words): {valid destination, shift.target xyz, shift.partialJacobian, surfKMin1Transmissive, k, replay throughput.x}
    void orc_probe_rpt_shift(void* scene_, const float* ray6, const zr_rpt_reservoir* rec, float alpha_min, uint32_t* out)
    {
        const Scene& sc = *(const Scene*)scene_;
        memset(out, 0, 8 * 4);
        const float3 o = f3(ray6[0], ray6[1], ray6[2]), d = f3(ray6[3], ray6[4], ray6[5]);
        // the camera ray as a "path vertex" query: start slightly behind o along -d with d as the normal
        Hit h = FindClosest(sc, o, d, d, false);
        if (!h.hit) return;
        BSDF::ShadingData surface = BSDF::ShadingData::InitEmpty(); float eta;
        if (!GetMaterialData(sc, -d, BSDF::ETA_AIR, h, surface, eta)) return;
        const float3 pos = mad(h.t, d, RTU::OffsetRayRTG(o, d));
        RPT::Reservoir r = RPT::Reservoir::Load(*rec);
        if (r.rc.Empty()) return;
        out[0] = 1; out[6] = r.rc.k;
        RPT::OffsetPathContext ctx = RPT::OffsetPathContext::Init(); const RPT::OffsetPathContext* pctx = nullptr;
        if (r.rc.k > 2)
        {
            ctx = RPT::Replay_kGt2(sc, pos, h.normal, eta, surface, r.rc, alpha_min).Quantize();
            pctx = &ctx;
            out[7] = asuint(ctx.throughput.x);
        }
        RPT::OffsetPath shift = RPT::Shift2(sc, pos, h.normal, eta, surface, r.rc, pctx, alpha_min);
        out[1] = asuint(shift.target.x); out[2] = asuint(shift.target.y); out[3] = asuint(shift.target.z);
        out[4] = asuint(shift.partialJacobian); out[5] = shift.surfKMin1Tramsmissive;
    }

    // LoadPixel (the per-pixel reconstruction every lighting kernel starts with) over a whole G-buffer.
    // out: 16 words per pixel {flags byte, roughness, z, pos(3), normal(3), origin(3), eta_next, then a BSDF sample's wi.x, pdf, bsdfOverPdf.x}
    void orc_probe_load_pixels(void* scene_, const zr_frame_constants* fc, const uint32_t* core_, const uint32_t* coat_, int prev, uint32_t* out)
    {
        const uint4* core = (const uint4*)core_;
        const uint2* coat = (const uint2*)coat_;
        Frame f;
        f.sc = (const Scene*)scene_; f.fc = fc; f.core = core; f.me = nullptr; f.coat = coat; f.pcore = core; f.pcoat = coat;
        f.W = fc->RenderWidth; f.H = fc->RenderHeight;
        for (uint32_t y = 0; y < f.H; y++)
            for (uint32_t x = 0; x < f.W; x++)
            {
                uint32_t* o = out + ((size_t)y * f.W + x) * 16;
                memset(o, 0, 64);
                const GFlags fl = FlagsAt(core, f.W, x, y);
                if (fl.invalid) { o[0] = 0xffffffffu; continue; }
                Pixel p = LoadPixel(f, core, coat, (int)x, (int)y, prev != 0, (int)x, (int)y);
                o[0] = (p.flags.transmissive) | (p.flags.emissive << 1) | (p.flags.trDepthGt0 << 3) | (p.flags.subsurface << 4) | (p.flags.coated << 5) | (p.flags.metallic << 7);
                o[1] = asuint(p.roughness); o[2] = asuint(p.z);
                o[3] = asuint(p.pos.x); o[4] = asuint(p.pos.y); o[5] = asuint(p.pos.z);
                o[6] = asuint(p.normal.x); o[7] = asuint(p.normal.y); o[8] = asuint(p.normal.z);
                o[9] = asuint(p.origin.x); o[10] = asuint(p.origin.y); o[11] = asuint(p.origin.z);
                o[12] = asuint(p.eta_next);
                RNG rng = RNG::InitSeed(x * 7919u + y * 104729u + 1u);
                BSDF::BSDFSample b = BSDF::SampleBSDF(p.normal, p.surface, rng);
                o[13] = asuint(b.wi.x); o[14] = asuint(b.pdf); o[15] = asuint(b.bsdfOverPdf.x);
            }
    }

    // LVG::Sample (Common/LightVoxelGrid.hlsli:54-68) at a position, with the frame's view matrix; out: 13 words
    void orc_probe_lvg_sample(void* scene_, const zr_frame_constants* fc, const float* pos3, uint32_t seed, uint32_t* out)
    {
        const Scene& sc = *(const Scene*)scene_;
        memset(out, 0, 13 * 4);
        RNG rng = RNG::InitSeed(seed);
        zr_voxel_sample v;
        const bool ok = LVG::Sample(sc, f3(pos3[0], pos3[1], pos3[2]), f3(sc.lvgExtents[0], sc.lvgExtents[1], sc.lvgExtents[2]), sc.lvgOffsetY,
            fc->CurrView, v, rng);
        out[0] = ok; out[12] = rng.State;
        if (!ok) return;
        const float3 n = Math::DecodeOct32(v.normal);
        out[1] = asuint(v.pos[0]); out[2] = asuint(v.pos[1]); out[3] = asuint(v.pos[2]);
        out[4] = asuint(n.x); out[5] = asuint(n.y); out[6] = asuint(n.z);
        out[7] = asuint(zr_f16_to_f32(v.le[0])); out[8] = asuint(zr_f16_to_f32(v.le[1])); out[9] = asuint(zr_f16_to_f32(v.le[2]));
        out[10] = asuint(v.pdf); out[11] = v.ID;
    }
}
