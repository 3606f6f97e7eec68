// scene.cu -- scene upload, host BVH build and the ray-query test entry points.
//
// Replaces what ZetaCore/RayTracing/RtAccelerationStructure.cpp gets from the DXR driver (BLAS/TLAS
// build) with an own builder: binned-SAH binary BVH over world-space triangles -> collapsed to
// 8-wide nodes -> child boxes quantised to 8 bits (conservatively rounded outwards).
// World-space triangles are produced on the device with the same TransformTRS arithmetic the
// shading code uses (quantised rotation / half scale of RT::MeshInstance), so traversal geometry and
// shading geometry agree bit for bit.
#include "zr_scene.cuh"
#include <vector>
#include <algorithm>
#include <cmath>
#include <cstring>

namespace zr
{
namespace
{
    __global__ void k_world_tris(SceneDev sc, const uint32_t* __restrict__ triMesh, const uint32_t* __restrict__ meshFirstTri,
        uint32_t numTris, float* __restrict__ out /* 9 floats per tri */)
    {
        const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
        if (g >= numTris) return;
        const uint32_t m = triMesh[g];
        const uint32_t p = g - meshFirstTri[m];
        const zr_mesh_instance md = LoadInstance(sc, m);
        const float4 q = normalize(Math::DecodeNormalized4(md.Rotation));
        const float3 s = h3(md.Scale);
        const float3 t = f3(md.Translation[0], md.Translation[1], md.Translation[2]);
        const uint32_t tri = p * 3 + md.BaseIdxOffset;
        float3 pw[3];
        for (int k = 0; k < 3; k++)
        {
            const VertexD V = LoadVertex(sc, sc.indices[tri + k] + md.BaseVtxOffset);
            pw[k] = Math::TransformTRS(V.pos, t, q, s);
        }
        const float3 e1 = pw[1] - pw[0], e2 = pw[2] - pw[0];
        float* o = out + (size_t)g * 9;
        o[0] = pw[0].x; o[1] = pw[0].y; o[2] = pw[0].z;
        o[3] = e1.x; o[4] = e1.y; o[5] = e1.z;
        o[6] = e2.x; o[7] = e2.y; o[8] = e2.z;
    }

    // The emissive triangles [first[r], first[r] + start[r + 1] - start[r]) of range r take the material-derived bits packedA[r] /
    // packedB[r] (emissive_bits). One job holds up to EDIT_RANGES ranges; it travels as a kernel parameter, so an edit needs no device
    // allocation.
    constexpr uint32_t EDIT_RANGES = 96;
    struct EmissiveRefresh
    {
        uint32_t numRanges;
        uint32_t start[EDIT_RANGES + 1];    // exclusive prefix sum of the range lengths: thread t belongs to the r with start[r] <= t < start[r + 1]
        uint32_t first[EDIT_RANGES];
        uint32_t packedA[EDIT_RANGES];
        uint32_t packedB[EDIT_RANGES];
    };
    // PackedA bits the material sets: the emissive factor [0, 24), double sided (25) and the strength's low 4 bits [28, 32). The
    // id-patched bit (24) and bits 26-27 are the triangle's own; PackedB keeps its texture index [0, 16).
    constexpr uint32_t EMISSIVE_A_MATERIAL_BITS = 0xffffffu | (1u << 25) | (0xfu << 28);

    __global__ void k_refresh_emissives(const __grid_constant__ EmissiveRefresh job, zr_emissive_tri* __restrict__ emissives)
    {
        const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
        if (t >= job.start[job.numRanges]) return;
        uint32_t lo = 0, hi = job.numRanges - 1;
        while (lo < hi)
        {
            const uint32_t mid = (lo + hi + 1) >> 1;
            if (job.start[mid] <= t) lo = mid; else hi = mid - 1;
        }
        zr_emissive_tri& e = emissives[job.first[lo] + (t - job.start[lo])];
        e.PackedA = (e.PackedA & ~EMISSIVE_A_MATERIAL_BITS) | job.packedA[lo];
        e.PackedB = (e.PackedB & 0xffffu) | job.packedB[lo];
    }

    __global__ void k_trace_closest(SceneDev sc, const float* __restrict__ rays, uint32_t n, float* __restrict__ hits)
    {
        const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= n) return;
        const float* r = rays + (size_t)i * 8;
        RayHit h = TraceClosest(sc, f3(r[0], r[1], r[2]), f3(r[4], r[5], r[6]), r[3], r[7]);
        float* o = hits + (size_t)i * 4;
        o[0] = h.hit ? h.t : FLT_MAX_; o[1] = h.bary.x; o[2] = h.bary.y; o[3] = asfloat(h.tri);
    }

    __global__ void k_trace_any(SceneDev sc, const float* __restrict__ rays, uint32_t n, uint32_t* __restrict__ flags)
    {
        const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= n) return;
        const float* r = rays + (size_t)i * 8;
        flags[i] = TraceAnyExcept(sc, f3(r[0], r[1], r[2]), f3(r[4], r[5], r[6]), r[3], r[7], 0xffffffffu) ? 1u : 0u;
    }
}

// The optional BSDF features a material table uses. The per-pixel coat / transmissive / subsurface bits of the G-buffer and the
// surfaces built at path vertices come from these material fields alone (no textures or instance overrides in this build), read as
// Mat::GetCoatWeight, Mat::Transmissive and Mat::ThinWalled ? Mat::GetSubsurface : 0 do.
static uint32_t material_features(const zr_material* mats, size_t n)
{
    uint32_t f = 0;
    for (size_t i = 0; i < n; i++)
    {
        const zr_material& m = mats[i];
        if ((m.BaseColorTex_Subsurf_CoatWeight >> 24) & 0xff) f |= ZR_MATERIAL_COAT;
        if (m.CoatColor_Flags & (1u << 26)) f |= ZR_MATERIAL_TRANSMISSION;
        if ((m.CoatColor_Flags & (1u << 29)) && ((m.BaseColorTex_Subsurf_CoatWeight >> 16) & 0xff)) f |= ZR_MATERIAL_THIN_WALLED;
    }
    return f;
}

static uint32_t emissive_factor(const zr_material& m) { return m.EmissiveFactor_NormalScale & 0xffffffu; }
static uint32_t emissive_strength(const zr_material& m) { return m.EmissiveStrength_IOR & 0xffffu; }      // half bits

// The bits an emissive triangle takes from its instance's material, as RT::EmissiveTriangle's constructor stores them (the factor,
// the double-sided flag and the strength, whose low 4 bits also go to PackedA[28, 32)).
static void emissive_bits(const zr_material& m, uint32_t& packedA, uint32_t& packedB)
{
    const uint32_t strength = emissive_strength(m);
    packedA = emissive_factor(m) | (m.CoatColor_Flags & (1u << 25)) | ((strength & 0xfu) << 28);
    packedB = strength << 16;
}

template<typename T>
static zr_status upload(zr_scene* sc, const T* h, size_t n, const T** d)
{
    void* p = nullptr;
    ZR_CUDA(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)));
    sc->allocs[sc->numAllocs++] = p;        // owned by the scene from here on: released by zr_scene_destroy on every error path
    if (n) ZR_CUDA(cudaMemcpy(p, h, n * sizeof(T), cudaMemcpyHostToDevice));
    *d = (const T*)p;
    return ZR_OK;
}

zr_status scene_create(const zr_scene_desc* desc, zr_scene** out)
{
    if (!desc || !out || !desc->h_vertices || !desc->h_indices || !desc->h_instances || !desc->h_instance_num_tris ||
        !desc->h_materials || desc->num_instances == 0)
    {
        set_error("zr_scene_create: null input");
        return ZR_ERR_INVALID_ARG;
    }
    // Everything the kernels will index is checked here, on the host, in 64-bit arithmetic, before anything is allocated: a malformed
    // description is an error code, not an out-of-bounds device read in k_world_tris and every lighting kernel.
    {
        uint64_t totalTris = 0;
        for (uint32_t m = 0; m < desc->num_instances; m++)
        {
            const zr_mesh_instance& mi = desc->h_instances[m];
            const uint64_t nt = desc->h_instance_num_tris[m];
            if ((uint64_t)mi.BaseIdxOffset + 3 * nt > desc->num_indices)
            {
                set_error("zr_scene_create: instance %u indexes past the index buffer", m);
                return ZR_ERR_INVALID_ARG;
            }
            if (mi.MatIdx >= desc->num_materials)
            {
                set_error("zr_scene_create: instance %u uses material %u of %u", m, (unsigned)mi.MatIdx, desc->num_materials);
                return ZR_ERR_INVALID_ARG;
            }
            for (uint64_t i = 0; i < 3 * nt; i++)
                if ((uint64_t)mi.BaseVtxOffset + desc->h_indices[mi.BaseIdxOffset + i] >= desc->num_vertices)
                {
                    set_error("zr_scene_create: instance %u, index %llu points past the vertex buffer", m, (unsigned long long)i);
                    return ZR_ERR_INVALID_ARG;
                }
            if (mi.BaseEmissiveTriOffset != 0xffffffffu && (uint64_t)mi.BaseEmissiveTriOffset + nt > desc->num_emissives)
            {
                set_error("zr_scene_create: instance %u's emissive triangles [%u, %llu) lie past the %u emissive triangles", m,
                    mi.BaseEmissiveTriOffset, (unsigned long long)(mi.BaseEmissiveTriOffset + nt), desc->num_emissives);
                return ZR_ERR_INVALID_ARG;
            }
            totalTris += nt;
        }
        if (totalTris == 0) { set_error("zr_scene_create: scene has no triangles"); return ZR_ERR_INVALID_ARG; }
        if (totalTris > 0x7fffffffull) { set_error("zr_scene_create: more than 2^31 triangles"); return ZR_ERR_INVALID_ARG; }
        if (desc->num_emissives && !desc->h_emissives) { set_error("zr_scene_create: null emissive buffer"); return ZR_ERR_INVALID_ARG; }
    }
    zr_scene* sc = new zr_scene();
    zr_status st;
#define UP(field, ptr, n) if ((st = upload(sc, ptr, n, &sc->dev.field)) != ZR_OK) { zr_scene_destroy(sc); return st; }
    UP(vertices, desc->h_vertices, desc->num_vertices);
    UP(indices, desc->h_indices, desc->num_indices);
    UP(instances, desc->h_instances, desc->num_instances);
    UP(materials, desc->h_materials, desc->num_materials);
    UP(emissives, desc->h_emissives, desc->num_emissives);
    sc->dev.numInstances = desc->num_instances;
    sc->dev.numEmissives = desc->num_emissives;
    sc->materialFeatures = material_features(desc->h_materials, desc->num_materials);
    sc->hostMaterials.assign(desc->h_materials, desc->h_materials + desc->num_materials);
    sc->hostInstances.resize(desc->num_instances);
    for (uint32_t m = 0; m < desc->num_instances; m++)
        sc->hostInstances[m] = SceneHostInstance{ desc->h_instances[m].MatIdx, desc->h_instances[m].BaseEmissiveTriOffset,
            desc->h_instance_num_tris[m] };

    // triangle -> mesh maps
    std::vector<uint32_t> triMesh, meshFirst(desc->num_instances);
    uint32_t total = 0;
    for (uint32_t m = 0; m < desc->num_instances; m++)
    {
        meshFirst[m] = total;
        if (desc->h_instances[m].BaseIdxOffset + 3 * desc->h_instance_num_tris[m] > desc->num_indices)
        {
            set_error("zr_scene_create: instance %u indexes past the index buffer", m);
            zr_scene_destroy(sc);
            return ZR_ERR_INVALID_ARG;
        }
        for (uint32_t p = 0; p < desc->h_instance_num_tris[m]; p++) triMesh.push_back(m);
        total += desc->h_instance_num_tris[m];
    }
    if (total == 0) { set_error("zr_scene_create: scene has no triangles"); zr_scene_destroy(sc); return ZR_ERR_INVALID_ARG; }
    sc->dev.numTris = total;
    UP(triMesh, triMesh.data(), triMesh.size());
    UP(meshFirstTri, meshFirst.data(), meshFirst.size());

    // directional-albedo table
    {
        std::vector<uint16_t> rho(64 * 32 * 16);
        if ((st = read_asset("zr_scene_create", "rho_lut.bin", rho.data(), rho.size() * sizeof(uint16_t))) != ZR_OK) { zr_scene_destroy(sc); return st; }
        UP(rho, rho.data(), rho.size());
    }

    // world-space triangles on the device, then BVH on the host
    float* d_wt = nullptr;
    cudaError_t e = cudaMalloc(&d_wt, (size_t)total * 9 * sizeof(float));
    if (e != cudaSuccess) { zr_scene_destroy(sc); return cuda_fail(e, "world triangles (alloc)"); }
    k_world_tris<<<(total + 127) / 128, 128>>>(sc->dev, sc->dev.triMesh, sc->dev.meshFirstTri, total, d_wt);
    count_launch();
    e = cudaGetLastError();
    std::vector<float> wt((size_t)total * 9);
    if (e == cudaSuccess) e = cudaMemcpy(wt.data(), d_wt, wt.size() * sizeof(float), cudaMemcpyDeviceToHost);
    cudaFree(d_wt);
    if (e != cudaSuccess) { zr_scene_destroy(sc); return cuda_fail(e, "world triangles"); }

    BvhBuild w;
    build_bvh8(wt.data(), total, w);
    if (w.maxDepth - 1 > (uint32_t)BVH_STACK_ENTRIES)
    {
        set_error("zr_scene_create: the BVH is %u levels deep, the kernels' traversal stack holds %d levels below the root", w.maxDepth,
            BVH_STACK_ENTRIES);
        zr_scene_destroy(sc);
        return ZR_ERR_INVALID_ARG;
    }
    std::vector<float4> tris((size_t)total * 3);
    for (uint32_t s = 0; s < total; s++)
    {
        const uint32_t g = w.leafOrder[s];
        const float* t = &wt[(size_t)g * 9];
        uint32_t gb = g; float gf; memcpy(&gf, &gb, 4);
        tris[(size_t)s * 3 + 0] = make_float4(t[0], t[1], t[2], gf);
        tris[(size_t)s * 3 + 1] = make_float4(t[3], t[4], t[5], 0.0f);
        tris[(size_t)s * 3 + 2] = make_float4(t[6], t[7], t[8], 0.0f);
    }
    {
        const uint4* d_nodes = nullptr;
        if ((st = upload(sc, reinterpret_cast<const uint4*>(w.nodes.data()), w.nodes.size() * 5, &d_nodes)) != ZR_OK) { zr_scene_destroy(sc); return st; }
        sc->dev.nodes = d_nodes;
    }
    UP(tris, tris.data(), tris.size());
#undef UP
    sc->info.numNodes = (uint32_t)w.nodes.size();
    sc->info.numTris = total;
    sc->info.maxDepth = w.maxDepth;
    sc->info.maxStack = w.maxStack;
    sc->info.bytes = (uint32_t)(w.nodes.size() * sizeof(BVH8Node) + tris.size() * sizeof(float4));

    // alias table storage (built by zr_prelighting_render)
    if (desc->num_emissives)
    {
        e = cudaMalloc(&sc->d_alias, (size_t)desc->num_emissives * sizeof(zr_alias_entry));
        if (e == cudaSuccess) e = cudaMalloc(&sc->d_power, (size_t)(desc->num_emissives + 8) * sizeof(float));
        if (e == cudaSuccess) e = cudaMalloc(&sc->d_aliasScratch, ((size_t)desc->num_emissives * 2 + 16) * sizeof(uint32_t));
        if (e != cudaSuccess) { zr_scene_destroy(sc); return cuda_fail(e, "alias table storage"); }
        sc->dev.aliasTable = sc->d_alias;
    }
    *out = sc;
    return ZR_OK;
}

zr_status scene_update_materials(zr_scene* sc, uint32_t first, uint32_t count, const zr_material* h, cudaStream_t stream)
{
    // Every refusal happens here, before anything on the host or the device changes.
    if (!sc || !h || count == 0)
    {
        set_error("zr_scene_update_materials: null scene or materials, or count == 0");
        return ZR_ERR_INVALID_ARG;
    }
    const uint32_t numMaterials = (uint32_t)sc->hostMaterials.size();
    if ((uint64_t)first + count > numMaterials)
    {
        set_error("zr_scene_update_materials: materials [%u, %llu) lie past the %u materials of the scene", first,
            (unsigned long long)first + count, numMaterials);
        return ZR_ERR_INVALID_ARG;
    }
    std::vector<zr_material> next(sc->hostMaterials);
    std::copy(h, h + count, next.begin() + first);
    bool anyPower = false, anyEmissiveInstance = false;
    for (uint32_t m = 0; m < (uint32_t)sc->hostInstances.size(); m++)
    {
        const SceneHostInstance& in = sc->hostInstances[m];
        const zr_material& mat = next[in.matIdx];
        const bool hasEmissives = in.baseEmissiveTri != 0xffffffffu && in.numTris != 0;
        if (!hasEmissives && emissive_factor(mat) != 0 && emissive_factor(sc->hostMaterials[in.matIdx]) == 0)
        {
            set_error("zr_scene_update_materials: material %u becomes emissive, but instance %u, which uses it, has no emissive "
                "triangles (the emissive set is fixed at zr_scene_create)", (unsigned)in.matIdx, m);
            return ZR_ERR_INVALID_ARG;
        }
        if (hasEmissives)
        {
            anyEmissiveInstance = true;
            anyPower |= emissive_factor(mat) != 0 && (emissive_strength(mat) & 0x7fffu) != 0;
        }
    }
    if (sc->dev.numEmissives && anyEmissiveInstance && !anyPower)
    {
        set_error("zr_scene_update_materials: the edit leaves every emissive triangle with a zero emissive factor or strength; the "
            "light distribution cannot be normalised over zero power");
        return ZR_ERR_INVALID_ARG;
    }

    // The emissive triangles whose bits change: those of the instances whose material's factor, double-sided flag or strength the
    // edit changes. Consecutive triangles that take the same bits form one range.
    std::vector<uint32_t> rFirst, rCount, rA, rB;
    for (const SceneHostInstance& in : sc->hostInstances)
    {
        if (in.baseEmissiveTri == 0xffffffffu || in.numTris == 0 || in.matIdx < first || in.matIdx >= first + count) continue;
        uint32_t a, b, a0, b0;
        emissive_bits(next[in.matIdx], a, b);
        emissive_bits(sc->hostMaterials[in.matIdx], a0, b0);
        if (a == a0 && b == b0) continue;
        if (!rFirst.empty() && rFirst.back() + rCount.back() == in.baseEmissiveTri && rA.back() == a && rB.back() == b)
            rCount.back() += in.numTris;
        else
        {
            rFirst.push_back(in.baseEmissiveTri); rCount.push_back(in.numTris); rA.push_back(a); rB.push_back(b);
        }
    }

    ZR_CLEAR_BEGIN();       // a frame still in flight may read the old materials
    ZR_CUDA(cudaMemcpy(const_cast<zr_material*>(sc->dev.materials) + first, h, (size_t)count * sizeof(zr_material), cudaMemcpyHostToDevice));
    ZR_CLEAR_END();
    sc->hostMaterials.swap(next);
    sc->materialFeatures = material_features(sc->hostMaterials.data(), sc->hostMaterials.size());

    zr_emissive_tri* emissives = const_cast<zr_emissive_tri*>(sc->dev.emissives);
    for (size_t r0 = 0; r0 < rFirst.size(); r0 += EDIT_RANGES)
    {
        EmissiveRefresh job;
        job.numRanges = (uint32_t)std::min<size_t>(EDIT_RANGES, rFirst.size() - r0);
        job.start[0] = 0;
        for (uint32_t r = 0; r < job.numRanges; r++)
        {
            job.first[r] = rFirst[r0 + r]; job.packedA[r] = rA[r0 + r]; job.packedB[r] = rB[r0 + r];
            job.start[r + 1] = job.start[r] + rCount[r0 + r];       // <= numEmissives < 2^32 (checked at create)
        }
        const uint32_t n = job.start[job.numRanges];
        ZR_PROF("k_refresh_emissives", stream);
        k_refresh_emissives<<<(n + 255) / 256, 256, 0, stream>>>(job, emissives);
        ZR_LAUNCH_CHECK();
    }
    // The next frame samples the new light distribution. Before the first zr_prelighting_render there is none to rebuild.
    if (!rFirst.empty() && sc->aliasBuilt)
        return zr_prelighting_render(sc, stream);
    return ZR_OK;
}
} // namespace zr

extern "C"
{
    zr_status zr_scene_create(const zr_scene_desc* desc, zr_scene** out) { return zr::scene_create(desc, out); }
    void zr_scene_destroy(zr_scene* sc)
    {
        if (!sc) return;
        for (int i = 0; i < sc->numAllocs; i++) cudaFree(sc->allocs[i]);
        if (sc->d_alias) cudaFree(sc->d_alias);
        if (sc->d_power) cudaFree(sc->d_power);
        if (sc->d_aliasScratch) cudaFree(sc->d_aliasScratch);
        if (sc->d_sampleSets) cudaFree(sc->d_sampleSets);
        if (sc->d_lvg) cudaFree(sc->d_lvg);
        delete sc;
    }
    zr_status zr_bvh_build_host(const float* h_world_tris, uint32_t num_tris, void* h_nodes, uint32_t node_capacity,
        uint32_t* h_leaf_order, uint32_t out_info[4])
    {
        if (!h_world_tris || !out_info || num_tris == 0) { zr::set_error("zr_bvh_build_host: null argument"); return ZR_ERR_INVALID_ARG; }
        zr::BvhBuild w;
        zr::build_bvh8(h_world_tris, num_tris, w);
        out_info[0] = (uint32_t)w.nodes.size(); out_info[1] = num_tris; out_info[2] = w.maxDepth; out_info[3] = w.maxStack;
        if (h_nodes)
        {
            if (node_capacity < w.nodes.size()) { zr::set_error("zr_bvh_build_host: %zu nodes, capacity %u", w.nodes.size(), node_capacity); return ZR_ERR_INVALID_ARG; }
            memcpy(h_nodes, w.nodes.data(), w.nodes.size() * sizeof(zr::BVH8Node));
        }
        if (h_leaf_order) memcpy(h_leaf_order, w.leafOrder.data(), (size_t)num_tris * sizeof(uint32_t));
        return ZR_OK;
    }
    zr_status zr_scene_update_materials(zr_scene* sc, uint32_t first, uint32_t count, const zr_material* h_materials, void* stream)
    {
        return zr::scene_update_materials(sc, first, count, h_materials, (cudaStream_t)stream);
    }
    zr_status zr_scene_get_tables(const zr_scene* sc, const zr_material** d_materials, uint32_t* num_materials,
        const zr_emissive_tri** d_emissives, uint32_t* num_emissives)
    {
        if (!sc || !d_materials || !num_materials || !d_emissives || !num_emissives) return ZR_ERR_INVALID_ARG;
        *d_materials = sc->dev.materials; *num_materials = (uint32_t)sc->hostMaterials.size();
        *d_emissives = sc->dev.emissives; *num_emissives = sc->dev.numEmissives;
        return ZR_OK;
    }
    zr_status zr_scene_bvh_stats(const zr_scene* sc, uint32_t out[4])
    {
        if (!sc || !out) return ZR_ERR_INVALID_ARG;
        out[0] = sc->info.numNodes; out[1] = sc->info.numTris; out[2] = sc->info.maxDepth; out[3] = sc->info.bytes;
        return ZR_OK;
    }
    zr_status zr_scene_material_features(const zr_scene* sc, uint32_t* out)
    {
        if (!sc || !out) return ZR_ERR_INVALID_ARG;
        *out = sc->materialFeatures;
        return ZR_OK;
    }
    zr_status zr_scene_trace_closest(const zr_scene* sc, const float* d_rays, uint32_t n, float* d_hits, void* stream)
    {
        if (!sc || !d_rays || !d_hits) { zr::set_error("zr_scene_trace_closest: null argument"); return ZR_ERR_INVALID_ARG; }
        if (n == 0) return ZR_OK;
        ZR_PROF("k_trace_closest", (cudaStream_t)stream);
        zr::k_trace_closest<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(sc->dev, d_rays, n, d_hits);
        ZR_LAUNCH_CHECK();
        return ZR_OK;
    }
    zr_status zr_scene_trace_any(const zr_scene* sc, const float* d_rays, uint32_t n, uint32_t* d_flags, void* stream)
    {
        if (!sc || !d_rays || !d_flags) { zr::set_error("zr_scene_trace_any: null argument"); return ZR_ERR_INVALID_ARG; }
        if (n == 0) return ZR_OK;
        ZR_PROF("k_trace_any", (cudaStream_t)stream);
        zr::k_trace_any<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(sc->dev, d_rays, n, d_flags);
        ZR_LAUNCH_CHECK();
        return ZR_OK;
    }
    zr_status zr_scene_get_alias_table(const zr_scene* sc, const zr_alias_entry** d_table, uint32_t* n)
    {
        if (!sc || !d_table || !n) return ZR_ERR_INVALID_ARG;
        *d_table = sc->d_alias; *n = sc->dev.numEmissives;
        return ZR_OK;
    }
}
