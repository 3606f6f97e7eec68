// comm.cu -- strip-halo transport for sharded frames (SURVEY 8e) behind the C-ABI: grouped NCCL send / recv of 32-row bands
// between neighbouring strips, issued from C++ on the stream the producing kernels run on (no host callback, no packing: a band is
// a contiguous row range of a plane). NCCL is bound at run time with dlopen / dlsym (libnccl.so.2: torch's bundled copy when the
// host process is a torch.distributed rank, the system library otherwise), so the library has no link-time dependency on it.
// A host without NCCL supplies its own transport instead (zr_comm_create_transport); every zr_comm_* entry checks its arguments,
// returns early at world == 1 and counts its traffic in one place, then hands the bands to NCCL or to that transport.
#include <dlfcn.h>
#include <cuda_runtime.h>
#include <cstring>
#include "../../include/zr_abi.h"
#include "zr_common.cuh"

namespace
{
    struct NcclUniqueId { char internal[128]; };
    typedef void* NcclComm;
    enum { NCCL_UINT8 = 1, NCCL_UINT32 = 3 };      // nccl.h: ncclInt8 = 0, ncclUint8 = 1, ncclInt32 = 2, ncclUint32 = 3
    enum { NCCL_SUM = 0 };

    struct NcclApi
    {
        int (*GetUniqueId)(NcclUniqueId*) = nullptr;
        int (*CommInitRank)(NcclComm*, int, NcclUniqueId, int) = nullptr;
        int (*CommDestroy)(NcclComm) = nullptr;
        int (*Send)(const void*, size_t, int, int, NcclComm, cudaStream_t) = nullptr;
        int (*Recv)(void*, size_t, int, int, NcclComm, cudaStream_t) = nullptr;
        int (*GroupStart)() = nullptr;
        int (*GroupEnd)() = nullptr;
        int (*AllReduce)(const void*, void*, size_t, int, int, NcclComm, cudaStream_t) = nullptr;
        const char* (*GetErrorString)(int) = nullptr;
        bool ok = false;
    };

    NcclApi& Api()
    {
        static NcclApi api;
        static bool tried = false;
        if (tried) return api;
        tried = true;
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return api;
#define ZR_SYM(field, name) api.field = (decltype(api.field))dlsym(h, name)
        ZR_SYM(GetUniqueId, "ncclGetUniqueId"); ZR_SYM(CommInitRank, "ncclCommInitRank"); ZR_SYM(CommDestroy, "ncclCommDestroy");
        ZR_SYM(Send, "ncclSend"); ZR_SYM(Recv, "ncclRecv"); ZR_SYM(GroupStart, "ncclGroupStart"); ZR_SYM(GroupEnd, "ncclGroupEnd");
        ZR_SYM(AllReduce, "ncclAllReduce");
        ZR_SYM(GetErrorString, "ncclGetErrorString");
#undef ZR_SYM
        api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.Send && api.Recv && api.GroupStart && api.GroupEnd && api.AllReduce;
        return api;
    }

    zr_status NcclFail(int rc, const char* what)
    {
        const NcclApi& a = Api();
        zr::set_error("%s: NCCL error %d (%s)", what, rc, a.GetErrorString ? a.GetErrorString(rc) : "?");
        return ZR_ERR_CUDA;
    }
}
#define ZR_NCCL(expr) do { int rc__ = (expr); if (rc__ != 0) return NcclFail(rc__, #expr); } while (0)

struct zr_comm
{
    int rank = 0, world = 1;
    NcclComm comm[2] = { nullptr, nullptr };       // [0] main streams, [1] second stream (DirectLighting): never used by two streams at once
    zr_comm_transport transport{};                  // set (and comm[] unused) for a comm made by zr_comm_create_transport
    void* user = nullptr;
    uint64_t bytesSent = 0, calls = 0;
    bool external() const { return transport.exchange_halos != nullptr; }
};

namespace
{
    // one grouped call (zr_comm_exchange_halos)
    zr_status NcclExchangeHalos(zr_comm* c, int which_comm, const uint32_t* bounds, uint32_t halo, const zr_image2d* planes, int n_planes,
        cudaStream_t stream)
    {
        NcclApi& a = Api();
        const int r = c->rank;
        auto bands = [&](int q, uint32_t& t0, uint32_t& t1, uint32_t& b0, uint32_t& b1)
        {
            const uint32_t y0 = bounds[q], y1 = bounds[q + 1];
            t0 = y0; t1 = y0 + halo < y1 ? y0 + halo : y1;
            b0 = y1 > y0 + halo ? y1 - halo : y0; b1 = y1;
        };
        uint32_t t0, t1, b0, b1;
        bands(r, t0, t1, b0, b1);
        ZR_NCCL(a.GroupStart());
        for (int i = 0; i < n_planes; i++)
        {
            unsigned char* base = (unsigned char*)planes[i].d_ptr;
            const size_t pitch = planes[i].pitch_bytes;
            if (r > 0)
            {
                uint32_t nt0, nt1, nb0, nb1;
                bands(r - 1, nt0, nt1, nb0, nb1);
                ZR_NCCL(a.Send(base + (size_t)t0 * pitch, (size_t)(t1 - t0) * pitch, NCCL_UINT8, r - 1, c->comm[which_comm], stream));
                ZR_NCCL(a.Recv(base + (size_t)nb0 * pitch, (size_t)(nb1 - nb0) * pitch, NCCL_UINT8, r - 1, c->comm[which_comm], stream));
            }
            if (r < c->world - 1)
            {
                uint32_t nt0, nt1, nb0, nb1;
                bands(r + 1, nt0, nt1, nb0, nb1);
                ZR_NCCL(a.Send(base + (size_t)b0 * pitch, (size_t)(b1 - b0) * pitch, NCCL_UINT8, r + 1, c->comm[which_comm], stream));
                ZR_NCCL(a.Recv(base + (size_t)nt0 * pitch, (size_t)(nt1 - nt0) * pitch, NCCL_UINT8, r + 1, c->comm[which_comm], stream));
            }
        }
        ZR_NCCL(a.GroupEnd());
        return ZR_OK;
    }

    zr_status NcclGatherRows(zr_comm* c, const uint32_t* bounds, const zr_image2d* plane, int root, cudaStream_t stream)
    {
        NcclApi& a = Api();
        unsigned char* base = (unsigned char*)plane->d_ptr;
        const size_t pitch = plane->pitch_bytes;
        ZR_NCCL(a.GroupStart());
        if (c->rank == root)
        {
            for (int q = 0; q < c->world; q++)
                if (q != root)
                    ZR_NCCL(a.Recv(base + (size_t)bounds[q] * pitch, (size_t)(bounds[q + 1] - bounds[q]) * pitch, NCCL_UINT8, q, c->comm[0], stream));
        }
        else
            ZR_NCCL(a.Send(base + (size_t)bounds[c->rank] * pitch, (size_t)(bounds[c->rank + 1] - bounds[c->rank]) * pitch, NCCL_UINT8, root, c->comm[0], stream));
        ZR_NCCL(a.GroupEnd());
        return ZR_OK;
    }

    zr_status TransportStatus(zr_status s, const char* what)
    {
        if (s != ZR_OK) zr::set_error("%s: the caller's transport returned %d", what, (int)s);
        return s;
    }
}

extern "C"
{
    zr_status zr_comm_unique_id(void* out128)
    {
        if (!out128) return ZR_ERR_INVALID_ARG;
        NcclApi& a = Api();
        if (!a.ok) { zr::set_error("zr_comm_unique_id: libnccl.so.2 not found"); return ZR_ERR_NOT_INITIALIZED; }
        NcclUniqueId id[2];
        ZR_NCCL(a.GetUniqueId(&id[0]));
        ZR_NCCL(a.GetUniqueId(&id[1]));
        memcpy(out128, id, sizeof(id));
        return ZR_OK;
    }

    // id256: what zr_comm_unique_id produced on rank 0 (256 bytes: two NCCL ids), distributed to every rank by the caller
    zr_status zr_comm_create(const void* id256, int rank, int world, zr_comm** out)
    {
        if (!id256 || !out || world < 1 || rank < 0 || rank >= world) { zr::set_error("zr_comm_create: bad args"); return ZR_ERR_INVALID_ARG; }
        NcclApi& a = Api();
        if (!a.ok) { zr::set_error("zr_comm_create: libnccl.so.2 not found"); return ZR_ERR_NOT_INITIALIZED; }
        zr_comm* c = new zr_comm();
        c->rank = rank; c->world = world;
        NcclUniqueId id[2];
        memcpy(id, id256, sizeof(id));
        for (int i = 0; i < 2; i++)
        {
            const int rc = a.CommInitRank(&c->comm[i], world, id[i], rank);
            if (rc != 0) { delete c; return NcclFail(rc, "ncclCommInitRank"); }
        }
        *out = c;
        return ZR_OK;
    }

    zr_status zr_comm_create_transport(const zr_comm_transport* t, void* user, int rank, int world, zr_comm** out)
    {
        if (!t || !out || !t->exchange_halos || !t->gather_rows || !t->allreduce_u32 || world < 1 || rank < 0 || rank >= world)
        {
            zr::set_error("zr_comm_create_transport: bad args (three callbacks and 0 <= rank < world)");
            return ZR_ERR_INVALID_ARG;
        }
        zr_comm* c = new zr_comm();
        c->rank = rank; c->world = world;
        c->transport = *t;
        c->user = user;
        *out = c;
        return ZR_OK;
    }

    void zr_comm_destroy(zr_comm* c)
    {
        if (!c) return;
        for (int i = 0; i < 2; i++) if (c->comm[i]) Api().CommDestroy(c->comm[i]);
        delete c;
    }

    zr_status zr_comm_rank(zr_comm* c, int* rank, int* world)
    {
        if (!c) return ZR_ERR_INVALID_ARG;
        if (rank) *rank = c->rank;
        if (world) *world = c->world;
        return ZR_OK;
    }
    zr_status zr_comm_stats(zr_comm* c, uint64_t* bytes_sent, uint64_t* calls)
    {
        if (!c) return ZR_ERR_INVALID_ARG;
        if (bytes_sent) *bytes_sent = c->bytesSent;
        if (calls) *calls = c->calls;
        return ZR_OK;
    }

    // Makes the boundary bands of `planes` coherent between neighbouring strips: this rank's top / bottom `halo` rows go to the strip
    // above / below, their facing bands arrive in the rows just outside [bounds[rank], bounds[rank + 1]).
    zr_status zr_comm_exchange_halos(zr_comm* c, int which_comm, const uint32_t* bounds, uint32_t halo, const zr_image2d* planes, int n_planes,
        void* stream)
    {
        if (!c || !bounds || !planes || n_planes < 1 || which_comm < 0 || which_comm > 1) return ZR_ERR_INVALID_ARG;
        if (c->world == 1) return ZR_OK;
        const zr_status s = c->external()
            ? TransportStatus(c->transport.exchange_halos(c->user, which_comm, bounds, halo, planes, n_planes, stream), "zr_comm_exchange_halos")
            : NcclExchangeHalos(c, which_comm, bounds, halo, planes, n_planes, (cudaStream_t)stream);
        if (s != ZR_OK) return s;
        // both bands are min(halo, strip height) rows; the first strip has no band above, the last none below
        const uint32_t rows = bounds[c->rank + 1] - bounds[c->rank] < halo ? bounds[c->rank + 1] - bounds[c->rank] : halo;
        const int bands = (c->rank > 0) + (c->rank < c->world - 1);
        for (int i = 0; i < n_planes; i++) c->bytesSent += (uint64_t)bands * rows * planes[i].pitch_bytes;
        c->calls++;
        return ZR_OK;
    }

    // Every rank's own rows of `plane` arrive on rank `root` (the other ranks keep only their strip).
    zr_status zr_comm_gather_rows(zr_comm* c, const uint32_t* bounds, const zr_image2d* plane, int root, void* stream)
    {
        if (!c || !bounds || !plane || root < 0 || root >= c->world) return ZR_ERR_INVALID_ARG;
        if (c->world == 1) return ZR_OK;
        const zr_status s = c->external()
            ? TransportStatus(c->transport.gather_rows(c->user, bounds, plane, root, stream), "zr_comm_gather_rows")
            : NcclGatherRows(c, bounds, plane, root, (cudaStream_t)stream);
        if (s != ZR_OK) return s;
        if (c->rank != root) c->bytesSent += (uint64_t)(bounds[c->rank + 1] - bounds[c->rank]) * plane->pitch_bytes;
        return ZR_OK;
    }

    zr_status zr_comm_allreduce_u32(zr_comm* c, int which_comm, uint32_t* d_values, uint32_t n, void* stream)
    {
        if (!c || !d_values || which_comm < 0 || which_comm > 1) return ZR_ERR_INVALID_ARG;
        if (c->world == 1) return ZR_OK;
        if (c->external())
            return TransportStatus(c->transport.allreduce_u32(c->user, which_comm, d_values, n, stream), "zr_comm_allreduce_u32");
        ZR_NCCL(Api().AllReduce(d_values, d_values, n, NCCL_UINT32, NCCL_SUM, c->comm[which_comm], (cudaStream_t)stream));
        return ZR_OK;
    }
}
