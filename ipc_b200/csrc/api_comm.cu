// api_comm.cu -- the cross-rank layer: NCCL loaded at run time, the communicator entry points and the typed collectives every other
// translation unit issues its reductions through (abi.h).
#include "abi.h"
#include <cstring>
#include <dlfcn.h>

// ---------------------------------------------------------------------------------------------------
// NCCL through dlopen: the library that torch already loaded (libnccl.so.2) is reused when present.
// ---------------------------------------------------------------------------------------------------
namespace {
struct Id128 {
    char b[128];
};
struct Nccl {
    void* h = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, /* ncclUniqueId by value: 128 bytes */ Id128, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
Nccl g_nccl;
bool nccl_load(std::string& err)
{
    if (g_nccl.h) return true;
    const char* names[] = { "libnccl.so.2", "libnccl.so" };
    for (const char* n : names) {
        g_nccl.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (g_nccl.h) break;
    }
    if (!g_nccl.h) {
        err = "dlopen(libnccl.so.2) failed";
        return false;
    }
    g_nccl.GetUniqueId = (int (*)(void*))dlsym(g_nccl.h, "ncclGetUniqueId");
    g_nccl.CommInitRank = (int (*)(void**, int, Id128, int))dlsym(g_nccl.h, "ncclCommInitRank");
    g_nccl.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(g_nccl.h, "ncclAllReduce");
    g_nccl.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(g_nccl.h, "ncclAllGather");
    g_nccl.CommDestroy = (int (*)(void*))dlsym(g_nccl.h, "ncclCommDestroy");
    g_nccl.GetErrorString = (const char* (*)(int))dlsym(g_nccl.h, "ncclGetErrorString");
    if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.AllGather) {
        err = "NCCL symbols missing";
        return false;
    }
    return true;
}
constexpr int kNcclInt32 = 2;   // ncclInt32
constexpr int kNcclFloat64 = 8; // ncclDouble
constexpr int kNcclUint64 = 5;  // ncclUint64
constexpr int kNcclSum = 0, kNcclMin = 3;

int all_reduce(ipcgpu_ctx* ctx, void* buf, size_t n, int type, int op, const char* what)
{
    if (ctx->nranks <= 1) return IPCGPU_OK;
    int r = g_nccl.AllReduce(buf, buf, n, type, op, ctx->nccl_comm, ctx->stream);
    REQUIRE(r == 0, IPCGPU_ERR_NCCL, what);
    return IPCGPU_OK;
}
} // namespace

int nccl_sum(ipcgpu_ctx* ctx, double* buf, size_t n, const char* what) { return all_reduce(ctx, buf, n, kNcclFloat64, kNcclSum, what); }
int nccl_sum(ipcgpu_ctx* ctx, int* buf, size_t n, const char* what) { return all_reduce(ctx, buf, n, kNcclInt32, kNcclSum, what); }

int nccl_min_u64(ipcgpu_ctx* ctx, unsigned long long* word)
{
    if (ctx->nranks <= 1) return IPCGPU_OK;
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ALLREDUCE);
    int rc = all_reduce(ctx, word, 1, kNcclUint64, kNcclMin, "ncclAllReduce(min step) failed");
    ctx->prof_end(pe);
    return rc;
}

int nccl_all_gather(ipcgpu_ctx* ctx, const int4* send, int4* recv, size_t n, const char* what)
{
    int r = g_nccl.AllGather(send, recv, n * 4, kNcclInt32, ctx->nccl_comm, ctx->stream);
    REQUIRE(r == 0, IPCGPU_ERR_NCCL, what);
    return IPCGPU_OK;
}

void nccl_comm_destroy(ipcgpu_ctx* ctx)
{
    if (ctx->nccl_comm && g_nccl.CommDestroy) g_nccl.CommDestroy(ctx->nccl_comm);
}

extern "C" {

int ipcgpu_comm_unique_id(void* id128)
{
    std::string err;
    if (!id128 || !nccl_load(err)) return IPCGPU_ERR_NCCL;
    return g_nccl.GetUniqueId(id128) == 0 ? IPCGPU_OK : IPCGPU_ERR_NCCL;
}

int ipcgpu_comm_init(ipcgpu_ctx* ctx, int rank, int nranks, const void* id128)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    REQUIRE(nranks >= 1 && rank >= 0 && rank < nranks, IPCGPU_ERR_ARG, "bad rank/nranks");
    REQUIRE(nranks == 1 || ctx->canonical_order != 2, IPCGPU_ERR_STATE, "the reproducible mode (canonical order level 2) runs on one rank");
    ctx->rank = rank;
    ctx->nranks = nranks;
    if (nranks > 1) {
        REQUIRE(id128 != nullptr, IPCGPU_ERR_ARG, "nccl unique id required for nranks>1");
        REQUIRE(nccl_load(ctx->err), IPCGPU_ERR_NCCL, ctx->err);
        Id128 id;
        std::memcpy(id.b, id128, 128);
        int r = g_nccl.CommInitRank(&ctx->nccl_comm, nranks, id, rank);
        REQUIRE(r == 0, IPCGPU_ERR_NCCL, std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"));
    }
    if (ctx->nT > 0) { // re-partition an already loaded mesh
        int rc = build_maps(ctx);
        if (rc) return rc;
        owned_value_range(ctx);
        if (ctx->surface_ready && (rc = contact_alloc(ctx))) return rc;
    }
    return IPCGPU_OK;
}

int ipcgpu_partition_info(ipcgpu_ctx* ctx, int* rank, int* nranks, int* tet_begin, int* tet_end, int* row_vertex_begin, int* row_vertex_end, int64_t* value_begin,
    int64_t* value_end, int* n_assembled_tets)
{
    if (rank) *rank = ctx->rank;
    if (nranks) *nranks = ctx->nranks;
    if (tet_begin) *tet_begin = ctx->t_begin;
    if (tet_end) *tet_end = ctx->t_end;
    if (row_vertex_begin) *row_vertex_begin = ctx->v_begin;
    if (row_vertex_end) *row_vertex_end = ctx->v_end;
    if (value_begin) *value_begin = ctx->a_begin;
    if (value_end) *value_end = ctx->a_end;
    if (n_assembled_tets) *n_assembled_tets = ctx->n_list;
    return IPCGPU_OK;
}

} // extern "C"
