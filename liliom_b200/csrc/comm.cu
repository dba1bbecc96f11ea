// Multi-GPU plumbing: NCCL is resolved at run time with dlopen so that single-GPU users need no
// NCCL at all, and so that inside a PyTorch process the already-loaded libnccl.so.2 is reused.
// The only collective on the path is the per-iteration all-reduce of the 29 fp64 scalars
// (21 J^T J + 6 J^T r + cost + count): 232 bytes, latency-bound over NVLink 5 / NVSwitch.
#include "ctx.cuh"
#include <dlfcn.h>

namespace lili {

struct Id128 { char b[128]; };   // ncclUniqueId (passed by value)

struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, Id128, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};

static NcclApi g_nccl;

static bool load_nccl(std::string* err) {
    if (g_nccl.lib) return true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
        g_nccl.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (g_nccl.lib) break;
    }
    if (!g_nccl.lib) { if (err) *err = std::string("dlopen libnccl.so.2 failed: ") + dlerror(); return false; }
    g_nccl.GetUniqueId = (int (*)(void*))dlsym(g_nccl.lib, "ncclGetUniqueId");
    g_nccl.CommInitRank = (int (*)(void**, int, Id128, int))dlsym(g_nccl.lib, "ncclCommInitRank");
    g_nccl.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(g_nccl.lib, "ncclAllReduce");
    g_nccl.CommDestroy = (int (*)(void*))dlsym(g_nccl.lib, "ncclCommDestroy");
    g_nccl.GetErrorString = (const char* (*)(int))dlsym(g_nccl.lib, "ncclGetErrorString");
    if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce) {
        if (err) *err = "libnccl is missing ncclGetUniqueId/ncclCommInitRank/ncclAllReduce";
        return false;
    }
    return true;
}

int nccl_allreduce_sum_f64(liliom_ctx* c, double* buf, int count) {
    if (!c->nccl_comm) return LILIOM_E_NCCL;
    // ncclFloat64 = 8, ncclSum = 0
    int r = g_nccl.AllReduce(buf, buf, (size_t)count, 8, 0, c->nccl_comm, c->stream);
    if (r != 0) {
        c->last_error = std::string("ncclAllReduce: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "error");
        return LILIOM_E_NCCL;
    }
    c->cnt.lib_launches++;
    return LILIOM_OK;
}

void nccl_destroy(liliom_ctx* c) {
    if (c->nccl_comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->nccl_comm);
    c->nccl_comm = nullptr;
    for (int p = 0; p < kMaxPeers; ++p) {      // peer mappings of the fused exchange (own buffer is a DevBuf)
        if (c->peer_ptrs[p] && c->peer_ptrs[p] != c->peer_buf.p) cudaIpcCloseMemHandle(c->peer_ptrs[p]);
        c->peer_ptrs[p] = nullptr;
    }
    c->peer_ready = false;
    c->peer_buf.release();
    c->peer_local.release();
}

}  // namespace lili

extern "C" int liliom_comm_get_unique_id(void* id128) {
    if (!id128) return LILIOM_E_ARG;
    std::string err;
    if (!lili::load_nccl(&err)) return LILIOM_E_NCCL;
    return lili::g_nccl.GetUniqueId(id128) == 0 ? LILIOM_OK : LILIOM_E_NCCL;
}

extern "C" int liliom_comm_init(liliom_ctx* c, const void* id128, int nranks, int rank) {
    if (!c || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return LILIOM_E_ARG;
    std::string err;
    if (!lili::load_nccl(&err)) { c->last_error = err; return LILIOM_E_NCCL; }
    LILI_CUDA(c, cudaSetDevice(c->device));
    lili::Id128 id;
    memcpy(id.b, id128, 128);
    void* comm = nullptr;
    int r = lili::g_nccl.CommInitRank(&comm, nranks, id, rank);
    if (r != 0) {
        c->last_error = std::string("ncclCommInitRank: ") + (lili::g_nccl.GetErrorString ? lili::g_nccl.GetErrorString(r) : "error");
        return LILIOM_E_NCCL;
    }
    c->nccl_comm = comm;
    c->nranks = nranks;
    c->rank = rank;
    return LILIOM_OK;
}

extern "C" int liliom_comm_set_shard_block(liliom_ctx* c, int metres) {
    if (!c || metres < 8 || metres > 256 || (metres & (metres - 1)) != 0) return LILIOM_E_ARG;
    c->shard_inv_block = 1.0f / (float)metres;
    return LILIOM_OK;
}

// ---- fused exchange over NVLink / NVSwitch peer memory (SURVEY.md §8 e, "one kernel that does both") -------------------------
// The NCCL path costs, per GN iteration, a kernel, an all-reduce of 232 bytes (tens of microseconds of latency on 2 GPUs, more than the
// sharded search saves at 1.4k queries) and an update kernel.  Here every rank runs its persistent GN kernel; after the local
// grid reduction block 0 stores the rank's 29 sums straight into EVERY peer's exchange buffer (flag-in-data words, system scope)
// and all blocks read the ranks' sums from their own buffer: all iterations of a scan in one launch per rank, no collective call.
static size_t peer_buf_bytes() { return (size_t)2 * lili::kMaxPeers * 32 * sizeof(ulonglong2); }

extern "C" int liliom_comm_peer_export(liliom_ctx* c, void* handle64) {
    if (!c || !handle64) return LILIOM_E_ARG;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (!c->peer_buf.p) {
        LILI_CUDA(c, c->peer_buf.ensure(peer_buf_bytes()));
        LILI_CUDA(c, cudaMemset(c->peer_buf.p, 0, c->peer_buf.cap));      // epochs start at 1: a zero word never matches
        LILI_CUDA(c, c->peer_local.ensure(1024));
        LILI_CUDA(c, cudaMemset(c->peer_local.p, 0, c->peer_local.cap));
        c->peer_epoch = 0;
    }
    cudaIpcMemHandle_t h;
    LILI_CUDA(c, cudaIpcGetMemHandle(&h, c->peer_buf.p));
    memcpy(handle64, &h, 64);
    return LILIOM_OK;
}

extern "C" int liliom_comm_peer_attach(liliom_ctx* c, const void* handles, int nranks, int rank) {
    if (!c || !handles || nranks < 1 || nranks > lili::kMaxPeers || rank < 0 || rank >= nranks) return LILIOM_E_ARG;
    LILI_CUDA(c, cudaSetDevice(c->device));
    if (!c->peer_buf.p) { c->last_error = "liliom_comm_peer_attach: call liliom_comm_peer_export first"; return LILIOM_E_ARG; }
    if (c->nranks != nranks || c->rank != rank) {
        if (nranks > 1 && !c->nccl_comm) { c->last_error = "liliom_comm_peer_attach: call liliom_comm_init first (map sharding and the map-size guard use it)"; return LILIOM_E_ARG; }
        if (nranks > 1) { c->last_error = "liliom_comm_peer_attach: nranks/rank differ from liliom_comm_init"; return LILIOM_E_ARG; }
    }
    for (int p = 0; p < nranks; ++p) {
        if (p == rank) { c->peer_ptrs[p] = c->peer_buf.p; continue; }
        cudaIpcMemHandle_t h;
        memcpy(&h, (const char*)handles + (size_t)p * 64, 64);
        void* ptr = nullptr;
        LILI_CUDA(c, cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
        c->peer_ptrs[p] = ptr;
    }
    c->peer_ready = true;
    return LILIOM_OK;
}

// ADVICE r1: no way back after one lost exchange (the survivors' epochs ran ahead of the lost rank's) — see include/liliom.h
extern "C" int liliom_comm_peer_epoch(liliom_ctx* c, unsigned int* epoch) {
    if (!c || !epoch) return LILIOM_E_ARG;
    *epoch = c->peer_epoch;
    return LILIOM_OK;
}

extern "C" int liliom_comm_peer_set_epoch(liliom_ctx* c, unsigned int epoch) {
    if (!c) return LILIOM_E_ARG;
    if (epoch < c->peer_epoch) { c->last_error = "liliom_comm_peer_set_epoch: epochs only move forward (stale words in the exchange buffers must stay older)"; return LILIOM_E_ARG; }
    c->peer_epoch = epoch;
    return LILIOM_OK;
}
