// Multi-GPU exchange of node-range sharding: NCCL (loaded with dlopen), the row exchange after a sweep, the fused
// peer-store epochs (K5) and the hrag_comm_* / hrag_p2p_* entries.
#include <dlfcn.h>

#include <cstring>

#include "handle.h"

namespace hrag {

// ---- NCCL through dlopen: only sharded runs need it ---------------------------------------

static int load_nccl() {
    if (g_nccl.lib) return 0;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
        g_nccl.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (g_nccl.lib) break;
    }
    HRAG_CHECK(g_nccl.lib != nullptr, "cannot dlopen libnccl.so.2 (needed for node-range sharding)");
#define HRAG_SYM(field, name)                                                         \
    *(void**)(&g_nccl.field) = dlsym(g_nccl.lib, name);                               \
    HRAG_CHECK(g_nccl.field != nullptr, std::string("libnccl lacks ") + name)
    HRAG_SYM(GetUniqueId, "ncclGetUniqueId");
    HRAG_SYM(CommInitRank, "ncclCommInitRank");
    HRAG_SYM(CommDestroy, "ncclCommDestroy");
    HRAG_SYM(AllGather, "ncclAllGather");
    HRAG_SYM(AllReduce, "ncclAllReduce");
    HRAG_SYM(Broadcast, "ncclBroadcast");
    HRAG_SYM(GroupStart, "ncclGroupStart");
    HRAG_SYM(GroupEnd, "ncclGroupEnd");
    HRAG_SYM(GetErrorString, "ncclGetErrorString");
#undef HRAG_SYM
    return 0;
}

// After a sweep wrote the owned rows of y: make every rank hold all rows (node-range sharding).
int exchange_rows_bytes(hrag_t* h, void* y, size_t row_bytes) {
    if (h->world == 1) return 0;
    StageTimer tm(h, ST_COMM);
    if (!h->row_bounds.empty()) {            // unequal ranges: one broadcast per owner, grouped into one NCCL operation
        HRAG_NCCL(g_nccl.GroupStart());
        for (int r = 0; r < h->world; ++r) {
            char* p = static_cast<char*>(y) + (size_t)h->row_bounds[r] * row_bytes;
            const size_t cnt = (size_t)(h->row_bounds[r + 1] - h->row_bounds[r]) * row_bytes;
            if (cnt) HRAG_NCCL(g_nccl.Broadcast(p, p, cnt, ncclInt8, r, h->comm, h->stream));
        }
        HRAG_NCCL(g_nccl.GroupEnd());
        return 0;
    }
    const size_t count = (size_t)h->chunk_rows * row_bytes;
    HRAG_NCCL(g_nccl.AllGather(static_cast<char*>(y) + (size_t)h->rank * count, y, count, ncclInt8, h->comm,
                               h->stream));
    return 0;
}
int exchange_rows(hrag_t* h, float* y, int B) { return exchange_rows_bytes(h, y, (size_t)B * sizeof(float)); }

PeerOut peers_for(hrag_t* h, void* y) {
    PeerOut po;
    if (!h->p2p) return po;
    const size_t off = static_cast<char*>(y) - static_cast<char*>(h->slab.p);
    for (int r = 0; r < h->world; ++r)
        if (r != h->rank) po.y[po.n++] = static_cast<char*>(h->peer_slab[r]) + off;
    return po;
}
// K5 epochs.  Every exchange point of the sharded solver is one epoch: all ranks run the same sequence, a rank
// waits until every peer has published everything up to the previous point and then publishes its own.  A sweep
// carries both halves itself (first instruction of every CTA / last CTA out); the two places where a non-sweep
// kernel touches exchanged state use the stand-alone wait / signal kernels.
SweepSync sync_for_sweep(hrag_t* h) {
    SweepSync sy;
    if (!h->p2p) return sy;
    sy.flags = epoch_flags(h, h->slab.p);
    sy.need = h->epoch;
    sy.world = h->world;
    sy.rank = h->rank;
    sy.error_flag = h->p2p_err.as<int>();
    sy.done_ctr = h->done_ctr.as<unsigned int>();
    for (int r = 0; r < h->world; ++r)
        if (r != h->rank) sy.remote[sy.n_remote++] = epoch_flags(h, h->peer_slab[r]) + h->rank;
    h->epoch += 1;
    sy.epoch = h->epoch;
    return sy;
}
int p2p_wait(hrag_t* h) {
    if (!h->p2p) return 0;
    SweepSync sy = sync_for_sweep(h);
    h->epoch -= 1;                       // a pure wait publishes nothing
    sy.need = h->epoch;
    StageTimer tc(h, ST_COMM);
    return epoch_wait(sy, h->stream);
}
int p2p_signal(hrag_t* h) {
    if (!h->p2p) return 0;
    const SweepSync sy = sync_for_sweep(h);
    StageTimer tc(h, ST_COMM);
    return epoch_signal(sy, h->stream);
}

}  // namespace hrag

using namespace hrag;

extern "C" {

int hrag_comm_unique_id(void* id128) {
    HRAG_TRY(load_nccl());
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    HRAG_NCCL(g_nccl.GetUniqueId(reinterpret_cast<ncclUniqueId*>(id128)));
    return 0;
}

int hrag_comm_init(hrag_t* h, const void* id128, int rank, int world) {
    HRAG_CHECK(h && id128, "hrag_comm_init: null argument");
    HRAG_CHECK(world >= 1 && rank >= 0 && rank < world, "hrag_comm_init: bad rank/world");
    HRAG_TRY(load_nccl());
    HRAG_CUDA(cudaSetDevice(h->device));
    ncclUniqueId id;
    memcpy(&id, id128, sizeof(id));
    HRAG_NCCL(g_nccl.CommInitRank(&h->comm, world, id, rank));
    h->rank = rank;
    h->world = world;
    return 0;
}

int hrag_comm_set_row_bounds(hrag_t* h, const int64_t* bounds, int world) {
    HRAG_CHECK(h && bounds, "hrag_comm_set_row_bounds: null argument");
    HRAG_CHECK(world == h->world && world >= 1, "hrag_comm_set_row_bounds: world must match hrag_comm_init");
    HRAG_CHECK(!h->p2p, "hrag_comm_set_row_bounds: set the partition before hrag_p2p_export / import");
    HRAG_CHECK(bounds[0] == 0, "hrag_comm_set_row_bounds: bounds[0] must be 0");
    for (int r = 0; r < world; ++r) HRAG_CHECK(bounds[r] <= bounds[r + 1], "hrag_comm_set_row_bounds: bounds must not decrease");
    h->row_bounds.assign(bounds, bounds + world + 1);
    return 0;
}

int hrag_p2p_export(hrag_t* h, void* handle64) {
    HRAG_CHECK(h && handle64, "hrag_p2p_export: null argument");
    HRAG_CHECK(h->g.n_global > 0, "hrag_p2p_export: load the graph first");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    HRAG_CUDA(cudaSetDevice(h->device));
    HRAG_TRY(ensure_state_mixed(h));
    cudaIpcMemHandle_t mh;
    HRAG_CUDA(cudaIpcGetMemHandle(&mh, h->slab.p));
    memcpy(handle64, &mh, 64);
    return 0;
}

int hrag_p2p_import(hrag_t* h, const void* handles, int world) {
    HRAG_CHECK(h && handles, "hrag_p2p_import: null argument");
    HRAG_CHECK(world == h->world && world >= 2 && world <= 8, "hrag_p2p_import: world must match hrag_comm_init (2..8)");
    HRAG_CHECK(h->slab.p != nullptr, "hrag_p2p_import: call hrag_p2p_export first");
    HRAG_CUDA(cudaSetDevice(h->device));
    for (int r = 0; r < world; ++r) {
        if (r == h->rank) continue;
        cudaIpcMemHandle_t mh;
        memcpy(&mh, static_cast<const char*>(handles) + (size_t)r * 64, 64);
        HRAG_CUDA(cudaIpcOpenMemHandle(&h->peer_slab[r], mh, cudaIpcMemLazyEnablePeerAccess));
    }
    h->p2p = true;
    h->epoch = 0;
    return 0;
}

}  // extern "C"
