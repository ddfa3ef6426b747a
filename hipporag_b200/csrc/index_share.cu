// One loaded index served to several processes on the same GPU: the owner exports the read-only allocations of its
// index through CUDA IPC (hrag_index_export), and handles in other processes map them (hrag_index_attach) instead of
// loading their own copy.  Each attached handle keeps everything a call writes -- streams, solver state, right-hand
// sides, scratch, captured solves, stats, the long-row segment partials, the synonymy KNN -- to itself; the shared
// allocations are only read at query time.
//
// What is shared, and why it is safe: the graph planes row_ptr, cv, row_order, long_rows, long_seg_ptr, segs and
// val_lo, the four seed tables, and per embedding matrix the bf16 hi / lo planes and the owned fp32 rows.  Query
// code never writes any of them: they are written by the loaders (ingest.cu, graph_build.cu install_graph) and the
// update entries (index_update.cu) only, and both are rejected on an exporting owner and on an attached handle
// (check_index_private).  graph.seg_partial is written by the long-row segment kernels in every sweep, so it stays
// per handle; the resident edge list (graph.edges) is kept only for updates and is not shared.
//
// Lifetime: cudaFree of an exported allocation while another process maps it is undefined, so an owner counts its
// attached handles in an 8-byte device counter it exports with the index.  Attach adds 1 and detach subtracts 1, each
// with a one-thread atomic kernel (two workers may attach at once); hrag_index_unexport is rejected while the count is
// non-zero, and hrag_destroy of an owner with live attachments leaves the exported allocations to the process exit.
// The owner process must outlive its workers.
#include <unistd.h>

#include <cstring>

#include "handle.h"

namespace hrag {
namespace {

constexpr char kShareMagic[8] = {'h', 'r', 'a', 'g', 'i', 'd', 'x', '\0'};
// Bumped whenever the layout of ShareBlob, or what its allocations hold, changes.
constexpr uint32_t kShareVersion = 1;

enum Alloc {
    A_ROW_PTR, A_CV, A_ROW_ORDER, A_LONG_ROWS, A_LONG_SEG_PTR, A_SEGS, A_VAL_LO,
    A_PASSAGE_VID, A_FACT_SUBJ, A_FACT_OBJ, A_CHUNK_COUNT,
    A_FACT_HI, A_FACT_LO, A_FACT_F32, A_PASS_HI, A_PASS_LO, A_PASS_F32,
    A_COUNTER, kAllocs
};
struct SharedAlloc {
    cudaIpcMemHandle_t handle;
    uint64_t bytes;          // 0: the owner holds no such allocation
};
// The blob hrag_index_export writes: self-describing, fixed size, read back field by field by hrag_index_attach.
struct ShareBlob {
    char magic[8];
    uint32_t version;
    uint32_t blob_bytes;     // sizeof(ShareBlob) of the writer
    unsigned char uuid[16];  // cudaDeviceProp::uuid of the owner's GPU (ordinals differ under CUDA_VISIBLE_DEVICES)
    int64_t owner_pid;
    int32_t n_global, row_lo, n_rows, long_thresh, n_long, n_seg, max_batch, has_val_lo;   // PprGraph
    int64_t nnz;
    int32_t t_nodes, t_passages;                                                         // SeedTables
    int64_t t_facts;
    int32_t dim, n_bounds;
    int64_t bounds[2];       // row_bounds of a one-GPU handle: empty, or {0, N}
    int64_t emb_rows[2], n_facts_global;
    SharedAlloc alloc[kAllocs];
};
static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
static_assert(sizeof(ShareBlob) % 8 == 0, "ShareBlob is padded to 8 bytes");

__global__ void k_attach_count(unsigned long long* counter, long long delta) {
    atomicAdd(counter, (unsigned long long)delta);
}

// counter += delta on the handle's stream, then synchronised
int count_attach(hrag_t* h, long long delta) {
    k_attach_count<<<1, 1, 0, h->stream>>>(h->share.counter.as<unsigned long long>(), delta);
    HRAG_CUDA(cudaGetLastError());
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    return 0;
}

int read_count(const hrag_t* h, int64_t* n) {
    HRAG_CUDA(cudaMemcpy(n, h->share.counter.p, sizeof(int64_t), cudaMemcpyDeviceToHost));
    return 0;
}

// The handle's Buf of every shared allocation, in Alloc order (the counter last).
void shared_bufs(hrag_t* h, Buf* (&out)[kAllocs]) {
    GraphMem& G = h->graph;
    TableMem& T = h->tables;
    Buf* b[kAllocs] = {&G.row_ptr, &G.cv, &G.row_order, &G.long_rows, &G.long_seg_ptr, &G.segs, &G.val_lo,
                       &T.passage_vid, &T.fact_subj_vid, &T.fact_obj_vid, &T.ent_chunk_count,
                       &h->emb[0].hi, &h->emb[0].lo, &h->emb[0].own, &h->emb[1].hi, &h->emb[1].lo, &h->emb[1].own,
                       &h->share.counter};
    for (int i = 0; i < kAllocs; ++i) out[i] = b[i];
}

// Device bytes of the handle's own allocations (not the mapped ones).
int64_t owned_device_bytes(const hrag_t* h) {
    int64_t n = 0;
    auto add = [&](const Buf& b) { if (!b.ipc) n += (int64_t)b.cap; };
    const GraphMem& G = h->graph;
    for (const Buf* b : {&G.row_ptr, &G.cv, &G.row_order, &G.long_rows, &G.long_seg_ptr, &G.segs, &G.seg_partial,
                         &G.val_lo, &G.edges.src, &G.edges.dst, &G.edges.w})
        add(*b);
    const TableMem& T = h->tables;
    for (const Buf* b : {&T.passage_vid, &T.fact_subj_vid, &T.fact_obj_vid, &T.ent_chunk_count}) add(*b);
    for (const EmbMem& e : h->emb) for (const Buf* b : {&e.own, &e.hi, &e.lo}) add(*b);
    const FactPlanes& fp = h->fplanes;
    for (const Buf* b : {&fp.ring, &fp.run_mm, &fp.run_keys, &fp.sl_ids, &fp.sl_scores, &fp.sl_mm, &fp.tail}) add(*b);
    for (const Buf* b : {&h->knn.hi, &h->knn.lo, &h->knn.ids, &h->knn.scores}) add(*b);
    add(h->share.counter);
    for (const Buf* b : {&h->V, &h->XA, &h->XC, &h->partials, &h->sums, &h->X64, &h->V64, &h->io64, &h->part64,
                         &h->sums64, &h->slab, &h->slab_pair, &h->mixed_part[0], &h->mixed_part[1], &h->mixed_sums,
                         &h->rho, &h->p2p_err, &h->done_ctr, &h->prep_scratch})
        add(*b);
    for (const RhsSet& r : h->rhs)
        for (const Buf* b : {&r.slot_map, &r.slot_vid, &r.Vc, &r.R16, &r.scale, &r.vsum}) add(*b);
    for (const Buf* b : {&h->S_fact, &h->S_pass, &h->mm_fact, &h->mm_pass, &h->mode, &h->seed_vid, &h->seed_w,
                         &h->q_hi, &h->q_lo, &h->part_mm, &h->part_keys, &h->part_bound, &h->xr_mm, &h->xr_keys,
                         &h->fs_top_idx, &h->fs_top_score, &h->fs_nvalid, &h->d_q, &h->d_q2, &h->d_top_idx,
                         &h->d_top_score, &h->d_nvalid, &h->d_kept_idx, &h->d_kept_score, &h->d_dpr, &h->d_out_ids,
                         &h->d_out_scores, &h->d_reset, &h->d_scores, &h->pipe.top_idx, &h->pipe.top_score,
                         &h->pipe.nvalid, &h->pipe.S_pass, &h->pipe.mm_pass})
        add(*b);
    return n;
}

bool holds_index(const hrag_t* h) { return h->g.cv || h->t.passage_vid || h->dim > 0 || emb_planes(h, 0).streams(); }

// The attached handle's index goes: every mapping is closed (Buf::reset bumps g_buf_generation, so no captured solve
// that points into them is replayed).  The caller has synchronised `stream`.
void drop_attached_index(hrag_t* h) {
    h->graph = GraphMem{};
    h->g = PprGraph();
    h->tables = TableMem{};
    h->t = SeedTables();
    h->emb[0] = EmbMem{};
    h->emb[1] = EmbMem{};
    h->dim = 0;
    h->n_facts_global = h->fact_row_lo = 0;
    h->row_bounds.clear();
    h->chunk_rows = 0;
}

}  // namespace

int check_index_private(const hrag_t* h, const std::string& who) {
    HRAG_CHECK(h->share.role != SHARE_OWNER,
               who + ": the index is exported to other processes (hrag_index_export) and must not change; have every "
                     "attached handle detach, call hrag_index_unexport, then load or update it");
    HRAG_CHECK(h->share.role != SHARE_ATTACHED,
               who + ": the handle is attached to another process's index (hrag_index_attach), which it only reads; "
                     "call hrag_index_detach first");
    return 0;
}

void index_share_destroy(hrag_t* h) {
    if (h->share.role == SHARE_ATTACHED) {
        hrag_index_detach(h);
        return;
    }
    if (h->share.role != SHARE_OWNER) return;
    int64_t n = 1;
    if (read_count(h, &n) == 0 && n == 0) return;   // nobody maps the index: the buffers free themselves
    // Other processes still map the exported allocations (or the count could not be read): freeing them would be
    // undefined behaviour in those processes, so they stay allocated until this process exits.
    Buf* bufs[kAllocs];
    shared_bufs(h, bufs);
    for (Buf* b : bufs) { b->p = nullptr; b->cap = 0; }
}

}  // namespace hrag

using namespace hrag;

extern "C" {

int hrag_index_export(hrag_t* h, void* blob, int64_t cap, int64_t* size) {
    const std::string who = "hrag_index_export";
    HRAG_CHECK(h && size, who + ": null argument");
    *size = (int64_t)sizeof(ShareBlob);
    if (!blob) return 0;
    HRAG_CHECK(cap >= (int64_t)sizeof(ShareBlob), who + ": the blob needs " + std::to_string(sizeof(ShareBlob)) +
                                                      " bytes, " + std::to_string(cap) + " given");
    HRAG_CHECK(h->share.role != SHARE_ATTACHED,
               who + ": the handle is attached to another process's index; only the process that loaded it exports it");
    HRAG_CHECK(h->g.cv && h->t.passage_vid && h->dim > 0, who + ": no index loaded (graph, tables and embeddings)");
    HRAG_CHECK(h->world == 1, who + ": a node-range-sharded handle (world > 1) cannot be shared");
    HRAG_CHECK(!emb_planes(h, 0).streams(), who + ": the fact planes are held in pinned host memory (hrag_set_fact_memory), "
                                         "which belongs to this process alone; load them resident to share the index");
    for (int w = 0; w < 2; ++w)
        HRAG_CHECK(!(h->emb[w].f32 && !h->emb[w].own.p),
                   who + ": the fp32 " + (w ? "passage" : "fact") + " rows are borrowed from the caller (device load); "
                   "load them from host memory to share the index");
    HRAG_CHECK(h->row_bounds.size() <= 2, "internal: " + who + ": row bounds of a one-GPU handle");
    HRAG_CUDA(cudaSetDevice(h->device));
    cudaDeviceProp prop;
    HRAG_CUDA(cudaGetDeviceProperties(&prop, h->device));

    ShareBlob b;
    memset(&b, 0, sizeof b);
    memcpy(b.magic, kShareMagic, sizeof b.magic);
    b.version = kShareVersion;
    b.blob_bytes = (uint32_t)sizeof(ShareBlob);
    memcpy(b.uuid, prop.uuid.bytes, sizeof b.uuid);
    b.owner_pid = (int64_t)getpid();
    const PprGraph& g = h->g;
    b.n_global = g.n_global; b.row_lo = g.row_lo; b.n_rows = g.n_rows; b.long_thresh = g.long_thresh;
    b.n_long = g.n_long; b.n_seg = g.n_seg; b.max_batch = g.max_batch; b.has_val_lo = g.val_lo != nullptr;
    b.nnz = g.nnz;
    b.t_nodes = h->t.n_nodes; b.t_passages = h->t.n_passages; b.t_facts = h->t.n_facts;
    b.dim = h->dim;
    b.n_bounds = (int32_t)h->row_bounds.size();
    for (int i = 0; i < b.n_bounds; ++i) b.bounds[i] = h->row_bounds[(size_t)i];
    b.emb_rows[0] = h->emb[0].rows; b.emb_rows[1] = h->emb[1].rows;
    b.n_facts_global = h->n_facts_global;

    if (h->share.role == SHARE_NONE) {   // the attach counter, kept until hrag_index_unexport
        Buf c;
        HRAG_TRY(c.ensure(sizeof(int64_t)));
        HRAG_CUDA(cudaMemsetAsync(c.p, 0, sizeof(int64_t), h->stream));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
        h->share.counter = std::move(c);
    }
    Buf* bufs[kAllocs];
    shared_bufs(h, bufs);
    int64_t shared = 0;
    for (int i = 0; i < kAllocs; ++i) {
        if (!bufs[i]->p) continue;
        HRAG_CUDA(cudaIpcGetMemHandle(&b.alloc[i].handle, bufs[i]->p));
        b.alloc[i].bytes = bufs[i]->cap;
        if (i != A_COUNTER) shared += (int64_t)bufs[i]->cap;
    }
    h->share.role = SHARE_OWNER;
    h->share.shared_bytes = shared;
    memcpy(blob, &b, sizeof b);
    return 0;
}

int hrag_index_unexport(hrag_t* h) {
    HRAG_CHECK(h, "hrag_index_unexport: null handle");
    HRAG_CHECK(h->share.role == SHARE_OWNER, "hrag_index_unexport: the index is not exported");
    HRAG_CUDA(cudaSetDevice(h->device));
    int64_t n = 0;
    HRAG_TRY(read_count(h, &n));
    HRAG_CHECK(n == 0, "hrag_index_unexport: " + std::to_string(n) + " handle(s) in other processes are still "
                       "attached; they must call hrag_index_detach first");
    h->share = IndexShare{};
    return 0;
}

int hrag_index_attach(hrag_t* h, const void* blob, int64_t size) {
    const std::string who = "hrag_index_attach";
    HRAG_CHECK(h && blob, who + ": null argument");
    HRAG_CHECK(size >= 16 && memcmp(blob, kShareMagic, sizeof kShareMagic) == 0,
               who + ": not a blob written by hrag_index_export");
    uint32_t version = 0, blob_bytes = 0;
    memcpy(&version, static_cast<const char*>(blob) + 8, 4);
    memcpy(&blob_bytes, static_cast<const char*>(blob) + 12, 4);
    HRAG_CHECK(version == kShareVersion, who + ": the blob has layout version " + std::to_string(version) +
                                             ", this library reads version " + std::to_string(kShareVersion) +
                                             "; export and attach with the same build");
    HRAG_CHECK(size == (int64_t)sizeof(ShareBlob) && blob_bytes == sizeof(ShareBlob),
               who + ": the blob is " + std::to_string(size) + " bytes (it says " + std::to_string(blob_bytes) +
                   "), version " + std::to_string(kShareVersion) + " blobs are " + std::to_string(sizeof(ShareBlob)) +
                   ": truncated or corrupted");
    ShareBlob b;
    memcpy(&b, blob, sizeof b);
    HRAG_CHECK(h->share.role == SHARE_NONE, who + ": the handle already shares an index (exported or attached)");
    HRAG_CHECK(!holds_index(h), who + ": the handle already holds an index; attach on a fresh handle");
    HRAG_CHECK(h->world == 1, who + ": a node-range-sharded handle (world > 1) cannot attach");
    HRAG_CHECK(b.owner_pid != (int64_t)getpid(),
               who + ": the blob was exported by this process; CUDA IPC cannot map an allocation into the process "
                     "that exported it (cudaIpcOpenMemHandle), and the exporting handle serves this process already");
    HRAG_CUDA(cudaSetDevice(h->device));
    cudaDeviceProp prop;
    HRAG_CUDA(cudaGetDeviceProperties(&prop, h->device));
    HRAG_CHECK(memcmp(prop.uuid.bytes, b.uuid, sizeof b.uuid) == 0,
               who + ": the index was exported on another GPU (device UUIDs differ); attach a handle on the owner's "
                     "GPU (CUDA_VISIBLE_DEVICES may number it differently in each process)");
    HRAG_CHECK(b.dim > 0 && b.n_global > 0 && b.n_bounds >= 0 && b.n_bounds <= 2 && b.alloc[A_CV].bytes &&
                   b.alloc[A_PASSAGE_VID].bytes && b.alloc[A_CHUNK_COUNT].bytes && b.alloc[A_COUNTER].bytes,
               who + ": the blob describes no complete index");

    // map every allocation first: a failure leaves the handle as it was (the Bufs close what they opened)
    Buf m[kAllocs];
    int64_t shared = 0;
    for (int i = 0; i < kAllocs; ++i) {
        if (!b.alloc[i].bytes) continue;
        HRAG_CUDA(cudaIpcOpenMemHandle(&m[i].p, b.alloc[i].handle, cudaIpcMemLazyEnablePeerAccess));
        m[i].cap = (size_t)b.alloc[i].bytes;
        m[i].ipc = true;
        if (i != A_COUNTER) shared += (int64_t)b.alloc[i].bytes;
    }
    Buf seg_partial;   // written by every sweep: this handle's own
    if (b.n_long) HRAG_TRY(seg_partial.ensure((size_t)b.n_seg * b.max_batch * sizeof(float)));
    HRAG_TRY(invalidate_solves(h));
    h->V.reset(); h->XA.reset(); h->XC.reset(); h->partials.reset();
    h->share.counter = std::move(m[A_COUNTER]);
    if (const int rc = count_attach(h, 1)) { h->share = IndexShare{}; return rc; }

    // the views, as a load fills them
    GraphMem& G = h->graph;
    G = GraphMem{};
    Buf* bufs[kAllocs];
    shared_bufs(h, bufs);
    for (int i = 0; i < A_COUNTER; ++i) *bufs[i] = std::move(m[i]);
    G.seg_partial = std::move(seg_partial);
    PprGraph g;
    g.num_sms = h->num_sms;
    g.n_global = b.n_global; g.row_lo = b.row_lo; g.n_rows = b.n_rows; g.nnz = b.nnz;
    g.long_thresh = b.long_thresh; g.n_long = b.n_long; g.n_seg = b.n_seg; g.max_batch = b.max_batch;
    g.row_ptr = G.row_ptr.as<int>();
    g.cv = G.cv.as<int2>();
    g.row_order = G.row_order.as<int>();
    g.long_rows = G.long_rows.as<int>();
    g.long_seg_ptr = G.long_seg_ptr.as<int>();
    g.segs = G.segs.as<int4>();
    g.seg_partial = G.seg_partial.as<float>();
    g.val_lo = b.has_val_lo ? G.val_lo.as<float>() : nullptr;
    h->g = g;
    const TableMem& T = h->tables;
    h->t = SeedTables{b.t_nodes, b.t_passages, b.t_facts, T.passage_vid.as<int>(), T.fact_subj_vid.as<int>(),
                      T.fact_obj_vid.as<int>(), T.ent_chunk_count.as<int>()};
    for (int w = 0; w < 2; ++w) {
        h->emb[w].rows = b.emb_rows[w];
        h->emb[w].f32 = h->emb[w].own.as<float>();   // null when the owner keeps no fp32 rows
    }
    h->dim = b.dim;
    h->n_facts_global = b.n_facts_global;
    h->fact_row_lo = 0;
    HRAG_TRY(fact_norms_update(h, 0, h->emb[0].rows, true));   // this handle's own copy of the screen's bound
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    h->row_bounds.assign(b.bounds, b.bounds + b.n_bounds);
    h->chunk_rows = b.n_global;
    h->share.role = SHARE_ATTACHED;
    h->share.shared_bytes = shared;
    return 0;
}

int hrag_index_detach(hrag_t* h) {
    HRAG_CHECK(h, "hrag_index_detach: null handle");
    HRAG_CHECK(h->share.role == SHARE_ATTACHED, "hrag_index_detach: the handle is not attached (hrag_index_attach)");
    HRAG_CUDA(cudaSetDevice(h->device));
    HRAG_CUDA(cudaStreamSynchronize(h->stream_sim));
    HRAG_CUDA(cudaStreamSynchronize(h->stream2));
    HRAG_TRY(invalidate_solves(h));   // synchronises `stream`: nothing reads the mappings any more
    drop_attached_index(h);
    // the count goes down only once every mapping is closed; if it fails the handle stays attached (without an
    // index), and a second detach retries it
    HRAG_TRY(count_attach(h, -1));
    h->share = IndexShare{};
    return 0;
}

int hrag_index_share_info(hrag_t* h, int* role, int64_t* n_attached, int64_t* imported_bytes, int64_t* owned_bytes) {
    HRAG_CHECK(h && role && n_attached && imported_bytes && owned_bytes, "hrag_index_share_info: null argument");
    *role = h->share.role;
    *n_attached = 0;
    if (h->share.role != SHARE_NONE) {
        HRAG_CUDA(cudaSetDevice(h->device));
        HRAG_TRY(read_count(h, n_attached));
    }
    *imported_bytes = h->share.role != SHARE_NONE ? h->share.shared_bytes : 0;
    *owned_bytes = owned_device_bytes(h);
    return 0;
}

}  // extern "C"
