// The handle behind the C ABI of libhrag_b200.so and what the host sources share: api.cu (lifecycle, options, stages
// A/B, similarity, stats), ingest.cu (graph, tables, embeddings), graph_build.cu (the graph planes, built on the
// device), solve.cu (the PPR solvers), comm.cu (NCCL, peers) and index_share.cu (one index mapped into other processes).
//
// HBM layout per handle (N nodes, P passages, F facts, d dims; DESIGN.md section 3):
//   graph     row_ptr int32[n_rows+1], cv int2[nnz] {col, fp32 bits of P[i,j]}, row_order int32[n_rows]   (resident)
//             + val_lo fp32[nnz] = fp32(P64 - hi) when loaded from float64 values (the fp64 solver's operator)
//             + edges src/dst int32[E], w fp64[E]: the COO list as given, mutable handles only (index_update.cu)
//   tables    passage_vid[P], fact_subj/obj[F], ent_chunk_count[N]                                         (resident)
//   emb       bf16 hi/lo planes [rows, d] x 2 (wgmma similarity); fp32 [rows, d] only when uploaded whole    (resident)
//             facts over the hrag_set_fact_memory budget: the planes in pinned host memory, and on the device a
//             ring of two slices (fact_stream.cu) of at most the budget; under HRAG_FACT_LO_ON_HOST the hi plane
//             resident, the lo plane in mapped pinned host memory and a ring of two lo slices.  Where each plane
//             is: emb_planes; every path walks the planes with stream_slices, whatever their placement
//   shared    with hrag_index_export / hrag_index_attach the graph planes (but seg_partial), the tables and the embedding
//             planes of an attached handle are the owner's allocations, mapped through CUDA IPC (index_share.cu)
//   knn       self-KNN index (knn_index.cu): bf16 hi/lo [entities, d] x 2, ids / scores [entities, pad4(kmax + 1)]
//             (only after hrag_knn_index_update; independent of the retrieval index); planes over the
//             hrag_knn_set_memory budget in pinned host memory, streamed through a ring of two slices as the facts'
//   state     mixed solver: x0[2], A, C, R [N, 32] fp16 in one IPC-exportable slab, and for paired solves the same
//             [N, 2, 32] fp16 (two sub-batches interleaved row by row); fp32 solver: V, XA, XC [N, B] fp32
//   rhs       compact: slot_map [N] (node -> rhs slot), Vc [P + 2048, 32] fp32 (exact v) + R16 [P + 2048, 32] fp16
//             (scaled), two sets (double-buffered), four when sub-batches are solved in pairs
//   scores    S_pass [chunk, P] fp32; fact scores are never materialised in the fused modes (72 B per query x tile)
// Streams: `stream` runs the similarity, the solves and the selection; `stream2` builds the compact right-hand side of
// sub-batch i + 1 while sub-batch i is being solved.  On one GPU a sub-batch's solve is replayed as a CUDA graph.
// `stream_sim` (highest priority) runs the similarity GEMMs of chunk c + 1 of a multi-chunk hrag_retrieve_resident
// call while `stream` runs chunk c's solves; what it hands over lives in two slots (slot 1: `pipe`).
#pragma once
#include <nccl.h>

#include <algorithm>
#include <atomic>
#include <functional>
#include <string>
#include <utility>
#include <vector>

#include "../../include/hrag_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace hrag {

struct NcclApi {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t,
                              cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
inline NcclApi g_nccl;   // filled in by load_nccl (comm.cu): only sharded runs need NCCL
#define HRAG_NCCL(expr)                                                                        \
    do {                                                                                       \
        ncclResult_t _r = (expr);                                                              \
        if (_r != ncclSuccess) {                                                               \
            ::hrag::set_error(std::string(#expr) + " -> " + g_nccl.GetErrorString(_r));        \
            return 3;                                                                          \
        }                                                                                      \
    } while (0)

// Bumped whenever device storage is freed, so also by every reallocation (any handle, any thread): the captured CUDA
// graphs of the mixed solve hold raw pointers, so they are replayed only under the generation they were captured in.
inline std::atomic<int64_t> g_buf_generation{0};

// One device allocation, owned: move-only, freed by its destructor.  An imported Buf (ipc: mapped from another
// process by hrag_index_attach, index_share.cu) is unmapped instead of freed.
struct Buf {
    void* p = nullptr;
    size_t cap = 0;
    bool ipc = false;
    Buf() = default;
    Buf(Buf&& o) noexcept
        : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)), ipc(std::exchange(o.ipc, false)) {}
    Buf& operator=(Buf&& o) noexcept {   // o frees ours
        std::swap(p, o.p); std::swap(cap, o.cap); std::swap(ipc, o.ipc);
        return *this;
    }
    ~Buf() { reset(); }
    int ensure(size_t bytes) {    // grow-only; the contents are not kept
        if (bytes <= cap) return 0;
        reset();
        HRAG_CUDA(cudaMalloc(&p, bytes));
        cap = bytes;
        return 0;
    }
    template <class T, class V> int upload(const T* src, size_t n, V** view) {   // n elements; *view = the device copy
        HRAG_TRY(ensure(n ? n * sizeof(T) : 1));                          // non-null even when empty
        if (n) HRAG_CUDA(cudaMemcpy(p, src, n * sizeof(T), cudaMemcpyHostToDevice));
        *view = as<T>();
        return 0;
    }
    int zeros(size_t bytes) {     // ensure + clear
        HRAG_TRY(ensure(bytes));
        HRAG_CUDA(cudaMemset(p, 0, bytes));
        return 0;
    }
    void reset() {
        if (p) {
            g_buf_generation += 1;
            if (ipc) cudaIpcCloseMemHandle(p);
            else cudaFree(p);
        }
        p = nullptr; cap = 0; ipc = false;
    }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

enum Stage { ST_SIM_FACT = 0, ST_SEL_FACT, ST_SIM_PASS, ST_SEED, ST_PPR, ST_TOPK, ST_COMM, ST_COUNT };
struct Span { int stage; cudaEvent_t a, b; };

// The igraph edge list as the caller gave it (hrag_set_mutable handles loaded from a COO list only): int32 src, int32
// dst, fp64 w, 16 bytes per edge, n edges in use; capacity grows geometrically under hrag_index_append.
struct EdgeList { Buf src, dst, w; int64_t n = 0; };
// Storage behind the views the kernel launchers take (PprGraph g, SeedTables t), filled in by ingest.cu
struct GraphMem { Buf row_ptr, cv, row_order, long_rows, long_seg_ptr, segs, seg_partial, val_lo; EdgeList edges; };
struct TableMem { Buf passage_vid, fact_subj_vid, fact_obj_vid, ent_chunk_count; };
struct EmbMem {                   // one embedding matrix (0 = facts, 1 = passages)
    const float* f32 = nullptr;   // fp32 rows: borrowed from the caller (device upload, caller keeps it alive) or own
    Buf own, hi, lo;              // hi / lo: bf16 split for the tensor-core path (dim % 8 == 0)
    Buf nmax;                     // facts: float [2], upper bounds on the largest row norm of hi / lo (only grow;
                                  // the stage-A screen's bound, fact_norms_update)
    int64_t rows = 0;             // rows held by THIS handle (node-range sharding: the rank's slice of the facts)
};
// bf16 hi / lo planes [rows, dim] held in pinned host memory and streamed through a device ring of two halves, each
// slice_rows rows of the planes held here, hi then lo (fact_stream.cu): the fact planes over the hrag_set_fact_memory
// budget (FactPlanes) and the synonymy KNN planes over the hrag_knn_set_memory budget (KnnIndex::host).  `copy`
// carries the ring uploads; loaded[i] marks half i filled, freed[i] the last read of half i on `stream`.  Owned and
// move-only: freed by release().  Under HRAG_FACT_LO_ON_HOST only lo is held (hi stays null), and it is mapped.
struct HostPlanes {
    void *hi = nullptr, *lo = nullptr;   // pinned (cudaHostAlloc); null: that plane is not held here
    size_t plane_bytes = 0;              // of one of them (the capacity)
    int64_t slice_rows = 0;              // a multiple of 256, the K2 tile width
    Buf ring;                            // 2 halves, each [slice_rows, dim] bf16 per plane held
    cudaStream_t copy = nullptr;
    cudaEvent_t loaded[2] = {nullptr, nullptr}, freed[2] = {nullptr, nullptr};
    HostPlanes() = default;
    HostPlanes(HostPlanes&& o) noexcept { swap(o); }
    HostPlanes& operator=(HostPlanes&& o) noexcept {   // o frees ours
        swap(o);
        return *this;
    }
    ~HostPlanes() { release(); }
    void swap(HostPlanes& o) noexcept {
        std::swap(hi, o.hi); std::swap(lo, o.lo); std::swap(plane_bytes, o.plane_bytes);
        std::swap(slice_rows, o.slice_rows); std::swap(ring, o.ring); std::swap(copy, o.copy);
        std::swap(loaded, o.loaded); std::swap(freed, o.freed);
    }
    // pinned planes of `bytes` each (contents lost), a ring of two `slice`-row halves at `dim`, the copy stream;
    // !with_hi: the mapped lo plane only
    int alloc(size_t bytes, int64_t slice, int dim, bool with_hi = true);
    void release();
    bool held() const { return lo != nullptr; }                    // some plane is in host memory
};

// Where each plane of one hi / lo set lives, as the walker (stream_slices) and the fill (planes_fill) read it:
// plane[p] is a device address (read in place) or, when on_host[p], a pinned host address (streamed through host's
// ring).  plane_set builds it from the device planes and the host planes of a set; emb_planes is the one answer for
// the embedding matrices.
struct PlaneSet {
    char* plane[2] = {nullptr, nullptr};   // hi, lo
    bool on_host[2] = {false, false};
    const HostPlanes* host = nullptr;
    bool streams() const { return on_host[0] || on_host[1]; }
    int64_t host_bytes() const {
        return streams() ? (int64_t)host->plane_bytes * ((on_host[0] ? 1 : 0) + (on_host[1] ? 1 : 0)) : 0;
    }
};
inline PlaneSet plane_set(const Buf& hi, const Buf& lo, const HostPlanes* host) {
    PlaneSet P;
    P.on_host[0] = host && host->hi;
    P.on_host[1] = host && host->lo;
    P.plane[0] = P.on_host[0] ? static_cast<char*>(host->hi) : hi.as<char>();
    P.plane[1] = P.on_host[1] ? static_cast<char*>(host->lo) : lo.as<char>();
    P.host = host;
    return P;
}

// The resident self-KNN index (knn_index.cu), independent of the retrieval index: the bf16 hi / lo planes of its unit
// rows, and per row the first kmax keys with score >= thr, best first.  A list row is `width` = pad4(kmax + 1) int32
// ids (-1 padded) / fp32 scores; ids[row * width + kmax] holds the row's flags (kKnnComplete: the list holds every key
// >= thr).  held == false: no index (rows == 0 then too).  Planes over the hrag_knn_set_memory budget live in `host`
// (hi / lo then empty); the lists are always on the device.
struct KnnIndex {
    Buf hi, lo, ids, scores;
    HostPlanes host;
    int64_t rows = 0;
    int dim = 0, kmax = 0, width = 0;
    float thr = 0.f;
    bool held = false;
};
constexpr int kKnnComplete = 1, kKnnRefill = 2;

// Fact planes held in pinned host memory (hrag_set_fact_memory with a budget below rows x dim x 4 bytes;
// fact_stream.cu): byte for byte what a resident load builds, plus the state of a stage A over several slices.  Which
// plane is where: emb_planes(h, 0).
struct FactPlanes : HostPlanes {
    // a pass's per-query state: fused, (min, max) [3, B] and 8 keys [3, B, 8] (two running slots and this slice's);
    // materialised, the running (min, max) [B] and one chunk's slice top-k sl_ids / sl_scores [chunk, k], sl_mm
    Buf run_mm, run_keys, sl_ids, sl_scores, sl_mm;
    Buf tail;                            // sim_scores' scores of a ragged last slice
    FactPlanes() = default;
    FactPlanes(const FactPlanes&) = delete;
    FactPlanes& operator=(const FactPlanes&) = delete;
    ~FactPlanes() { release(); }
    void release();
};

// The read-only index shared between processes on one GPU through CUDA IPC (index_share.cu).  role 1 (owner,
// hrag_index_export): the index stays the handle's own, `counter` is the exported attach counter.  role 2 (attached,
// hrag_index_attach): the index Bufs are mapped from the owner (Buf::ipc), `counter` is the owner's counter, mapped.
// shared_bytes: of the shared index allocations, the counter not included.
enum ShareRole { SHARE_NONE = 0, SHARE_OWNER = 1, SHARE_ATTACHED = 2 };
struct IndexShare {
    int role = SHARE_NONE;
    Buf counter;   // int64: attached handles
    int64_t shared_bytes = 0;
};

}  // namespace hrag

namespace hrag {
// One fp16 state layout of the mixed solver (solve.cu): the first iterates x0[p] of the solves of parity p (a solve's
// dense first iterate, written while the solve before it runs, when it is built; either way the correction's first
// work buffer), and the work buffers A, C (Chebyshev iterates) and R
// (residual).  Rows are ld halves apart: 32 for one sub-batch, 64 for two sub-batches interleaved row by row.
struct StateLayout {
    void* x0[2] = {nullptr, nullptr};
    void *A = nullptr, *C = nullptr, *R = nullptr;
    int ld = 32;
    size_t bytes = 0;    // of one buffer
    // sub-batch k's part of one of these buffers (k = 1: the second 32 halves of every row of a pair); null stays null
    void* part(const void* buf, int k) const {
        return buf ? static_cast<char*>(const_cast<void*>(buf)) + 64 * k : nullptr;
    }
};
// One compact right-hand-side set of stage B's mixed solves: slot_map [N] (node -> slot, -1 = none), slot_vid [slots]
// (slot -> node), exact v Vc [slots, 32] fp32 and R16 = fp16(scale * Vc), with slots = P + 2048; its 32 column scales
// (float) and column sums of v (double).  hrag_ppr's dense solves use set 0's scale and vsum only.
struct RhsSet { Buf slot_map, slot_vid, Vc, R16, scale, vsum; };
// Column sums of one sub-batch's mixed solve: of the first solve's iterate, of the correction and of |residual|.
// Contiguous, so the sharded solve all-reduces the three at once.
struct MixedSums { double x0[32], d[32], r[32]; };
// What the mixed solves of a call report, read and cleared by resolve_spans: the running maximum of the measured
// relative L1 residual of their fp16 first solves, and whether an fp16 iterate left fp16's range.
struct MixedRho { float rho_max; int overflow; };
// The inputs of one sub-batch's mixed solve: its right-hand side (compact through slot_map, or dense), exact v, the
// dense first iterate, column scales and sums of v.  In a pair, x0_dense is the [N, 2, 32] buffer of both.
// x0_compact: the first iterate is not built in x0_dense; the first solve reads it through slot_map (solve.cu).
struct MixedRhs {
    const int* slot_map = nullptr;
    const float* Vexact = nullptr;
    const void* rhs16 = nullptr;
    void* x0_dense = nullptr;
    const float* scale = nullptr;
    const double* vsum = nullptr;
    bool x0_compact = false;
    bool operator==(const MixedRhs& o) const {
        return slot_map == o.slot_map && Vexact == o.Vexact && rhs16 == o.rhs16 && x0_dense == o.x0_dense &&
               scale == o.scale && vsum == o.vsum && x0_compact == o.x0_compact;
    }
};
}  // namespace hrag

struct hrag_handle {
    int device = 0;
    int shard_mode = 0;
    int rank = 0, world = 1;
    ncclComm_t comm = nullptr;
    cudaStream_t stream = nullptr;

    hrag::PprGraph g;                  // view of `graph`
    hrag::GraphMem graph;
    bool mutable_index = false;        // hrag_set_mutable: the next COO load keeps its edge list (graph.edges)
    int64_t chunk_rows = 0;      // rows per rank (sharded) = ceil(N / world)
    std::vector<int64_t> row_bounds;   // optional [world + 1]: rank r owns rows [row_bounds[r], row_bounds[r + 1]) -- a
                                       // work-balanced partition (non-zeros + 4 per row) instead of equal row counts
    hrag::SeedTables t;                // view of `tables`
    hrag::TableMem tables;
    hrag::EmbMem emb[2];
    int64_t fact_budget = 0;           // hrag_set_fact_memory: device bytes the fact planes may take (0 = no limit)
    int fact_placement = HRAG_FACT_PLANES_BY_BUDGET;   // hrag_set_fact_placement: applied by the next fact load
    hrag::FactPlanes fplanes;          // the fact planes in pinned host memory when they exceed fact_budget
    hrag::KnnIndex knn;                // hrag_knn_index_update: the synonymy KNN of the entities, kept between calls
    int64_t knn_budget = 0;            // hrag_knn_set_memory: device bytes the KNN planes may take (0 = no limit)
    hrag::IndexShare share;            // hrag_index_export / hrag_index_attach: the index shared with other processes
    int num_sms = 132;
    int64_t fact_row_lo = 0;        // first global fact row of the local slice
    int64_t n_facts_global = 0;
    int dim = 0;

    int ppr_method = HRAG_PPR_CHEBYSHEV;
    int ppr_iters = 0;    // 0 = derived from damping / tol (plan_sweeps): 14 Chebyshev sweeps at damping 0.5
    int ppr_batch = 16;
    int sim_mode = HRAG_SIM_BF16X3;
    bool keep_fact_scores = false;   // debugging: materialise S_fact even in tensor-core modes
    int debug_sim_ctas = 0;          // hrag_debug_sim_ctas: > 0 GEMM CTAs, < 0 no chunk overlap, 0 defaults
    bool debug_dense_first_sweep = false;   // hrag_debug_dense_first_sweep: stage B builds the dense first iterate
    bool debug_exact_stage_a = false;       // hrag_debug_exact_stage_a: stage A runs the split K2 over all facts
    int ppr_precision = HRAG_PPR_MIXED;   // applies to batches of > 16 queries; smaller ones run fp32
    int mixed_m1 = 0, mixed_m2 = 0;   // 0 = derived from damping (8 / 7 at damping 0.5)
    double check_tol = 0.0, check_kappa = 0.0;   // > 0: this call's mixed solves are verified in resolve_spans
    double last_rho = 0.0;            // measured relative L1 residual: of the fp16 first solve (last mixed call), of
                                      // the final refinement round (last hrag_ppr_f64 call)
    bool rho_dirty = false;           // a mixed solve ran in this call: rho must be read / cleared in resolve_spans
    double last_bound = 0.0;          // a-posteriori bound on the relative L1 error of the last mixed / fp64 call

    // fp32 solver state [N, B], its column-sum partials and sums (V also holds hrag_ppr's exact v for the mixed solver)
    hrag::Buf V, XA, XC, partials, sums;
    // fp64 solver (hrag_ppr_f64, hrag_stage_b_f64): iterate X64 and reset V64 [N, B] fp64, host-layout staging io64
    // [B, max(N, pad4(P))] fp64 (reset in; probabilities, or stage B's passage scores, out), column-sum partials
    // part64, sums64 = [vsum | rsum | xsum] x 16
    hrag::Buf X64, V64, io64, part64, sums64;
    // mixed solver, laid out by solve.cu: the single state layout lives in `slab` ([x0[0] | A | C | R | x0[1] | epoch
    // flags], so a single IPC handle exposes every buffer a peer sweep may have to write into: K5, fused exchange for
    // node-range sharding), the pair layout of paired solves (single GPU, stage B) in slab_pair
    hrag::Buf slab, slab_pair;
    hrag::StateLayout single, pair;
    hrag::Buf mixed_part[2], mixed_sums;      // sub-batch k's column-sum partials; MixedSums [2]
    hrag::Buf rho, p2p_err, done_ctr;         // rho: MixedRho
    // stage B's compact right-hand sides: stream2 prepares solve i + 1's while `stream` sweeps solve i's
    hrag::RhsSet rhs[4];
    hrag::Buf prep_scratch;
    int slot_maps_built = 0;                  // sets 0 .. slot_maps_built - 1 hold valid slot maps
    // scratch and I/O staging
    hrag::Buf S_fact, S_pass, mm_fact, mm_pass, mode, seed_vid, seed_w, q_hi, q_lo, part_mm, part_keys;
    hrag::Buf part_bound;                 // fused stage A: [Bq] per-query bound on the 8th best key (sim_tc's scratch)
    hrag::Buf xr_mm, xr_keys;             // fact-sharded stage A: [world, Bq] min/max and [world, Bq, 8] best keys
    // the stage-A screen (api.cu screened_stage_a): per query err [Bq], the s1 tile lows part_low [Bq, n_tiles] (its
    // keys in part_keys), candidates cand_ids / cand_s1 [Bq, 256], cand_n, saturated tiles sat [Bq, 8], sat_n; per
    // m-tile pos_of [m, F], slot_ids [m, 48, 256], res_count [m, 256], stage_count [m], the staging planes st_hi / st_lo
    // [m * 48 * 256, d] and the rescored scores st_S [Bq, 48 * 256]; flag: this chunk falls back; fallbacks: counted
    // on the device, drained into stats by resolve_spans.  About 0.6 GB at C3 (F = 2.75 M, d = 768), on top of the
    // fused buffers and outside the hrag_set_fact_memory budget.  lo on the host (fact_stream.cu): call_flags holds
    // the lo bytes the gathers read (uint64) and then one flag per query chunk of the call (int32)
    struct {
        hrag::Buf err, part_low, cand_ids, cand_s1, cand_n, sat, sat_n, pos_of, slot_ids, res_count, stage_count,
            st_hi, st_lo, st_S, flag, fallbacks, call_flags;
    } scr;
    hrag::Buf fs_top_idx, fs_top_score, fs_nvalid;   // hrag_retrieve_resident on host fact planes: stage A [B, k]
    hrag::Buf d_q, d_q2, d_top_idx, d_top_score, d_nvalid, d_kept_idx, d_kept_score, d_dpr, d_out_ids, d_out_scores;
    hrag::Buf d_reset, d_scores;
    // second slot of what stream_sim hands to `stream` in hrag_retrieve_resident (slot 0: d_top_*, d_nvalid,
    // S_pass, mm_pass); allocated by the first call with two or more chunks
    struct { hrag::Buf top_idx, top_score, nvalid, S_pass, mm_pass; } pipe;
    // CUDA graphs of the mixed solve, one per (buffer sets, sweep plan, g_buf_generation)
    struct SolveGraph {
        int n = 0;                        // sub-batches solved together (1, or 2 = a pair)
        hrag::MixedRhs in[2];
        int m1 = 0, m2 = 0;
        float alpha = 0.f;
        int64_t generation = 0;
        cudaGraphExec_t exec = nullptr;
        void *X0[2] = {nullptr, nullptr}, *D[2] = {nullptr, nullptr};
        int64_t sweeps = 0, columns = 0, launches = 0;
    };
    std::vector<SolveGraph> solve_graphs;
    bool p2p = false;
    void* peer_slab[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    unsigned long long epoch = 0;             // exchange epochs signalled so far (same sequence on every rank)
    cudaStream_t stream2 = nullptr;
    cudaEvent_t ev_ready[2] = {nullptr, nullptr}, ev_released[2] = {nullptr, nullptr}, ev_inputs = nullptr;
    cudaStream_t stream_sim = nullptr;
    // sim_ready[s]: slot s holds a chunk's stage A and passage scores; sim_consumed[s]: its solves and top-k are done
    cudaEvent_t ev_sim_ready[2] = {nullptr, nullptr}, ev_sim_consumed[2] = {nullptr, nullptr}, ev_sim_start = nullptr;
    int64_t last_fact_rows = 0, last_pass_rows = 0;
    int64_t last_mm_rows = 0;   // rows of mm_fact the last device stage-A chunk wrote (hrag_debug_fact_minmax)
    const hrag::Buf* last_pass_S = &S_pass;   // the passage scores hrag_debug_copy reads (last_pass_rows rows)

    hrag_stats_t stats{};
    std::vector<hrag::Span> spans;
    std::vector<cudaEvent_t> pool;
};

namespace hrag {

inline cudaEvent_t get_event(hrag_t* h) {
    if (!h->pool.empty()) { cudaEvent_t e = h->pool.back(); h->pool.pop_back(); return e; }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}
// Times the work enqueued on `s` during its lifetime as one span of `stage`.  Spans on different streams may overlap.
struct StageTimer {
    hrag_t* h; cudaStream_t s; int idx;
    StageTimer(hrag_t* h_, int stage, cudaStream_t s_) : h(h_), s(s_) {
        Span sp{stage, get_event(h), get_event(h)};
        cudaEventRecord(sp.a, s);
        h->spans.push_back(sp);
        idx = (int)h->spans.size() - 1;
    }
    StageTimer(hrag_t* h_, int stage) : StageTimer(h_, stage, h_->stream) {}
    ~StageTimer() { cudaEventRecord(h->spans[idx].b, s); }
};

inline int h2d(hrag_t* h, void* dst, const void* src, size_t bytes) {
    HRAG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream));
    h->stats.h2d_bytes += (int64_t)bytes;
    return 0;
}
inline int d2h(hrag_t* h, void* dst, const void* src, size_t bytes) {
    HRAG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, h->stream));
    h->stats.d2h_bytes += (int64_t)bytes;
    return 0;
}

// The one answer to "which plane of embedding matrix `which` is where": only the facts' may be in host memory.
inline PlaneSet emb_planes(const hrag_t* h, int which) {
    return plane_set(h->emb[which].hi, h->emb[which].lo, which == 0 ? &h->fplanes : nullptr);
}

constexpr int kQueryChunk = 1024;  // queries per similarity GEMM launch (stage A, stage B, the similarity entries)
constexpr int kSeedSlots = kSeedSlotsPerQuery;   // 2 phrases per kept fact, <= 32 kept facts
constexpr float kMixedT = 64.f;    // residual scale: r ~ 5e-4 x, keeps it in fp16's normal range
constexpr double kDefaultTol = 1e-6;     // relative L1 accuracy of the PPR vector when the caller passes tol <= 0
struct SweepPlan {
    bool mixed = false;
    int iters = 14;          // fp32 solver
    int m1 = 8, m2 = 7;      // mixed solver
    double kappa = 0.0;      // predicted contraction of the refinement round (mixed)
    double tol = kDefaultTol;
    bool check = false;      // verify the measured residual bound at the end of the call
};
SweepPlan plan_sweeps(const hrag_t* h, float alpha, int iters_arg, float tol_arg, bool want_mixed);
int round_batch(int b);
int ensure_state(hrag_t* h, int B);
int ensure_state_mixed(hrag_t* h);
// The epoch flag words of the fused exchange inside a state slab (this rank's or a peer's), one per rank
unsigned long long* epoch_flags(const hrag_t* h, void* slab);
// Stage B's mixed solves of Bq queries (kept facts k_facts): ensure_stage_b_mixed allocates their state before the
// seeds; stage_b_mixed (k_facts > 0) runs them after the seeds and gathers the PPR scores into S in place.
int ensure_stage_b_mixed(hrag_t* h, int Bq, int k_facts);
int stage_b_mixed(hrag_t* h, const SweepPlan& plan, int Bq, float* S, int64_t ldS, const float2* mm_pass, float pnw,
                  float damping);
// A new graph, new tables or an index update: the slot maps and the captured solves are stale.  drop_captured_solves
// synchronises `stream` and destroys the captured solves only.
int invalidate_solves(hrag_t* h);
int drop_captured_solves(hrag_t* h);
int resolve_spans(hrag_t* h);   // end of a call: checks the mixed solves, accumulates the stage times
int dev_ppr(hrag_t* h, int B, int iters, float alpha, float** result);

// Float64 PPR by iterative refinement (solve.cu), shared by hrag_ppr_f64 and hrag_stage_b_f64.
// check_f64_call: the argument / handle checks of a float64 solve, messages prefixed by `who`.
int check_f64_call(hrag_t* h, const char* who, double damping, double tol);
double f64_target(double tol);                       // tol 0 = 1e-10
// state of sub-batches Bp wide; io64 holds Bp rows of max(N, io_cols)
int ensure_state_f64(hrag_t* h, int Bp, int64_t io_cols);
// io64 [nb, N] (host-layout reset) -> V64, h->V = fp32(V64), X64 = 0, sums64[0, Bp) = column sums of v
int reset_f64(hrag_t* h, int Bp, int nb);
struct F64Refined {
    double resid = 0.0;      // max over the columns of ||r||_1 / ||v||_1 after the last round
    double bound = 0.0;      // 2 resid / (1 - damping)
    unsigned active = 0;     // columns whose bound still misses the target (the solve failed if any)
};
// Up to 4 rounds of fp32 solve + fp64 correction + fp64 residual on the state reset_f64 prepared; every column stops
// once its own bound meets `target`.  Leaves X64 and xsum = sums64 + 32 (its column sums).
int refine_f64(hrag_t* h, int Bp, int nb, double damping, double target, F64Refined* out);
// End of a call whose sub-batch missed the target: stats report the call so far, error message, status 4.
int f64_missed(hrag_t* h, const char* who, const F64Refined& r, double target, double call_resid, double call_bound);

// graph_build.cu: the graph built on the device, on `stream`; both return once the device work is done.
struct DeviceCsr { Buf row_ptr, col, val; int64_t nnz = 0; };   // int64 [N + 1], int32 [nnz], fp64 [nnz]
// CSR of P = W D^-1 from a device edge list with n_edges < 2^30 (device pointers); *bad_edges = an endpoint lies
// outside [0, n_nodes), and then nothing was built.
int coo_to_csr(hrag_t* h, int64_t n_nodes, int64_t n_edges, const int32_t* src, const int32_t* dst, const double* w,
               DeviceCsr* out, bool* bad_edges);
// Replaces the handle's graph by rows [row_lo, row_hi) of a validated device CSR: row_ptr[0 .. n_rows] (offsets minus
// `base` index col / val), exactly one of val (fp32) / val64 given; bounds = the row partition to install.
int install_graph(hrag_t* h, int64_t n_nodes, int64_t row_lo, int64_t row_hi, int64_t nnz, const int64_t* row_ptr,
                  int64_t base, const int32_t* col, const float* val, const double* val64,
                  const std::vector<int64_t>& bounds);

// index_update.cu: *out = a copy of a device edge list of n edges (what a mutable handle keeps).
int copy_edge_list(hrag_t* h, int64_t n, const int32_t* src, const int32_t* dst, const double* w, EdgeList* out);
// Grows b to `need` bytes (by half its capacity at least), keeping its first `used` bytes.
int grow_keep(hrag_t* h, Buf& b, size_t used, size_t need);
// In place: rows [0, n_new) of the plane at `base` become its rows row_src[0 .. n_new) (device, ascending), rows
// before `first` staying put; row_bytes % 16 == 0; staging is a bounded scratch buffer.
int compact_rows(hrag_t* h, void* base, size_t row_bytes, int64_t n_new, int64_t first, const int* row_src,
                 Buf& staging);
// out row r = base row row_src[r] (device), r < n_rows, on h->stream; row_bytes % 16 == 0.
int gather_rows(hrag_t* h, const void* base, size_t row_bytes, const int* row_src, int64_t n_rows, void* out);

// fact_stream.cu: planes in pinned host memory, streamed through a device ring.
// host_planes_plan: *slice_rows = 0 when the planes of `rows` x `dim` fit `budget` (0 = no limit), else the rows of
// one ring slice, the largest multiple of 256 of which two fit the budget; a budget below two 256-row slices is
// rejected with a message naming `who` and the entry that set the budget, `setter`.
int host_planes_plan(int64_t budget, const std::string& who, const char* setter, int64_t rows, int dim,
                     int64_t* slice_rows);
// fact_planes_plan, before a fact load touches the handle: host_planes_plan of the fact budget, or under
// HRAG_FACT_LO_ON_HOST the lo ring's slice rows (*hi_resident set); rejects sharded handles and dim % 8 != 0.
// fact_planes_alloc, after reset_embeddings: the pinned planes and the ring for the handle's fact rows, and with
// hi_resident the resident hi plane and the zeroed norm maxima as well.
int fact_planes_plan(const hrag_t* h, const std::string& who, int64_t rows, int dim, int64_t* slice_rows,
                     bool* hi_resident);
int fact_planes_alloc(hrag_t* h, int64_t slice_rows, bool hi_resident);
// Fills plane rows [row0, row0 + n) of `P` (dim wide, some plane on the host) from fp32 rows (host or device): ring
// half 0 stages as many fp32 rows as its bytes hold, half 1 takes their split; a host plane's rows go back to the
// pinned plane, a resident plane takes its rows directly.  before_write(r, m, hi, lo), when given, runs on `stream`
// after rows [row0 + r, row0 + r + m) are split into hi / lo and before they are written back; half 0 is free then.
// Returns once the rows are written.
using BeforeWrite = std::function<int(int64_t r, int64_t m, const char* hi, const char* lo)>;
int planes_fill(hrag_t* h, const PlaneSet& P, int dim, int64_t row0, int64_t n, const float* src, bool src_on_device,
                const BeforeWrite& before_write = nullptr);
int fact_planes_fill(hrag_t* h, int64_t row0, int64_t n, const float* src, bool src_on_device);
// Walks rows [row0, row1) of the planes `P` (dim wide): body(s, first row, rows, hi, lo) reads slice s.  Both planes
// resident: body runs once over [row0, row1) with their device addresses, and the walk records, copies and counts
// nothing.  Else slices of slice_rows from row0 on `stream`: a plane on the host is read from its ring half while the
// copy stream fills the other half with slice s + 1, a resident plane in place.  `both`: the lo plane is read too
// (HRAG_SIM_BF16 reads only hi; lo = hi when lo is not copied).  Every copy is joined into `stream` before its slice
// is read, so the caller's later work on `stream` sees the whole walk.
template <class Body>
int stream_slices(hrag_t* h, const PlaneSet& P, int64_t dim, int64_t row0, int64_t row1, bool both, Body body) {
    const size_t rb = (size_t)dim * 2;
    if (!P.streams()) return body(0, row0, row1 - row0, P.plane[0] + row0 * rb, P.plane[1] + row0 * rb);
    const HostPlanes& ps = *P.host;
    const int64_t S = ps.slice_rows, n_slices = ceil_div(row1 - row0, S);
    const bool copy_lo = both && P.on_host[1];
    const size_t lo_at = P.on_host[0] ? (size_t)S * rb : 0;   // of the lo rows in a ring half
    const size_t half_bytes = lo_at + (P.on_host[1] ? (size_t)S * rb : 0);
    char* ring = ps.ring.as<char>();
    auto copy = [&](int64_t s) -> int {
        const int64_t r0 = row0 + s * S, n = std::min(S, row1 - r0);
        const int half = (int)(s & 1);
        char* dst = ring + half * half_bytes;
        HRAG_CUDA(cudaStreamWaitEvent(ps.copy, ps.freed[half], 0));   // the last read of this half is done
        if (P.on_host[0])
            HRAG_CUDA(cudaMemcpyAsync(dst, P.plane[0] + (size_t)r0 * rb, (size_t)n * rb, cudaMemcpyHostToDevice,
                                      ps.copy));
        if (copy_lo)
            HRAG_CUDA(cudaMemcpyAsync(dst + lo_at, P.plane[1] + (size_t)r0 * rb, (size_t)n * rb,
                                      cudaMemcpyHostToDevice, ps.copy));
        h->stats.h2d_bytes += (int64_t)n * (int64_t)rb * ((P.on_host[0] ? 1 : 0) + (copy_lo ? 1 : 0));
        HRAG_CUDA(cudaEventRecord(ps.loaded[half], ps.copy));
        return 0;
    };
    if (n_slices <= 0) return 0;
    for (int i = 0; i < 2; ++i) HRAG_CUDA(cudaEventRecord(ps.freed[i], h->stream));   // after the earlier reads
    HRAG_TRY(copy(0));
    for (int64_t s = 0; s < n_slices; ++s) {
        if (s + 1 < n_slices) HRAG_TRY(copy(s + 1));
        const int half = (int)(s & 1);
        HRAG_CUDA(cudaStreamWaitEvent(h->stream, ps.loaded[half], 0));
        const int64_t r0 = row0 + s * S;
        const char* h_half = ring + half * half_bytes;
        const char* e_hi = P.on_host[0] ? h_half : P.plane[0] + (size_t)r0 * rb;
        const char* e_lo = copy_lo ? h_half + lo_at : P.on_host[1] ? e_hi : P.plane[1] + (size_t)r0 * rb;
        HRAG_TRY(body(s, r0, std::min(S, row1 - r0), e_hi, e_lo));
        HRAG_CUDA(cudaEventRecord(ps.freed[half], h->stream));
    }
    return 0;
}
// fused_stage_a: stage A selects the facts in the GEMM epilogue (tensor-core modes, k <= 8, no kept scores);
// chunk_a: queries per stage-A chunk over the resident facts.
bool fused_stage_a(const hrag_t* h, int k);
int64_t chunk_a(const hrag_t* h, int k);
// Stage A of B queries (fp32 [B, dim], host or device) into device top_idx / top_score [B, k] and nvalid [B], on
// stream s with n_ctas GEMM CTAs: the split K2 walked over the fact planes (or the stage-A screen), in passes of a
// query chunk on resident planes and of fact_stream_pass_cap queries, each walking the planes once, when one streams
// (on `stream` then).  Every placement gives the same outputs, bit for bit.
int fact_stage_a(hrag_t* h, int B, const float* q, bool q_on_device, int k, int* top_idx, float* top_score,
                 int* nvalid, cudaStream_t s, int n_ctas);
// Raw scores of nb (<= 1024) device queries against embedding matrix `which` into S [nb, ldS] on stream s: the
// tensor-core GEMM walked over the planes, or sim_fp32 over resident fp32 rows.
int sim_scores(hrag_t* h, int which, const float* dQ, int nb, float* S, int64_t ldS, cudaStream_t s, int n_ctas);

// api.cu: the stage-A screen on one query chunk.  screened(h): the screen applies to this handle's facts.
// screened_stage_a: Bq <= 1024 queries (fp32 on the device); with the lo plane in host memory
// it gathers the staged lo rows from the mapped plane, adds their bytes to *lo_bytes, raises *chunk_flag instead of
// running the gated exact path (the caller reruns a flagged chunk) and counts no fallback.
bool screened(const hrag_t* h);
int screened_stage_a(hrag_t* h, int Bq, const float* d_qf, int k, int* d_top_idx, float* d_top_score, int* d_nvalid,
                     cudaStream_t s, int n_ctas, int* chunk_flag = nullptr, unsigned long long* lo_bytes = nullptr);

// api.cu: emb[0].nmax (reset to 0 first when `reset`) raised to the row norms of fact plane rows [row0, row0 + n), on
// `stream`.  Every writer of resident fact planes calls it, so nmax bounds every row the stage-A screen scores.
int fact_norms_update(hrag_t* h, int64_t row0, int64_t n, bool reset);

// index_share.cu: status 1 with a message naming `who` when the handle's index is exported or attached (loads and
// in-place updates would change, or free, memory other processes map); index_share_destroy is hrag_destroy's part:
// an attached handle detaches, an owner with live attachments leaves the exported allocations mapped.
int check_index_private(const hrag_t* h, const std::string& who);
void index_share_destroy(hrag_t* h);

int exchange_rows(hrag_t* h, float* y, int B);
int exchange_rows_bytes(hrag_t* h, void* y, size_t row_bytes);
// a sweep's fused exchange (K5): the peers' copies of y, and the sweep's epoch (null flags when the peers are not mapped)
PeerOut peers_for(hrag_t* h, void* y);
SweepSync sync_for_sweep(hrag_t* h);
int p2p_wait(hrag_t* h);
int p2p_signal(hrag_t* h);

}  // namespace hrag
