// Updates of a loaded index in place, the device side of HippoRAG.index() / HippoRAG.delete() (reference
// HippoRAG.py:262-335, :337-411): hrag_index_append appends vertices, edges, passages and facts; hrag_index_delete
// removes vertices and facts, keeping the order of what stays.  Both end in the state a fresh load of the resulting
// arrays gives, byte for byte: the graph planes are rebuilt from the resident edge list by the loaders' own builder
// (coo_to_csr + install_graph) -- a new edge changes the strength, and so every value, of both endpoint columns, and a
// patched CSR would have to reproduce the builder's summation orders -- the tables and embedding planes are appended
// to or compacted stably.  Call contract as the loaders' (ingest.cu): every input is checked before the handle is
// touched, so a rejected call leaves it as it was; a failure after that (out of memory) leaves no index at all.
#include <cub/cub.cuh>

#include <algorithm>

#include "handle.h"

namespace hrag {
namespace {

constexpr int kThreads = 256;
constexpr size_t kStagingBytes = (size_t)64 << 20;   // bound of the in-place row compaction's staging buffer

int blocks_for(int64_t n) { return (int)ceil_div(std::max<int64_t>(n, 1), kThreads); }

__device__ __forceinline__ int64_t thread_index() { return blockIdx.x * (int64_t)blockDim.x + threadIdx.x; }

__device__ __forceinline__ bool listed(const int32_t* __restrict__ sorted, int64_t n, int64_t v) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) / 2;
        if (sorted[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && sorted[lo] == v;
}

// flags[i] = i is not in the sorted list `del`, for i < n; flags[n] = 0 (so the exclusive scan ends in the total)
__global__ void k_keep_unlisted(int64_t n, const int32_t* __restrict__ del, int64_t n_del, int* __restrict__ flags) {
    const int64_t i = thread_index();
    if (i <= n) flags[i] = i < n && !listed(del, n_del, i);
}

// pos = exclusive scan of the vertex flags -> the old -> new vertex map, -1 for a deleted vertex (in place)
__global__ void k_vertex_map(int64_t n, const int* __restrict__ flags, int* __restrict__ pos) {
    const int64_t v = thread_index();
    if (v < n && !flags[v]) pos[v] = -1;
}

__device__ __forceinline__ int relabel(const int* __restrict__ map, int v) { return v >= 0 ? map[v] : -1; }

__global__ void k_edge_flags(int64_t n, const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                             const int* __restrict__ map, int* __restrict__ flags) {
    const int64_t i = thread_index();
    if (i <= n) flags[i] = i < n && map[src[i]] >= 0 && map[dst[i]] >= 0;
}

// every kept edge goes to its rank among the kept ones (the exclusive scan): the input order survives, and with it
// the order in which coo_to_csr sums parallel edges
__global__ void k_edge_scatter(int64_t n, const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                               const double* __restrict__ w, const int* __restrict__ map, const int* __restrict__ flags,
                               const int* __restrict__ pos, int32_t* __restrict__ osrc, int32_t* __restrict__ odst,
                               double* __restrict__ ow) {
    const int64_t i = thread_index();
    if (i >= n || !flags[i]) return;
    const int k = pos[i];
    osrc[k] = map[src[i]];
    odst[k] = map[dst[i]];
    ow[k] = w[i];
}

__global__ void k_passage_flags(int64_t n, const int32_t* __restrict__ vid, const int* __restrict__ map,
                                int* __restrict__ flags) {
    const int64_t p = thread_index();
    if (p <= n) flags[p] = p < n && map[vid[p]] >= 0;
}

// kept passage p -> row pos[p]: its relabelled vertex, and row_src[pos[p]] = p for the embedding compaction
__global__ void k_passage_scatter(int64_t n, const int32_t* __restrict__ vid, const int* __restrict__ map,
                                  const int* __restrict__ flags, const int* __restrict__ pos, int32_t* __restrict__ ovid,
                                  int* __restrict__ row_src) {
    const int64_t p = thread_index();
    if (p >= n || !flags[p]) return;
    ovid[pos[p]] = map[vid[p]];
    row_src[pos[p]] = (int)p;
}

// kept fact f -> row pos[f]: subject / object relabelled (a deleted or absent vertex becomes -1), row_src as above
__global__ void k_fact_scatter(int64_t n, const int32_t* __restrict__ subj, const int32_t* __restrict__ obj,
                               const int* __restrict__ map, const int* __restrict__ flags, const int* __restrict__ pos,
                               int32_t* __restrict__ osubj, int32_t* __restrict__ oobj, int* __restrict__ row_src) {
    const int64_t f = thread_index();
    if (f >= n || !flags[f]) return;
    const int k = pos[f];
    osubj[k] = relabel(map, subj[f]);
    oobj[k] = relabel(map, obj[f]);
    row_src[k] = (int)f;
}

// *first = min(*first, the first i < n with flags[i] == 0): the first row a compaction moves
__global__ void k_first_dropped(int64_t n, const int* __restrict__ flags, int* __restrict__ first) {
    const int64_t i = thread_index();
    if (i < n && !flags[i]) atomicMin(first, (int)i);
}

// staging row r = base row row_src[r0 + r], for r < n_rows; rows are `w16` 16-byte words long
__global__ void k_gather_rows(int64_t n_rows, int64_t w16, const int* __restrict__ row_src, int64_t r0,
                              const int4* __restrict__ base, int4* __restrict__ staging) {
    const int64_t i = thread_index();
    if (i >= n_rows * w16) return;
    const int64_t r = i / w16, c = i - r * w16;
    staging[i] = base[(int64_t)row_src[r0 + r] * w16 + c];
}

// *bad += the edges with an endpoint outside [0, n_nodes): a device edge list is checked before anything is written
__global__ void k_count_bad_edges(int64_t n, int64_t n_nodes, const int32_t* __restrict__ src,
                                  const int32_t* __restrict__ dst, unsigned long long* __restrict__ bad) {
    const int64_t i = thread_index();
    if (i < n && (src[i] < 0 || src[i] >= n_nodes || dst[i] < 0 || dst[i] >= n_nodes)) atomicAdd(bad, 1ull);
}

}  // namespace

// Grows b to hold `need` bytes, keeping its first `used` bytes: by half its capacity at least, so a stream of small
// appends copies a plane O(log) times, not once per append.
int grow_keep(hrag_t* h, Buf& b, size_t used, size_t need) {
    if (b.p && need <= b.cap) return 0;
    Buf nb;
    HRAG_TRY(nb.ensure(std::max<size_t>({need, b.cap + b.cap / 2, 1})));
    if (used) HRAG_CUDA(cudaMemcpyAsync(nb.p, b.p, used, cudaMemcpyDeviceToDevice, h->stream));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));   // the old allocation is freed below
    b = std::move(nb);
    return 0;
}

namespace {

// Copies n elements from host (counted in h2d_bytes) or device memory to dst, on h->stream.
template <class T> int copy_in(hrag_t* h, T* dst, const T* src, int64_t n, bool on_device) {
    if (n <= 0) return 0;
    if (!on_device) return h2d(h, dst, src, (size_t)n * sizeof(T));
    HRAG_CUDA(cudaMemcpyAsync(dst, src, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, h->stream));
    return 0;
}

// pos[0 .. n] = the exclusive scan of flags[0 .. n] (flags[n] = 0), *kept = pos[n]; with `first`, also the first
// i < n whose flag is 0 (n when none is): rows before it stay where they are
int scan_flags(hrag_t* h, int64_t n, const int* flags, int* pos, int64_t* kept, int64_t* first = nullptr) {
    Buf tmp, d_first;
    size_t tb = 0;
    HRAG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, flags, pos, (int)(n + 1), h->stream));
    HRAG_TRY(tmp.ensure(std::max<size_t>(tb, 1)));
    HRAG_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, flags, pos, (int)(n + 1), h->stream));
    int host[2] = {0, (int)n};
    if (first) {
        const int none = (int)n;
        HRAG_TRY(d_first.ensure(sizeof(int)));
        HRAG_CUDA(cudaMemcpy(d_first.p, &none, sizeof(int), cudaMemcpyHostToDevice));
        if (n) k_first_dropped<<<blocks_for(n), kThreads, 0, h->stream>>>(n, flags, d_first.as<int>());
        HRAG_CUDA(cudaGetLastError());
        HRAG_CUDA(cudaMemcpyAsync(&host[1], d_first.p, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    }
    HRAG_CUDA(cudaMemcpyAsync(&host[0], pos + n, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    *kept = host[0];
    if (first) *first = host[1];
    return 0;
}

}  // namespace

// Rows [0, n_new) of the plane at `base` (rows of row_bytes, a multiple of 16) become its rows row_src[0 .. n_new),
// in place; rows before `first` (row_src[i] == i there) do not move.  row_src is ascending, so row_src[i] >= i:
// destinations never lie after their sources.  The rows move chunk by chunk through a bounded staging buffer, each
// chunk gathered into it and then copied back to its destination rows, in stream order.  A chunk writes rows
// [r0, r0 + n) and every later chunk reads rows row_src[i] >= i >= r0 + n only, so no chunk overwrites a row that is
// still to be read, and no second copy of the plane is ever held.
int compact_rows(hrag_t* h, void* base, size_t row_bytes, int64_t n_new, int64_t first, const int* row_src,
                 Buf& staging) {
    if (first >= n_new || base == nullptr) return 0;
    const int64_t w16 = (int64_t)(row_bytes / 16);
    const int64_t chunk = std::max<int64_t>(1, (int64_t)(kStagingBytes / row_bytes));
    HRAG_TRY(staging.ensure((size_t)std::min(chunk, n_new - first) * row_bytes));
    for (int64_t r0 = first; r0 < n_new; r0 += chunk) {
        const int64_t n = std::min(chunk, n_new - r0);
        k_gather_rows<<<blocks_for(n * w16), kThreads, 0, h->stream>>>(n, w16, row_src, r0, (const int4*)base,
                                                                         staging.as<int4>());
        HRAG_CUDA(cudaGetLastError());
        HRAG_CUDA(cudaMemcpyAsync(static_cast<char*>(base) + (size_t)r0 * row_bytes, staging.p, (size_t)n * row_bytes,
                                  cudaMemcpyDeviceToDevice, h->stream));
    }
    return 0;
}

int gather_rows(hrag_t* h, const void* base, size_t row_bytes, const int* row_src, int64_t n_rows, void* out) {
    if (n_rows == 0) return 0;
    const int64_t w16 = (int64_t)(row_bytes / 16);
    k_gather_rows<<<blocks_for(n_rows * w16), kThreads, 0, h->stream>>>(n_rows, w16, row_src, 0, (const int4*)base,
                                                                          static_cast<int4*>(out));
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

namespace {

bool borrowed(const EmbMem& e) { return e.f32 != nullptr && e.own.p == nullptr; }
// the fp32 rows a fresh load of this matrix keeps: an owned matrix, or an empty one (loaded from host memory, it
// would own its rows); a streamed matrix (hrag_load_embeddings_begin) keeps only its bf16 planes
bool keeps_f32(const EmbMem& e) { return e.rows == 0 || e.own.p != nullptr; }
bool has_split(const hrag_t* h) { return h->dim % 8 == 0; }

// The preconditions every update entry shares.
int check_updatable(hrag_t* h, const std::string& who) {
    HRAG_CHECK(h, who + ": null handle");
    HRAG_TRY(check_index_private(h, who));
    HRAG_CHECK(h->world == 1, who + ": a node-range-sharded handle (world > 1) cannot be updated in place; reload it");
    HRAG_CHECK(!emb_planes(h, 0).streams(), who + ": the fact planes are held in host memory (hrag_set_fact_memory) and cannot "
                                         "be updated in place; reload the index");
    HRAG_CHECK(h->g.cv, who + ": no graph loaded");
    HRAG_CHECK(h->mutable_index, who + ": the handle is not mutable: call hrag_set_mutable(h, 1) before the graph is "
                                       "loaded through hrag_load_graph_coo or hrag_load_graph_coo_device");
    HRAG_CHECK(h->graph.edges.src.p, who + ": the handle keeps no edge list (the graph was loaded from a CSR, or "
                                           "before hrag_set_mutable(h, 1)): reload it through hrag_load_graph_coo");
    HRAG_CHECK(h->t.passage_vid, who + ": load the tables first");
    HRAG_CHECK(h->dim > 0 && h->emb[0].rows == h->t.n_facts && h->emb[1].rows == h->t.n_passages,
               who + ": load fact and passage embeddings with one row per fact / passage of the tables first");
    HRAG_CHECK(!borrowed(h->emb[0]), who + ": the fp32 fact embeddings are borrowed from the caller (device load) and "
                                           "cannot be changed in place; load them from host memory");
    HRAG_CHECK(!borrowed(h->emb[1]), who + ": the fp32 passage embeddings are borrowed from the caller (device load) "
                                           "and cannot be changed in place; load them from host memory");
    HRAG_CUDA(cudaSetDevice(h->device));
    return 0;
}

// After a failure past validation: no graph, no tables, no embeddings rather than a half-updated index.
void drop_index(hrag_t* h) {
    invalidate_solves(h);    // synchronises `stream` first: nothing still reads what is freed below
    h->graph = GraphMem{};
    h->g = PprGraph();
    h->tables = TableMem{};
    h->t = SeedTables();
    h->emb[0] = EmbMem{};
    h->emb[1] = EmbMem{};
    h->dim = 0;
    h->n_facts_global = h->fact_row_lo = 0;
}

// What every update ends with: the captured mixed solves were captured for the old N and P, so they go, whether or
// not an allocation they point into was freed; the slot maps are rebuilt from the new passage_vid.
int finish_update(hrag_t* h) {
    HRAG_TRY(invalidate_solves(h));
    g_buf_generation += 1;
    h->n_facts_global = h->emb[0].rows;
    h->fact_row_lo = 0;
    return 0;
}

// Installs the planes of `csr` (coo_to_csr of `edges`, n_nodes vertices) and keeps `edges` as the handle's list.
int rebuild_graph(hrag_t* h, int64_t n_nodes, const DeviceCsr& csr, EdgeList&& edges) {
    HRAG_TRY(install_graph(h, n_nodes, 0, n_nodes, csr.nnz, csr.row_ptr.as<int64_t>(), 0, csr.col.as<int32_t>(),
                           nullptr, csr.val.as<double>(), h->row_bounds));
    h->graph.edges = std::move(edges);
    return 0;
}

// n_new rows (host or device) appended to embedding matrix `which`: the owned fp32 rows grow, and the new rows alone
// are split into the tails of the bf16 hi / lo planes.
int append_rows(hrag_t* h, int which, int64_t n_new, const float* rows, bool on_device) {
    EmbMem& e = h->emb[which];
    if (n_new == 0) return 0;
    const size_t d = (size_t)h->dim, old = (size_t)e.rows, add = (size_t)n_new;
    const float* src = rows;
    Buf staging;
    if (keeps_f32(e)) {
        HRAG_TRY(grow_keep(h, e.own, old * d * 4, (old + add) * d * 4));
        e.f32 = e.own.as<float>();
        HRAG_TRY(copy_in(h, e.own.as<float>() + old * d, rows, (int64_t)(add * d), on_device));
        src = e.f32 + old * d;
    } else if (!on_device) {
        HRAG_TRY(staging.ensure(add * d * 4));
        HRAG_TRY(h2d(h, staging.p, rows, add * d * 4));
        src = staging.as<float>();
    }
    if (has_split(h)) {
        HRAG_TRY(grow_keep(h, e.hi, old * d * 2, (old + add) * d * 2));
        HRAG_TRY(grow_keep(h, e.lo, old * d * 2, (old + add) * d * 2));
        HRAG_TRY(split_bf16(src, (int64_t)(add * d), static_cast<char*>(e.hi.p) + old * d * 2,
                            static_cast<char*>(e.lo.p) + old * d * 2, h->stream));
        // the norm maxima only grow: still bounds after deletes (compact_matrix), raised here by the new rows
        if (which == 0) HRAG_TRY(fact_norms_update(h, (int64_t)old, (int64_t)add, false));
    }
    HRAG_CUDA(cudaStreamSynchronize(h->stream));   // the staging buffer is freed on return
    e.rows = (int64_t)(old + add);
    return 0;
}

// The rows of embedding matrix `which` become its rows row_src[0 .. n_new), every plane compacted in place from row
// `first` (the first dropped row) on.
int compact_matrix(hrag_t* h, int which, int64_t n_new, int64_t first, const int* row_src, Buf& staging) {
    EmbMem& e = h->emb[which];
    const size_t d = (size_t)h->dim;
    if (e.own.p) HRAG_TRY(compact_rows(h, e.own.p, d * 4, n_new, first, row_src, staging));
    HRAG_TRY(compact_rows(h, e.hi.p, d * 2, n_new, first, row_src, staging));
    HRAG_TRY(compact_rows(h, e.lo.p, d * 2, n_new, first, row_src, staging));
    e.rows = n_new;
    if (n_new == 0 && keeps_f32(e)) e.f32 = nullptr;   // as hrag_load_embeddings leaves an empty matrix
    return 0;
}

}  // namespace

int copy_edge_list(hrag_t* h, int64_t n, const int32_t* src, const int32_t* dst, const double* w, EdgeList* out) {
    const size_t m = (size_t)std::max<int64_t>(n, 1);
    HRAG_TRY(out->src.ensure(m * sizeof(int32_t)));
    HRAG_TRY(out->dst.ensure(m * sizeof(int32_t)));
    HRAG_TRY(out->w.ensure(m * sizeof(double)));
    HRAG_TRY(copy_in(h, out->src.as<int32_t>(), src, n, true));
    HRAG_TRY(copy_in(h, out->dst.as<int32_t>(), dst, n, true));
    HRAG_TRY(copy_in(h, out->w.as<double>(), w, n, true));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    out->n = n;
    return 0;
}

}  // namespace hrag

using namespace hrag;

extern "C" {

int hrag_set_mutable(hrag_t* h, int on) {
    HRAG_CHECK(h, "hrag_set_mutable: null handle");
    h->mutable_index = on != 0;
    return 0;
}

int hrag_index_reserve(hrag_t* h, int64_t nodes, int64_t edges, int64_t facts, int64_t passages) {
    const std::string who = "hrag_index_reserve";
    HRAG_TRY(check_updatable(h, who));
    HRAG_CHECK(nodes >= 0 && edges >= 0 && facts >= 0 && passages >= 0, who + ": negative capacity");
    HRAG_CHECK(nodes < (int64_t)1 << 30 && edges < (int64_t)1 << 30 && passages < (int64_t)1 << 31,
               who + ": capacity out of range");
    EdgeList& E = h->graph.edges;
    const size_t ne = (size_t)E.n, nf = (size_t)h->t.n_facts, np = (size_t)h->t.n_passages;
    const size_t N = (size_t)h->g.n_global, d = (size_t)h->dim;
    HRAG_TRY(grow_keep(h, E.src, ne * 4, (size_t)edges * 4));
    HRAG_TRY(grow_keep(h, E.dst, ne * 4, (size_t)edges * 4));
    HRAG_TRY(grow_keep(h, E.w, ne * 8, (size_t)edges * 8));
    TableMem& T = h->tables;
    HRAG_TRY(grow_keep(h, T.passage_vid, np * 4, (size_t)passages * 4));
    HRAG_TRY(grow_keep(h, T.fact_subj_vid, nf * 4, (size_t)facts * 4));
    HRAG_TRY(grow_keep(h, T.fact_obj_vid, nf * 4, (size_t)facts * 4));
    HRAG_TRY(grow_keep(h, T.ent_chunk_count, N * 4, (size_t)nodes * 4));
    for (int which = 0; which < 2; ++which) {
        EmbMem& e = h->emb[which];
        const size_t rows = (size_t)e.rows, want = (size_t)(which == 0 ? facts : passages);
        if (want <= rows) continue;
        if (keeps_f32(e)) {
            HRAG_TRY(grow_keep(h, e.own, rows * d * 4, want * d * 4));
            if (rows) e.f32 = e.own.as<float>();
        }
        if (has_split(h)) {
            HRAG_TRY(grow_keep(h, e.hi, rows * d * 2, want * d * 2));
            HRAG_TRY(grow_keep(h, e.lo, rows * d * 2, want * d * 2));
        }
    }
    h->t.passage_vid = T.passage_vid.as<int>();
    h->t.fact_subj_vid = T.fact_subj_vid.as<int>();
    h->t.fact_obj_vid = T.fact_obj_vid.as<int>();
    h->t.ent_chunk_count = T.ent_chunk_count.as<int>();
    return finish_update(h);
}

int hrag_index_append(hrag_t* h, int64_t n_new_nodes, int64_t n_new_edges, const int32_t* src, const int32_t* dst,
                      const double* w, int64_t n_new_passages, const int32_t* passage_vid, int64_t n_new_facts,
                      const int32_t* fact_subj_vid, const int32_t* fact_obj_vid, const int32_t* ent_chunk_count,
                      int32_t dim, const float* fact_emb, const float* passage_emb, int on_device) {
    const std::string who = "hrag_index_append";
    HRAG_TRY(check_updatable(h, who));
    HRAG_CHECK(n_new_nodes >= 0 && n_new_edges >= 0 && n_new_passages >= 0 && n_new_facts >= 0,
               who + ": negative count");
    HRAG_CHECK(ent_chunk_count && (n_new_edges == 0 || (src && dst && w)) &&
                   (n_new_passages == 0 || (passage_vid && passage_emb)) &&
                   (n_new_facts == 0 || (fact_subj_vid && fact_obj_vid && fact_emb)),
               who + ": null argument");
    HRAG_CHECK(dim == h->dim, who + ": the new embedding rows have dim " + std::to_string(dim) + ", the index " +
                                  std::to_string(h->dim));
    EdgeList& E = h->graph.edges;
    const int64_t N = h->g.n_global + n_new_nodes, n_edges = E.n + n_new_edges;
    const int64_t P = h->t.n_passages + n_new_passages, F = h->t.n_facts + n_new_facts;
    HRAG_CHECK(N < (int64_t)1 << 30 && n_edges < (int64_t)1 << 30 && P < (int64_t)1 << 31 && F < (int64_t)1 << 31,
               who + ": sizes out of range");
    const bool dev_edges = on_device & HRAG_DEVICE_EDGES;
    if (!dev_edges)
        for (int64_t i = 0; i < n_new_edges; ++i)
            HRAG_CHECK(src[i] >= 0 && src[i] < N && dst[i] >= 0 && dst[i] < N, who + ": edge endpoint out of range");
    for (int64_t p = 0; p < n_new_passages; ++p)
        HRAG_CHECK(passage_vid[p] >= 0 && passage_vid[p] < N, who + ": passage_vid out of range");
    for (int64_t f = 0; f < n_new_facts; ++f)
        HRAG_CHECK(fact_subj_vid[f] < N && fact_obj_vid[f] < N, who + ": fact vertex id out of range");
    if (dev_edges && n_new_edges) {   // a device edge list is checked on the device
        Buf bad;
        HRAG_TRY(bad.zeros(sizeof(unsigned long long)));
        k_count_bad_edges<<<blocks_for(n_new_edges), kThreads, 0, h->stream>>>(n_new_edges, N, src, dst,
                                                                                 bad.as<unsigned long long>());
        HRAG_CUDA(cudaGetLastError());
        unsigned long long n_bad = 0;
        HRAG_CUDA(cudaMemcpyAsync(&n_bad, bad.p, sizeof n_bad, cudaMemcpyDeviceToHost, h->stream));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
        HRAG_CHECK(n_bad == 0, who + ": edge endpoint out of range");
    }
    // The new edges go past the E.n edges in use (the list may move to a larger allocation, its contents do not
    // change) and the CSR of the grown list is built; the handle's index is unchanged until install_graph, so a list
    // whose CSR does not fit int32 is still rejected cleanly.
    HRAG_TRY(grow_keep(h, E.src, (size_t)E.n * 4, (size_t)n_edges * 4));
    HRAG_TRY(grow_keep(h, E.dst, (size_t)E.n * 4, (size_t)n_edges * 4));
    HRAG_TRY(grow_keep(h, E.w, (size_t)E.n * 8, (size_t)n_edges * 8));
    HRAG_TRY(copy_in(h, E.src.as<int32_t>() + E.n, src, n_new_edges, dev_edges));
    HRAG_TRY(copy_in(h, E.dst.as<int32_t>() + E.n, dst, n_new_edges, dev_edges));
    HRAG_TRY(copy_in(h, E.w.as<double>() + E.n, w, n_new_edges, dev_edges));
    DeviceCsr csr;
    bool bad_edges = false;
    HRAG_TRY(coo_to_csr(h, N, n_edges, E.src.as<int32_t>(), E.dst.as<int32_t>(), E.w.as<double>(), &csr, &bad_edges));
    HRAG_CHECK(!bad_edges, who + ": edge endpoint out of range");
    HRAG_CHECK(csr.nnz < ((int64_t)1 << 31) - 8, who + ": nnz must fit int32");

    auto apply = [&]() -> int {
        EdgeList edges = std::move(E);
        edges.n = n_edges;
        HRAG_TRY(rebuild_graph(h, N, csr, std::move(edges)));
        TableMem& T = h->tables;
        const int64_t P0 = h->t.n_passages, F0 = h->t.n_facts;
        HRAG_TRY(grow_keep(h, T.passage_vid, (size_t)P0 * 4, (size_t)P * 4));
        HRAG_TRY(grow_keep(h, T.fact_subj_vid, (size_t)F0 * 4, (size_t)F * 4));
        HRAG_TRY(grow_keep(h, T.fact_obj_vid, (size_t)F0 * 4, (size_t)F * 4));
        HRAG_TRY(T.ent_chunk_count.ensure((size_t)N * 4));
        HRAG_TRY(copy_in(h, T.passage_vid.as<int32_t>() + P0, passage_vid, n_new_passages, false));
        HRAG_TRY(copy_in(h, T.fact_subj_vid.as<int32_t>() + F0, fact_subj_vid, n_new_facts, false));
        HRAG_TRY(copy_in(h, T.fact_obj_vid.as<int32_t>() + F0, fact_obj_vid, n_new_facts, false));
        HRAG_TRY(copy_in(h, T.ent_chunk_count.as<int32_t>(), ent_chunk_count, N, false));
        h->t = SeedTables{(int)N, (int)P, F, T.passage_vid.as<int>(), T.fact_subj_vid.as<int>(),
                          T.fact_obj_vid.as<int>(), T.ent_chunk_count.as<int>()};
        HRAG_TRY(append_rows(h, 0, n_new_facts, fact_emb, on_device & HRAG_DEVICE_FACT_EMB));
        HRAG_TRY(append_rows(h, 1, n_new_passages, passage_emb, on_device & HRAG_DEVICE_PASSAGE_EMB));
        return finish_update(h);
    };
    if (const int rc = apply()) { drop_index(h); return rc; }
    return 0;
}

int hrag_index_delete(hrag_t* h, int64_t n_del_nodes, const int32_t* del_nodes, int64_t n_del_facts,
                      const int32_t* del_facts, const int32_t* ent_chunk_count) {
    const std::string who = "hrag_index_delete";
    HRAG_TRY(check_updatable(h, who));
    const int64_t N0 = h->g.n_global, F0 = h->t.n_facts, P0 = h->t.n_passages;
    HRAG_CHECK(n_del_nodes >= 0 && n_del_facts >= 0, who + ": negative count");
    HRAG_CHECK(ent_chunk_count && (n_del_nodes == 0 || del_nodes) && (n_del_facts == 0 || del_facts),
               who + ": null argument");
    HRAG_CHECK(n_del_nodes < N0, who + ": a graph keeps at least one vertex");
    for (int64_t i = 0; i < n_del_nodes; ++i)
        HRAG_CHECK(del_nodes[i] >= 0 && del_nodes[i] < N0 && (i == 0 || del_nodes[i] > del_nodes[i - 1]),
                   who + ": vertex ids must be sorted, unique and in range");
    for (int64_t i = 0; i < n_del_facts; ++i)
        HRAG_CHECK(del_facts[i] >= 0 && del_facts[i] < F0 && (i == 0 || del_facts[i] > del_facts[i - 1]),
                   who + ": fact rows must be sorted, unique and in range");
    const int64_t N = N0 - n_del_nodes;

    auto apply = [&]() -> int {
        cudaStream_t st = h->stream;
        Buf d_del_nodes, d_del_facts, vflags, vmap;
        HRAG_TRY(d_del_nodes.ensure((size_t)std::max<int64_t>(n_del_nodes, 1) * 4));
        HRAG_TRY(d_del_facts.ensure((size_t)std::max<int64_t>(n_del_facts, 1) * 4));
        HRAG_TRY(copy_in(h, d_del_nodes.as<int32_t>(), del_nodes, n_del_nodes, false));
        HRAG_TRY(copy_in(h, d_del_facts.as<int32_t>(), del_facts, n_del_facts, false));
        // vertex keep-flags -> exclusive scan -> old -> new id map (-1 = deleted)
        HRAG_TRY(vflags.ensure((size_t)(N0 + 1) * 4));
        HRAG_TRY(vmap.ensure((size_t)(N0 + 1) * 4));
        k_keep_unlisted<<<blocks_for(N0 + 1), kThreads, 0, st>>>(N0, d_del_nodes.as<int32_t>(), n_del_nodes,
                                                                  vflags.as<int>());
        HRAG_CUDA(cudaGetLastError());
        int64_t kept = 0;
        HRAG_TRY(scan_flags(h, N0, vflags.as<int>(), vmap.as<int>(), &kept));
        k_vertex_map<<<blocks_for(N0), kThreads, 0, st>>>(N0, vflags.as<int>(), vmap.as<int>());
        HRAG_CUDA(cudaGetLastError());
        const int* map = vmap.as<int>();

        // the edge list: stable compaction + relabel into a list of the same capacity, then the graph planes
        EdgeList& E = h->graph.edges;
        const int64_t n0 = E.n;
        Buf eflags, epos;
        HRAG_TRY(eflags.ensure((size_t)(n0 + 1) * 4));
        HRAG_TRY(epos.ensure((size_t)(n0 + 1) * 4));
        k_edge_flags<<<blocks_for(n0 + 1), kThreads, 0, st>>>(n0, E.src.as<int32_t>(), E.dst.as<int32_t>(), map,
                                                               eflags.as<int>());
        HRAG_CUDA(cudaGetLastError());
        int64_t n_edges = 0;
        HRAG_TRY(scan_flags(h, n0, eflags.as<int>(), epos.as<int>(), &n_edges));
        EdgeList edges;
        HRAG_TRY(edges.src.ensure(E.src.cap));
        HRAG_TRY(edges.dst.ensure(E.dst.cap));
        HRAG_TRY(edges.w.ensure(E.w.cap));
        if (n0)
            k_edge_scatter<<<blocks_for(n0), kThreads, 0, st>>>(n0, E.src.as<int32_t>(), E.dst.as<int32_t>(),
                                                                E.w.as<double>(), map, eflags.as<int>(), epos.as<int>(),
                                                                edges.src.as<int32_t>(), edges.dst.as<int32_t>(),
                                                                edges.w.as<double>());
        HRAG_CUDA(cudaGetLastError());
        edges.n = n_edges;
        eflags.reset();
        epos.reset();
        {
            DeviceCsr csr;
            bool bad_edges = false;
            HRAG_TRY(coo_to_csr(h, N, n_edges, edges.src.as<int32_t>(), edges.dst.as<int32_t>(), edges.w.as<double>(),
                                &csr, &bad_edges));
            HRAG_CHECK(!bad_edges, "internal: " + who + " relabelled an edge out of range");
            HRAG_TRY(rebuild_graph(h, N, csr, std::move(edges)));
        }

        // passages whose vertex went are dropped, the others relabelled; facts dropped as listed, ids relabelled
        TableMem& T = h->tables;
        TableMem nt;
        Buf pflags, ppos, prow, fflags, fpos, frow, staging;
        HRAG_TRY(pflags.ensure((size_t)(P0 + 1) * 4));
        HRAG_TRY(ppos.ensure((size_t)(P0 + 1) * 4));
        HRAG_TRY(prow.ensure((size_t)std::max<int64_t>(P0, 1) * 4));
        k_passage_flags<<<blocks_for(P0 + 1), kThreads, 0, st>>>(P0, T.passage_vid.as<int32_t>(), map,
                                                                  pflags.as<int>());
        HRAG_CUDA(cudaGetLastError());
        int64_t P = 0, p_first = 0;
        HRAG_TRY(scan_flags(h, P0, pflags.as<int>(), ppos.as<int>(), &P, &p_first));
        HRAG_TRY(nt.passage_vid.ensure(T.passage_vid.cap));
        if (P0)
            k_passage_scatter<<<blocks_for(P0), kThreads, 0, st>>>(P0, T.passage_vid.as<int32_t>(), map,
                                                                   pflags.as<int>(), ppos.as<int>(),
                                                                   nt.passage_vid.as<int32_t>(), prow.as<int>());
        HRAG_CUDA(cudaGetLastError());
        HRAG_TRY(fflags.ensure((size_t)(F0 + 1) * 4));
        HRAG_TRY(fpos.ensure((size_t)(F0 + 1) * 4));
        HRAG_TRY(frow.ensure((size_t)std::max<int64_t>(F0, 1) * 4));
        k_keep_unlisted<<<blocks_for(F0 + 1), kThreads, 0, st>>>(F0, d_del_facts.as<int32_t>(), n_del_facts,
                                                                  fflags.as<int>());
        HRAG_CUDA(cudaGetLastError());
        int64_t F = 0;
        HRAG_TRY(scan_flags(h, F0, fflags.as<int>(), fpos.as<int>(), &F));
        const int64_t f_first = n_del_facts ? del_facts[0] : F0;
        HRAG_TRY(nt.fact_subj_vid.ensure(T.fact_subj_vid.cap));
        HRAG_TRY(nt.fact_obj_vid.ensure(T.fact_obj_vid.cap));
        if (F0)
            k_fact_scatter<<<blocks_for(F0), kThreads, 0, st>>>(F0, T.fact_subj_vid.as<int32_t>(),
                                                                T.fact_obj_vid.as<int32_t>(), map, fflags.as<int>(),
                                                                fpos.as<int>(), nt.fact_subj_vid.as<int32_t>(),
                                                                nt.fact_obj_vid.as<int32_t>(), frow.as<int>());
        HRAG_CUDA(cudaGetLastError());
        nt.ent_chunk_count = std::move(T.ent_chunk_count);   // N <= N0 entries fit
        HRAG_TRY(copy_in(h, nt.ent_chunk_count.as<int32_t>(), ent_chunk_count, N, false));
        HRAG_CUDA(cudaStreamSynchronize(st));
        h->tables = std::move(nt);
        h->t = SeedTables{(int)N, (int)P, F, h->tables.passage_vid.as<int>(), h->tables.fact_subj_vid.as<int>(),
                          h->tables.fact_obj_vid.as<int>(), h->tables.ent_chunk_count.as<int>()};
        HRAG_TRY(compact_matrix(h, 0, F, f_first, frow.as<int>(), staging));
        HRAG_TRY(compact_matrix(h, 1, P, p_first, prow.as<int>(), staging));
        HRAG_CUDA(cudaStreamSynchronize(st));   // the staging and row lists are freed on return
        return finish_update(h);
    };
    if (const int rc = apply()) { drop_index(h); return rc; }
    return 0;
}

int hrag_debug_index(hrag_t* h, int plane, void* host_out, int64_t max_bytes, int64_t* n_written) {
    HRAG_CHECK(h && n_written, "hrag_debug_index: null argument");
    HRAG_CHECK(plane >= 0 && plane <= 12, "hrag_debug_index: plane must be in [0, 12]");
    const SeedTables& t = h->t;
    const EdgeList& E = h->graph.edges;
    const int64_t d = h->dim, F = h->emb[0].rows, P = h->emb[1].rows;
    const PlaneSet fp = emb_planes(h, 0);   // a fact plane may be in pinned host memory (hrag_set_fact_memory)
    const void* src[13] = {t.passage_vid, t.fact_subj_vid, t.fact_obj_vid, t.ent_chunk_count, fp.plane[0], fp.plane[1],
                           h->emb[1].hi.p, h->emb[1].lo.p,
                           h->emb[0].f32, h->emb[1].f32, E.src.p, E.dst.p, E.w.p};
    const int64_t bytes[13] = {4 * (int64_t)t.n_passages, 4 * t.n_facts, 4 * t.n_facts,
                               t.ent_chunk_count ? 4 * (int64_t)t.n_nodes : 0,
                               2 * F * d, 2 * F * d, 2 * P * d, 2 * P * d, 4 * F * d, 4 * P * d,
                               4 * E.n, 4 * E.n, 8 * E.n};
    *n_written = src[plane] ? bytes[plane] : 0;
    if (!host_out) return 0;
    HRAG_CHECK(*n_written <= max_bytes, "hrag_debug_index: host buffer too small");
    HRAG_CUDA(cudaSetDevice(h->device));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    if (*n_written) HRAG_CUDA(cudaMemcpy(host_out, src[plane], (size_t)*n_written, cudaMemcpyDefault));
    return 0;
}

}  // extern "C"
