// Uploads: the graph (CSR or COO, fp32 or fp64 values, COO from host or device arrays), the seed tables and the
// embedding matrices.  The graph and table loaders check every input (a device edge list: on the device) before they
// touch the handle, so a rejected load leaves the handle as it was; a load that fails after that leaves no graph (no
// tables) rather than a half-loaded one.  The graph planes themselves are built on the device (graph_build.cu).
#include <algorithm>

#include "handle.h"

namespace {
using namespace hrag;

// rank r gets rows [b[r], b[r + 1]) with equal shares of cost = non-zeros + 4 per row (the epilogue streams of a row
// cost about as much as four gathers); a contiguous split by row COUNT gives the rank that holds the passage rows
// (35 non-zeros each on the synthetic graphs, 12 elsewhere) 1.4x (2 ranks) to 2.3x (8 ranks) the work of the others
std::vector<int64_t> balanced_bounds(const int64_t* row_ptr, int64_t n_nodes, int world) {
    std::vector<int64_t> b((size_t)world + 1, n_nodes);
    b[0] = 0;
    const double total = (double)row_ptr[n_nodes] + 4.0 * (double)n_nodes;
    int64_t r = 0;
    for (int k = 1; k < world; ++k) {
        const double want = total * k / world;
        while (r < n_nodes && (double)row_ptr[r] + 4.0 * (double)r < want) ++r;
        b[(size_t)k] = r;
    }
    return b;
}

template <class T> int upload_to(hrag_t* h, Buf& b, const T* src, size_t n) {   // ordered before h->stream's work
    HRAG_TRY(b.ensure(n ? n * sizeof(T) : 1));
    if (n) HRAG_CUDA(cudaMemcpyAsync(b.p, src, n * sizeof(T), cudaMemcpyHostToDevice, h->stream));
    return 0;
}

// The two CSR entries share this: exactly one of val (fp32) / val64 is given.  Checks every input on the host, then
// uploads it and builds the planes on the device (install_graph: from val64 the fp32 plane cv stores fp32(val64) --
// bitwise what the fp32 entry stores for that rounding -- and the lo plane fp32(val64 - hi)).
int load_graph_csr_impl(hrag_t* h, const std::string& who, int64_t n_nodes, int64_t row_lo, int64_t row_hi,
                        int64_t nnz, const int64_t* row_ptr, const int32_t* col, const float* val,
                        const double* val64) {
    HRAG_CHECK(h && row_ptr && (nnz == 0 || (col && (val || val64))), who + ": null argument");
    HRAG_TRY(check_index_private(h, who));
    HRAG_CHECK(n_nodes > 0 && n_nodes < (int64_t)1 << 30, who + ": n_nodes out of range");
    HRAG_CHECK(nnz >= 0 && nnz < ((int64_t)1 << 31) - 8, who + ": nnz must fit int32");
    HRAG_CHECK(0 <= row_lo && row_lo <= row_hi && row_hi <= n_nodes, who + ": bad row range");
    HRAG_CUDA(cudaSetDevice(h->device));
    const std::vector<int64_t>& bounds = h->row_bounds;
    const int64_t n_rows = row_hi - row_lo;
    HRAG_CHECK(row_ptr[0] == 0 && row_ptr[n_rows] == nnz, who + ": row_ptr does not span nnz");
    if (h->world > 1) {
        HRAG_CHECK(bounds.empty() || bounds.back() == n_nodes,
                   who + ": hrag_comm_set_row_bounds was given bounds for a different vertex count");
        const int64_t chunk = ceil_div(n_nodes, h->world);   // the given bounds, else equal row counts
        const int64_t lo = bounds.empty() ? std::min<int64_t>(n_nodes, h->rank * chunk) : bounds[h->rank];
        const int64_t hi = bounds.empty() ? std::min<int64_t>(n_nodes, (h->rank + 1) * chunk) : bounds[h->rank + 1];
        HRAG_CHECK(row_lo == lo && row_hi == hi,
                   who + ": sharded ranks own rows [rank*ceil(N/world), (rank+1)*ceil(N/world)), or the range "
                   "given by hrag_comm_set_row_bounds");
    }
    for (int64_t r = 0; r < n_rows; ++r)
        HRAG_CHECK(row_ptr[r] <= row_ptr[r + 1] && row_ptr[r + 1] <= nnz, who + ": row_ptr not monotone");
    for (int64_t i = 0; i < nnz; ++i)
        HRAG_CHECK(col[i] >= 0 && col[i] < n_nodes, who + ": column index out of range");
    Buf d_row_ptr, d_col, d_val;   // the old graph stays until all of the input is on the device
    HRAG_TRY(upload_to(h, d_row_ptr, row_ptr, (size_t)n_rows + 1));
    HRAG_TRY(upload_to(h, d_col, col, (size_t)nnz));
    if (val64) HRAG_TRY(upload_to(h, d_val, val64, (size_t)nnz));
    else HRAG_TRY(upload_to(h, d_val, val, (size_t)nnz));
    return install_graph(h, n_nodes, row_lo, row_hi, nnz, d_row_ptr.as<int64_t>(), 0, d_col.as<int32_t>(),
                         val64 ? nullptr : d_val.as<float>(), val64 ? d_val.as<double>() : nullptr, bounds);
}

// The two COO entries share this: src / dst / w are device pointers, sizes checked.  The edge list is validated on
// the device before the handle is touched; with node-range sharding every rank builds the whole CSR, derives the same
// work-balanced partition from its row_ptr and keeps its own rows.
int load_graph_coo_impl(hrag_t* h, const std::string& who, int64_t n_nodes, int64_t n_edges, const int32_t* src,
                        const int32_t* dst, const double* w) {
    DeviceCsr csr;
    bool bad_edges = false;
    HRAG_TRY(coo_to_csr(h, n_nodes, n_edges, src, dst, w, &csr, &bad_edges));
    HRAG_CHECK(!bad_edges, who + ": edge endpoint out of range");
    int64_t lo = 0, hi = n_nodes, a = 0, b = csr.nnz;
    std::vector<int64_t> bounds = h->row_bounds;
    if (h->world > 1) {
        std::vector<int64_t> row_ptr((size_t)n_nodes + 1);
        HRAG_CUDA(cudaMemcpy(row_ptr.data(), csr.row_ptr.p, row_ptr.size() * sizeof(int64_t), cudaMemcpyDeviceToHost));
        bounds = balanced_bounds(row_ptr.data(), n_nodes, h->world);
        lo = bounds[h->rank], hi = bounds[h->rank + 1];
        a = row_ptr[(size_t)lo], b = row_ptr[(size_t)hi];
    }
    HRAG_CHECK(b - a < ((int64_t)1 << 31) - 8, who + ": nnz must fit int32");
    EdgeList kept;   // a mutable handle keeps the list itself for hrag_index_append / hrag_index_delete
    if (h->mutable_index && h->world == 1) HRAG_TRY(copy_edge_list(h, n_edges, src, dst, w, &kept));
    // fp64 values: the same fp32 plane as the fp64 CSR entry, plus the lo plane hrag_ppr_f64 needs
    HRAG_TRY(install_graph(h, n_nodes, lo, hi, b - a, csr.row_ptr.as<int64_t>() + lo, a, csr.col.as<int32_t>() + a,
                           nullptr, csr.val.as<double>() + a, bounds));
    if (kept.src.p) h->graph.edges = std::move(kept);
    return 0;
}

// Drops embedding matrix `which`, sets dim and the rows of a `rows`-row matrix that this handle keeps (node-range
// sharding gives rank r the fact rows [r * ceil(F / world), ...)); returns the first of them.
int64_t reset_embeddings(hrag_t* h, int which, int64_t rows, int32_t dim) {
    h->emb[which] = EmbMem{};
    if (which == 0) h->fplanes.release();
    h->dim = dim;
    int64_t lo = 0, hi = rows;
    if (which == 0) {
        h->n_facts_global = rows;
        if (h->world > 1) {
            const int64_t chunk = ceil_div(rows, h->world);
            lo = std::min<int64_t>(rows, h->rank * chunk);
            hi = std::min<int64_t>(rows, (h->rank + 1) * chunk);
        }
        h->fact_row_lo = lo;
    }
    h->emb[which].rows = hi - lo;
    return lo;
}

}  // namespace

extern "C" {

int hrag_load_graph_csr(hrag_t* h, int64_t n_nodes, int64_t row_lo, int64_t row_hi, int64_t nnz,
                        const int64_t* row_ptr, const int32_t* col, const float* val) {
    return load_graph_csr_impl(h, "hrag_load_graph_csr", n_nodes, row_lo, row_hi, nnz, row_ptr, col, val, nullptr);
}

int hrag_load_graph_csr_f64(hrag_t* h, int64_t n_nodes, int64_t row_lo, int64_t row_hi, int64_t nnz,
                            const int64_t* row_ptr, const int32_t* col, const double* val) {
    return load_graph_csr_impl(h, "hrag_load_graph_csr_f64", n_nodes, row_lo, row_hi, nnz, row_ptr, col, nullptr, val);
}

int hrag_load_graph_coo(hrag_t* h, int64_t n_nodes, int64_t n_edges, const int32_t* src, const int32_t* dst,
                        const double* w) {
    HRAG_CHECK(h && (n_edges == 0 || (src && dst && w)), "hrag_load_graph_coo: null argument");
    HRAG_TRY(check_index_private(h, "hrag_load_graph_coo"));
    HRAG_CHECK(n_nodes > 0 && n_nodes < (int64_t)1 << 30 && n_edges >= 0 && n_edges < (int64_t)1 << 30,
               "hrag_load_graph_coo: sizes out of range");
    for (int64_t i = 0; i < n_edges; ++i)
        HRAG_CHECK(src[i] >= 0 && src[i] < n_nodes && dst[i] >= 0 && dst[i] < n_nodes,
                   "hrag_load_graph_coo: edge endpoint out of range");
    HRAG_CUDA(cudaSetDevice(h->device));
    Buf d_src, d_dst, d_w;
    HRAG_TRY(upload_to(h, d_src, src, (size_t)n_edges));
    HRAG_TRY(upload_to(h, d_dst, dst, (size_t)n_edges));
    HRAG_TRY(upload_to(h, d_w, w, (size_t)n_edges));
    return load_graph_coo_impl(h, "hrag_load_graph_coo", n_nodes, n_edges, d_src.as<int32_t>(), d_dst.as<int32_t>(),
                               d_w.as<double>());
}

int hrag_load_graph_coo_device(hrag_t* h, int64_t n_nodes, int64_t n_edges, const int32_t* d_src,
                               const int32_t* d_dst, const double* d_w) {
    HRAG_CHECK(h && (n_edges == 0 || (d_src && d_dst && d_w)), "hrag_load_graph_coo_device: null argument");
    HRAG_TRY(check_index_private(h, "hrag_load_graph_coo_device"));
    HRAG_CHECK(n_nodes > 0 && n_nodes < (int64_t)1 << 30 && n_edges >= 0 && n_edges < (int64_t)1 << 30,
               "hrag_load_graph_coo_device: sizes out of range");
    HRAG_CUDA(cudaSetDevice(h->device));
    return load_graph_coo_impl(h, "hrag_load_graph_coo_device", n_nodes, n_edges, d_src, d_dst, d_w);
}

int hrag_load_tables(hrag_t* h, int64_t n_passages, const int32_t* passage_vid, int64_t n_facts,
                     const int32_t* fact_subj_vid, const int32_t* fact_obj_vid, const int32_t* ent_chunk_count) {
    HRAG_CHECK(h, "hrag_load_tables: null handle");
    HRAG_TRY(check_index_private(h, "hrag_load_tables"));
    HRAG_CHECK(h->g.n_global > 0, "hrag_load_tables: load the graph first");
    HRAG_CHECK(n_passages >= 0 && n_passages < (int64_t)1 << 31 && n_facts >= 0, "hrag_load_tables: bad sizes");
    HRAG_CUDA(cudaSetDevice(h->device));
    const int N = h->g.n_global;
    for (int64_t p = 0; p < n_passages; ++p)
        HRAG_CHECK(passage_vid[p] >= 0 && passage_vid[p] < N, "hrag_load_tables: passage_vid out of range");
    for (int64_t f = 0; f < n_facts; ++f)
        HRAG_CHECK(fact_subj_vid[f] < N && fact_obj_vid[f] < N, "hrag_load_tables: fact vertex id out of range");
    // every input is valid: the old tables go first; a failed upload leaves none (passage_vid, uploaded last, is null)
    HRAG_TRY(invalidate_solves(h));
    h->tables = TableMem{};
    h->t = SeedTables();
    HRAG_TRY(h->tables.fact_subj_vid.upload(fact_subj_vid, (size_t)n_facts, &h->t.fact_subj_vid));
    HRAG_TRY(h->tables.fact_obj_vid.upload(fact_obj_vid, (size_t)n_facts, &h->t.fact_obj_vid));
    HRAG_TRY(h->tables.ent_chunk_count.upload(ent_chunk_count, (size_t)N, &h->t.ent_chunk_count));
    HRAG_TRY(h->tables.passage_vid.upload(passage_vid, (size_t)n_passages, &h->t.passage_vid));
    h->t.n_nodes = N;
    h->t.n_passages = (int)n_passages;
    h->t.n_facts = n_facts;
    return 0;
}

int hrag_load_embeddings(hrag_t* h, int which, int64_t rows, int32_t dim, const float* emb, int on_device) {
    HRAG_CHECK(h && (which == 0 || which == 1), "hrag_load_embeddings: which must be 0 (fact) or 1 (passage)");
    HRAG_TRY(check_index_private(h, "hrag_load_embeddings"));
    HRAG_CHECK(rows >= 0 && dim > 0 && dim % 4 == 0, "hrag_load_embeddings: dim must be a positive multiple of 4");
    HRAG_CHECK(rows == 0 || emb != nullptr, "hrag_load_embeddings: null embeddings");
    HRAG_CHECK(h->dim == 0 || h->dim == dim || h->emb[1 - which].rows == 0,
               "hrag_load_embeddings: fact and passage embeddings must share dim");
    int64_t slice_rows = 0;   // > 0: the fact planes go to pinned host memory (hrag_set_fact_memory)
    bool hi_resident = false;   // only the lo plane does (HRAG_FACT_LO_ON_HOST)
    if (which == 0) HRAG_TRY(fact_planes_plan(h, "hrag_load_embeddings", rows, dim, &slice_rows, &hi_resident));
    HRAG_CHECK(!slice_rows || !on_device,
               "hrag_load_embeddings: the fact planes exceed the hrag_set_fact_memory budget and go to host memory; "
               "pass the fp32 fact rows from host memory (on the device they would take the memory the budget keeps "
               "free)");
    HRAG_CUDA(cudaSetDevice(h->device));
    emb += (size_t)reset_embeddings(h, which, rows, dim) * dim;
    EmbMem& e = h->emb[which];
    if (e.rows == 0) return 0;
    if (slice_rows) {   // no fp32 copy is kept, as with the streamed loader
        HRAG_TRY(fact_planes_alloc(h, slice_rows, hi_resident));
        return fact_planes_fill(h, 0, e.rows, emb, false);
    }
    if (on_device) e.f32 = emb;   // caller keeps it alive
    else HRAG_TRY(e.own.upload(emb, (size_t)e.rows * dim, &e.f32));
    if (dim % 8 == 0) {   // bf16 hi/lo split for the tensor-core similarity kernel
        const size_t n = (size_t)e.rows * dim;
        HRAG_TRY(e.hi.ensure(n * 2));
        HRAG_TRY(e.lo.ensure(n * 2));
        HRAG_TRY(split_bf16(e.f32, (int64_t)n, e.hi.p, e.lo.p, h->stream));
        if (which == 0) HRAG_TRY(fact_norms_update(h, 0, e.rows, true));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
    }
    return 0;
}

int hrag_load_embeddings_begin(hrag_t* h, int which, int64_t rows, int32_t dim) {
    HRAG_CHECK(h && (which == 0 || which == 1), "hrag_load_embeddings_begin: which must be 0 (fact) or 1 (passage)");
    HRAG_TRY(check_index_private(h, "hrag_load_embeddings_begin"));
    HRAG_CHECK(rows > 0 && dim > 0 && dim % 8 == 0, "hrag_load_embeddings_begin: rows > 0 and dim a multiple of 8");
    HRAG_CHECK(h->dim == 0 || h->dim == dim || h->emb[1 - which].rows == 0,
               "hrag_load_embeddings_begin: fact and passage embeddings must share dim");
    int64_t slice_rows = 0;
    bool hi_resident = false;
    if (which == 0) HRAG_TRY(fact_planes_plan(h, "hrag_load_embeddings_begin", rows, dim, &slice_rows, &hi_resident));
    HRAG_CUDA(cudaSetDevice(h->device));
    reset_embeddings(h, which, rows, dim);
    if (slice_rows) return fact_planes_alloc(h, slice_rows, hi_resident);
    const size_t n = (size_t)std::max<int64_t>(h->emb[which].rows, 1) * dim;
    HRAG_TRY(h->emb[which].hi.ensure(n * 2));
    HRAG_TRY(h->emb[which].lo.ensure(n * 2));
    if (which == 0) {   // the chunks raise the norm maxima from zero
        HRAG_TRY(fact_norms_update(h, 0, 0, true));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
    }
    return 0;
}

int hrag_load_embeddings_chunk(hrag_t* h, int which, int64_t row0, int64_t n_rows, const float* emb, int on_device) {
    HRAG_CHECK(h && (which == 0 || which == 1) && emb, "hrag_load_embeddings_chunk: bad arguments");
    HRAG_TRY(check_index_private(h, "hrag_load_embeddings_chunk"));
    const EmbMem& e = h->emb[which];
    const bool host_planes = emb_planes(h, which).streams();   // both planes, or lo only (fact_planes_fill)
    HRAG_CHECK((e.hi.p != nullptr || host_planes) && e.f32 == nullptr,
               "hrag_load_embeddings_chunk: call hrag_load_embeddings_begin first");
    HRAG_CUDA(cudaSetDevice(h->device));
    const int64_t lo = which == 0 ? h->fact_row_lo : 0, hi = lo + e.rows;
    const int64_t total = which == 0 ? h->n_facts_global : e.rows;
    HRAG_CHECK(row0 >= 0 && n_rows >= 0 && row0 + n_rows <= total, "hrag_load_embeddings_chunk: rows out of range");
    const int64_t a = std::max(row0, lo), b = std::min(row0 + n_rows, hi);      // the part this handle keeps
    if (a >= b) return 0;
    const size_t n = (size_t)(b - a) * h->dim;
    const float* src = emb + (size_t)(a - row0) * h->dim;
    if (host_planes) return fact_planes_fill(h, a, b - a, src, on_device != 0);
    if (!on_device) {
        HRAG_TRY(h->d_reset.ensure(n * sizeof(float)));                          // staging
        HRAG_CUDA(cudaMemcpyAsync(h->d_reset.p, src, n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
        src = h->d_reset.as<float>();
    }
    HRAG_TRY(split_bf16(src, (int64_t)n, static_cast<char*>(e.hi.p) + (size_t)(a - lo) * h->dim * 2,
                        static_cast<char*>(e.lo.p) + (size_t)(a - lo) * h->dim * 2, h->stream));
    if (which == 0) HRAG_TRY(fact_norms_update(h, a - lo, b - a, false));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    return 0;
}

}  // extern "C"
