// Uploads: the graph (CSR or COO, fp32 or fp64 values), the seed tables and the embedding matrices.  The graph and
// table loaders check every input on the host before they touch the handle, so a rejected load leaves the handle as
// it was; an upload that fails after that leaves no graph (no tables) rather than a half-loaded one.
#include <algorithm>
#include <cstring>

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

// The two CSR entries and the COO entry share this: exactly one of val (fp32) / val64 is given.  From val64 the fp32
// plane cv stores fp32(val64) -- bitwise what the fp32 entry stores for that rounding -- and the lo plane
// fp32(val64 - hi).  new_bounds: the row partition to install instead of the handle's (node-range sharding).
int load_graph_csr_impl(hrag_t* h, const std::string& who, int64_t n_nodes, int64_t row_lo, int64_t row_hi,
                        int64_t nnz, const int64_t* row_ptr, const int32_t* col, const float* val,
                        const double* val64, const std::vector<int64_t>* new_bounds = nullptr) {
    HRAG_CHECK(h && row_ptr && (nnz == 0 || (col && (val || val64))), who + ": null argument");
    HRAG_CHECK(n_nodes > 0 && n_nodes < (int64_t)1 << 30, who + ": n_nodes out of range");
    HRAG_CHECK(nnz >= 0 && nnz < ((int64_t)1 << 31) - 8, who + ": nnz must fit int32");
    HRAG_CHECK(0 <= row_lo && row_lo <= row_hi && row_hi <= n_nodes, who + ": bad row range");
    HRAG_CUDA(cudaSetDevice(h->device));
    const std::vector<int64_t>& bounds = new_bounds ? *new_bounds : h->row_bounds;
    const int n_rows = (int)(row_hi - row_lo);
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
    PprGraph g;
    g.num_sms = h->num_sms;
    g.n_global = (int)n_nodes;
    g.row_lo = (int)row_lo;
    g.n_rows = n_rows;
    g.nnz = nnz;
    g.long_thresh = 256;
    g.max_batch = 64;
    std::vector<int> rp(n_rows + 1);
    std::vector<int2> cv((size_t)nnz);
    std::vector<float> lo(val64 ? (size_t)nnz : 0);
    std::vector<int> long_rows, long_seg_ptr;
    std::vector<int4> segs;
    const int seg_len = 256;
    for (int r = 0; r < n_rows; ++r) {
        const int64_t s = row_ptr[r], e = row_ptr[r + 1];
        HRAG_CHECK(s <= e && e <= nnz, who + ": row_ptr not monotone");
        rp[r] = (int)s;
        if (e - s > g.long_thresh) {
            long_rows.push_back(r);
            long_seg_ptr.push_back((int)segs.size());
            for (int64_t a = s; a < e; a += seg_len)
                segs.push_back(make_int4(r, (int)a, (int)std::min<int64_t>(e, a + seg_len), 0));
        }
    }
    rp[n_rows] = (int)nnz;
    long_seg_ptr.push_back((int)segs.size());
    for (int64_t i = 0; i < nnz; ++i) {
        HRAG_CHECK(col[i] >= 0 && col[i] < n_nodes, who + ": column index out of range");
        const float hi = val64 ? (float)val64[i] : val[i];
        int bits;
        memcpy(&bits, &hi, 4);
        cv[(size_t)i] = make_int2(col[i], bits);
        if (val64) lo[(size_t)i] = (float)(val64[i] - (double)hi);
    }
    // fp16 sweep: within each block of 64 rows (one CTA) order the rows by length so a warp's 8 rows match
    std::vector<int> order(n_rows);
    for (int r = 0; r < n_rows; ++r) order[r] = r;
    for (int b0 = 0; b0 < n_rows; b0 += 64) {
        const int b1 = std::min(n_rows, b0 + 64);
        std::stable_sort(order.begin() + b0, order.begin() + b1,
                         [&](int x, int y) { return rp[x + 1] - rp[x] > rp[y + 1] - rp[y]; });
    }
    g.n_long = (int)long_rows.size();
    g.n_seg = (int)segs.size();

    // every input is valid: the old graph and the fp32 state sized for it go first (a reload never holds two graphs;
    // the frees bump g_buf_generation, which invalidates every captured solve); the new graph becomes the handle's
    // only once all of it is uploaded (a failed upload leaves no graph; the next load frees what it allocated)
    h->graph = GraphMem{};
    h->g = PprGraph();
    h->V.reset(); h->XA.reset(); h->XC.reset(); h->partials.reset();
    h->slot_maps_valid = false;
    h->row_bounds = bounds;
    h->chunk_rows = h->world > 1 ? ceil_div(n_nodes, h->world) : n_nodes;
    HRAG_TRY(h->graph.row_ptr.upload(rp.data(), rp.size(), &g.row_ptr));
    HRAG_TRY(h->graph.cv.upload(cv.data(), cv.size(), &g.cv));                    // non-null: marks a loaded graph
    HRAG_TRY(h->graph.row_order.upload(order.data(), order.size(), &g.row_order));
    if (val64) HRAG_TRY(h->graph.val_lo.upload(lo.data(), lo.size(), &g.val_lo));   // non-null: marks an fp64 operator
    if (g.n_long) {
        HRAG_TRY(h->graph.long_rows.upload(long_rows.data(), long_rows.size(), &g.long_rows));
        HRAG_TRY(h->graph.long_seg_ptr.upload(long_seg_ptr.data(), long_seg_ptr.size(), &g.long_seg_ptr));
        HRAG_TRY(h->graph.segs.upload(segs.data(), segs.size(), &g.segs));
        HRAG_TRY(h->graph.seg_partial.ensure(segs.size() * (size_t)g.max_batch * sizeof(float)));
        g.seg_partial = h->graph.seg_partial.as<float>();
        if (val64) HRAG_TRY(h->graph.seg_partial64.ensure(segs.size() * 16 * sizeof(double)));
        g.seg_partial64 = h->graph.seg_partial64.as<double>();
    }
    h->g = g;
    return 0;
}

// Drops embedding matrix `which`, sets dim and the rows of a `rows`-row matrix that this handle keeps (node-range
// sharding gives rank r the fact rows [r * ceil(F / world), ...)); returns the first of them.
int64_t reset_embeddings(hrag_t* h, int which, int64_t rows, int32_t dim) {
    h->emb[which] = EmbMem{};
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
    HRAG_CHECK(n_nodes > 0 && n_nodes < (int64_t)1 << 30 && n_edges >= 0 && n_edges < (int64_t)1 << 30,
               "hrag_load_graph_coo: sizes out of range");
    // symmetrise: (row, col, w) for both directions, keyed row-major
    struct Ent { uint64_t key; double w; };
    std::vector<Ent> e;
    e.reserve((size_t)n_edges * 2);
    for (int64_t i = 0; i < n_edges; ++i) {
        const int64_t a = src[i], b = dst[i];
        HRAG_CHECK(a >= 0 && a < n_nodes && b >= 0 && b < n_nodes, "hrag_load_graph_coo: edge endpoint out of range");
        if (!(w[i] > 0.0)) continue;                       // non-positive (and NaN) weights carry nothing
        e.push_back({((uint64_t)a << 32) | (uint64_t)b, w[i]});
        e.push_back({((uint64_t)b << 32) | (uint64_t)a, w[i]});
    }
    std::stable_sort(e.begin(), e.end(), [](const Ent& x, const Ent& y) { return x.key < y.key; });
    std::vector<int64_t> row_ptr((size_t)n_nodes + 1, 0);
    std::vector<int32_t> col;
    std::vector<double> wsum;
    col.reserve(e.size());
    wsum.reserve(e.size());
    for (size_t i = 0; i < e.size();) {                    // merge parallel edges in input order
        size_t j = i;
        double s = 0.0;
        while (j < e.size() && e[j].key == e[i].key) s += e[j++].w;
        col.push_back((int32_t)(e[i].key & 0xffffffffu));
        wsum.push_back(s);
        row_ptr[(size_t)(e[i].key >> 32) + 1] += 1;
        i = j;
    }
    for (int64_t r = 0; r < n_nodes; ++r) row_ptr[(size_t)r + 1] += row_ptr[(size_t)r];
    std::vector<double> strength((size_t)n_nodes, 0.0);    // W is symmetric: column sums = row sums
    for (int64_t r = 0; r < n_nodes; ++r)
        for (int64_t k = row_ptr[(size_t)r]; k < row_ptr[(size_t)r + 1]; ++k) strength[(size_t)r] += wsum[(size_t)k];
    std::vector<double> val(col.size());
    for (size_t k = 0; k < col.size(); ++k) val[k] = wsum[k] / strength[(size_t)col[k]];
    int64_t lo = 0, hi = n_nodes;
    std::vector<int64_t> bounds = h->row_bounds;
    if (h->world > 1) {
        // every rank sees the whole edge list here, so all of them derive the same work-balanced partition
        bounds = balanced_bounds(row_ptr.data(), n_nodes, h->world);
        lo = bounds[h->rank], hi = bounds[h->rank + 1];
    }
    const int64_t a = row_ptr[(size_t)lo], b = row_ptr[(size_t)hi];
    std::vector<int64_t> rp((size_t)(hi - lo) + 1);
    for (int64_t r = lo; r <= hi; ++r) rp[(size_t)(r - lo)] = row_ptr[(size_t)r] - a;
    // fp64 values: the same fp32 plane as before, plus the lo plane hrag_ppr_f64 needs
    return load_graph_csr_impl(h, "hrag_load_graph_csr", n_nodes, lo, hi, b - a, rp.data(), col.data() + a, nullptr,
                               val.data() + a, &bounds);
}

int hrag_load_tables(hrag_t* h, int64_t n_passages, const int32_t* passage_vid, int64_t n_facts,
                     const int32_t* fact_subj_vid, const int32_t* fact_obj_vid, const int32_t* ent_chunk_count) {
    HRAG_CHECK(h, "hrag_load_tables: null handle");
    HRAG_CHECK(h->g.n_global > 0, "hrag_load_tables: load the graph first");
    HRAG_CHECK(n_passages >= 0 && n_passages < (int64_t)1 << 31 && n_facts >= 0, "hrag_load_tables: bad sizes");
    HRAG_CUDA(cudaSetDevice(h->device));
    const int N = h->g.n_global;
    for (int64_t p = 0; p < n_passages; ++p)
        HRAG_CHECK(passage_vid[p] >= 0 && passage_vid[p] < N, "hrag_load_tables: passage_vid out of range");
    for (int64_t f = 0; f < n_facts; ++f)
        HRAG_CHECK(fact_subj_vid[f] < N && fact_obj_vid[f] < N, "hrag_load_tables: fact vertex id out of range");
    // every input is valid: the old tables go first; a failed upload leaves none (passage_vid, uploaded last, is null)
    h->tables = TableMem{};
    h->t = SeedTables();
    h->slot_maps_valid = false;
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
    HRAG_CHECK(rows >= 0 && dim > 0 && dim % 4 == 0, "hrag_load_embeddings: dim must be a positive multiple of 4");
    HRAG_CHECK(rows == 0 || emb != nullptr, "hrag_load_embeddings: null embeddings");
    HRAG_CHECK(h->dim == 0 || h->dim == dim || h->emb[1 - which].rows == 0,
               "hrag_load_embeddings: fact and passage embeddings must share dim");
    HRAG_CUDA(cudaSetDevice(h->device));
    emb += (size_t)reset_embeddings(h, which, rows, dim) * dim;
    EmbMem& e = h->emb[which];
    if (e.rows == 0) return 0;
    if (on_device) e.f32 = emb;   // caller keeps it alive
    else HRAG_TRY(e.own.upload(emb, (size_t)e.rows * dim, &e.f32));
    if (dim % 8 == 0) {   // bf16 hi/lo split for the tensor-core similarity kernel
        const size_t n = (size_t)e.rows * dim;
        HRAG_TRY(e.hi.ensure(n * 2));
        HRAG_TRY(e.lo.ensure(n * 2));
        HRAG_TRY(split_bf16(e.f32, (int64_t)n, e.hi.p, e.lo.p, h->stream));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
    }
    return 0;
}

int hrag_load_embeddings_begin(hrag_t* h, int which, int64_t rows, int32_t dim) {
    HRAG_CHECK(h && (which == 0 || which == 1), "hrag_load_embeddings_begin: which must be 0 (fact) or 1 (passage)");
    HRAG_CHECK(rows > 0 && dim > 0 && dim % 8 == 0, "hrag_load_embeddings_begin: rows > 0 and dim a multiple of 8");
    HRAG_CHECK(h->dim == 0 || h->dim == dim || h->emb[1 - which].rows == 0,
               "hrag_load_embeddings_begin: fact and passage embeddings must share dim");
    HRAG_CUDA(cudaSetDevice(h->device));
    reset_embeddings(h, which, rows, dim);
    const size_t n = (size_t)std::max<int64_t>(h->emb[which].rows, 1) * dim;
    HRAG_TRY(h->emb[which].hi.ensure(n * 2));
    HRAG_TRY(h->emb[which].lo.ensure(n * 2));
    return 0;
}

int hrag_load_embeddings_chunk(hrag_t* h, int which, int64_t row0, int64_t n_rows, const float* emb, int on_device) {
    HRAG_CHECK(h && (which == 0 || which == 1) && emb, "hrag_load_embeddings_chunk: bad arguments");
    const EmbMem& e = h->emb[which];
    HRAG_CHECK(e.hi.p != nullptr && e.f32 == nullptr,
               "hrag_load_embeddings_chunk: call hrag_load_embeddings_begin first");
    HRAG_CUDA(cudaSetDevice(h->device));
    const int64_t lo = which == 0 ? h->fact_row_lo : 0, hi = lo + e.rows;
    const int64_t total = which == 0 ? h->n_facts_global : e.rows;
    HRAG_CHECK(row0 >= 0 && n_rows >= 0 && row0 + n_rows <= total, "hrag_load_embeddings_chunk: rows out of range");
    const int64_t a = std::max(row0, lo), b = std::min(row0 + n_rows, hi);      // the part this handle keeps
    if (a >= b) return 0;
    const size_t n = (size_t)(b - a) * h->dim;
    const float* src = emb + (size_t)(a - row0) * h->dim;
    if (!on_device) {
        HRAG_TRY(h->d_reset.ensure(n * sizeof(float)));                          // staging
        HRAG_CUDA(cudaMemcpyAsync(h->d_reset.p, src, n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
        src = h->d_reset.as<float>();
    }
    HRAG_TRY(split_bf16(src, (int64_t)n, static_cast<char*>(e.hi.p) + (size_t)(a - lo) * h->dim * 2,
                        static_cast<char*>(e.lo.p) + (size_t)(a - lo) * h->dim * 2, h->stream));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    return 0;
}

}  // extern "C"
