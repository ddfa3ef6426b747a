// The PPR operator built on the device: every graph loader ends in install_graph, and the COO loaders start with
// coo_to_csr.  Together they build, byte for byte, the planes a sequential host build makes from the same input:
// parallel edges summed in input order, vertex strengths summed in column order within the row, one correctly rounded
// fp64 division per non-zero, round-to-nearest fp32 planes, the rows of each 64-row block ordered by length (stable)
// and rows longer than 256 non-zeros cut into 256-non-zero segments.  The summation orders are what a solver's last
// bits depend on, so no step reduces in a tree: each run and each row is summed by one thread, front to back.
#include <cub/cub.cuh>

#include "handle.h"

namespace hrag {
namespace {

constexpr int kThreads = 256;
constexpr int kSegLen = 256;     // long rows: segment length in non-zeros (and the length above which a row is long)

int blocks_for(int64_t n) { return (int)ceil_div(std::max<int64_t>(n, 1), kThreads); }

__device__ __forceinline__ int64_t thread_index() { return blockIdx.x * (int64_t)blockDim.x + threadIdx.x; }

// Edge i -> entry 2i = (a -> b) and entry 2i + 1 = (b -> a), keyed row << bits | col, payload w.  An edge whose
// weight is not > 0 (NaN included) carries nothing: both entries get the key `drop`, above every real key, so the sort
// moves them to the end.  flags[0] != 0: an endpoint lies outside [0, n); flags[1] = entries kept.
__global__ void k_coo_expand(int64_t n_edges, int64_t n, int bits, const int32_t* __restrict__ src,
                             const int32_t* __restrict__ dst, const double* __restrict__ w, uint64_t* __restrict__ keys,
                             double* __restrict__ vals, unsigned long long* flags) {
    const int64_t i = thread_index();
    bool kept = false;
    if (i < n_edges) {
        const int64_t a = src[i], b = dst[i];
        const double x = w[i];
        uint64_t k0 = 1ull << (2 * bits), k1 = k0;
        if (a < 0 || a >= n || b < 0 || b >= n) {
            flags[0] = 1;
        } else if (x > 0.0) {
            k0 = ((uint64_t)a << bits) | (uint64_t)b;
            k1 = ((uint64_t)b << bits) | (uint64_t)a;
            kept = true;
        }
        keys[2 * i] = k0;
        keys[2 * i + 1] = k1;
        vals[2 * i] = x;
        vals[2 * i + 1] = x;
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, kept);
    if ((threadIdx.x & 31) == 0 && ballot) atomicAdd(&flags[1], 2ull * (unsigned)__popc(ballot));
}

// head[i] = 1 where a run of equal keys starts (the inclusive scan of it numbers the merged entries from 1)
__global__ void k_run_heads(int64_t m, const uint64_t* __restrict__ keys, unsigned long long* __restrict__ head) {
    const int64_t i = thread_index();
    if (i < m) head[i] = i == 0 || keys[i] != keys[i - 1];
}

// One thread per run: the parallel edges of (row, col) summed in sorted (= input) order, starting from 0.0
__global__ void k_merge_runs(int64_t m, const uint64_t* __restrict__ keys, const double* __restrict__ vals,
                             const unsigned long long* __restrict__ slot, uint64_t col_mask, int32_t* __restrict__ col,
                             double* __restrict__ wsum) {
    const int64_t i = thread_index();
    if (i >= m || (i > 0 && keys[i] == keys[i - 1])) return;
    const uint64_t k = keys[i];
    double s = 0.0;
    for (int64_t j = i; j < m && keys[j] == k; ++j) s += vals[j];
    col[slot[i] - 1] = (int32_t)(k & col_mask);
    wsum[slot[i] - 1] = s;
}

// row_ptr[r] = merged entries with a row below r = slot[p - 1], p = the first sorted entry of a row >= r
__global__ void k_merged_row_ptr(int64_t n, int64_t m, const uint64_t* __restrict__ keys,
                                 const unsigned long long* __restrict__ slot, int bits, int64_t* __restrict__ row_ptr) {
    const int64_t r = thread_index();
    if (r > n) return;
    const uint64_t target = (uint64_t)r << bits;
    int64_t lo = 0, hi = m;
    while (lo < hi) {
        const int64_t mid = (lo + hi) / 2;
        if (keys[mid] < target) lo = mid + 1;
        else hi = mid;
    }
    row_ptr[r] = lo == 0 ? 0 : (int64_t)slot[lo - 1];
}

// strength[r] = the row's merged weights summed in column order, starting from 0.0 (W is symmetric: row sums = column
// sums); the hub rows of power-law graphs make this one long dependent chain per thread, by design
__global__ void k_strength(int64_t n, const int64_t* __restrict__ row_ptr, const double* __restrict__ wsum,
                           double* __restrict__ strength) {
    const int64_t r = thread_index();
    if (r >= n) return;
    double s = 0.0;
    for (int64_t k = row_ptr[r]; k < row_ptr[r + 1]; ++k) s += wsum[k];
    strength[r] = s;
}

__global__ void k_normalise(int64_t nnz, const int32_t* __restrict__ col, const double* __restrict__ strength,
                            double* __restrict__ val) {
    const int64_t k = thread_index();
    if (k < nnz) val[k] = val[k] / strength[col[k]];
}

// ---- finishing pass (every loader)

__global__ void k_local_row_ptr(int n_rows, const int64_t* __restrict__ row_ptr, int64_t base, int* __restrict__ rp) {
    const int64_t r = thread_index();
    if (r <= n_rows) rp[r] = (int)(row_ptr[r] - base);
}

// cv = {col, fp32 bits of the value}; from fp64 values hi = fp32(val) and lo = fp32(val - hi), both rounded to nearest
__global__ void k_pack(int64_t nnz, const int32_t* __restrict__ col, const float* __restrict__ val,
                       const double* __restrict__ val64, int2* __restrict__ cv, float* __restrict__ lo) {
    const int64_t k = thread_index();
    if (k >= nnz) return;
    if (val64) {
        const double v = val64[k];
        const float hi = __double2float_rn(v);
        cv[k] = make_int2(col[k], __float_as_int(hi));
        lo[k] = __double2float_rn(v - (double)hi);
    } else {
        cv[k] = make_int2(col[k], __float_as_int(val[k]));
    }
}

// One CTA of 64 threads per 64-row block: the rows by length descending, ties by row ascending (a stable sort of the
// block by length), each thread placing its row at its rank
__global__ void __launch_bounds__(64) k_row_order(int n_rows, const int* __restrict__ rp, int* __restrict__ order) {
    __shared__ int len[64];
    const int b0 = blockIdx.x * 64, t = threadIdx.x, cnt = min(64, n_rows - b0);
    if (t < cnt) len[t] = rp[b0 + t + 1] - rp[b0 + t];
    __syncthreads();
    if (t >= cnt) return;
    const int L = len[t];
    int rank = 0;
    for (int j = 0; j < cnt; ++j) rank += len[j] > L || (len[j] == L && j < t);
    order[b0 + rank] = b0 + t;
}

// cnt[r] = (1 << 32 | segments of row r) for a long row, 0 otherwise, and cnt[n_rows] = 0: one exclusive scan then
// gives every long row its index (high word) and its first segment (low word), and the totals at [n_rows]
__global__ void k_long_count(int n_rows, const int* __restrict__ rp, unsigned long long* __restrict__ cnt) {
    const int64_t r = thread_index();
    if (r > n_rows) return;
    const int len = r < n_rows ? rp[r + 1] - rp[r] : 0;
    cnt[r] = len > kSegLen ? (1ull << 32) | (unsigned long long)((len + kSegLen - 1) / kSegLen) : 0ull;
}

__global__ void k_long_fill(int n_rows, int n_long, const int* __restrict__ rp, const unsigned long long* __restrict__ scan,
                            int* __restrict__ long_rows, int* __restrict__ long_seg_ptr, int4* __restrict__ segs) {
    const int64_t r = thread_index();
    if (r >= n_rows) return;
    const int s = rp[r], e = rp[r + 1];
    if (e - s <= kSegLen) return;
    const int li = (int)(scan[r] >> 32);
    int so = (int)(scan[r] & 0xffffffffu);
    long_rows[li] = (int)r;
    long_seg_ptr[li] = so;
    for (int a = s; a < e; a += kSegLen) segs[so++] = make_int4((int)r, a, min(e, a + kSegLen), 0);
    if (li == n_long - 1) long_seg_ptr[n_long] = so;
}

template <class T> int read_back(T* host, const void* dev, cudaStream_t st) {
    HRAG_CUDA(cudaMemcpyAsync(host, dev, sizeof(T), cudaMemcpyDeviceToHost, st));
    HRAG_CUDA(cudaStreamSynchronize(st));
    return 0;
}

}  // namespace

int coo_to_csr(hrag_t* h, int64_t n, int64_t n_edges, const int32_t* src, const int32_t* dst, const double* w,
               DeviceCsr* out, bool* bad_edges) {
    cudaStream_t st = h->stream;
    int bits = 0;
    while (((int64_t)1 << bits) < n) ++bits;
    const int64_t entries = 2 * n_edges;
    // scratch: the double-buffered sort, 2 x (8-B key + 8-B weight) per entry
    Buf keys[2], vals[2], flags, tmp, strength;
    for (int b = 0; b < 2; ++b) {
        HRAG_TRY(keys[b].ensure((size_t)std::max<int64_t>(entries, 1) * sizeof(uint64_t)));
        HRAG_TRY(vals[b].ensure((size_t)std::max<int64_t>(entries, 1) * sizeof(double)));
    }
    HRAG_TRY(flags.ensure(2 * sizeof(unsigned long long)));
    HRAG_CUDA(cudaMemsetAsync(flags.p, 0, 2 * sizeof(unsigned long long), st));
    if (n_edges)
        k_coo_expand<<<blocks_for(n_edges), kThreads, 0, st>>>(n_edges, n, bits, src, dst, w, keys[0].as<uint64_t>(),
                                                                vals[0].as<double>(), flags.as<unsigned long long>());
    HRAG_CUDA(cudaGetLastError());
    unsigned long long hf[2];
    HRAG_CUDA(cudaMemcpyAsync(hf, flags.p, sizeof hf, cudaMemcpyDeviceToHost, st));
    HRAG_CUDA(cudaStreamSynchronize(st));
    *bad_edges = hf[0] != 0;
    if (*bad_edges) return 0;
    const int64_t m = (int64_t)hf[1];   // kept entries: the first m after the sort

    // stable LSD radix sort over the key bits in use (the dropped key is bit 2 * bits): parallel edges keep input order
    cub::DoubleBuffer<uint64_t> dk(keys[0].as<uint64_t>(), keys[1].as<uint64_t>());
    cub::DoubleBuffer<double> dv(vals[0].as<double>(), vals[1].as<double>());
    if (entries) {
        size_t tb = 0;
        HRAG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)entries, 0, 2 * bits + 1, st));
        HRAG_TRY(tmp.ensure(tb));
        HRAG_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, dk, dv, (int)entries, 0, 2 * bits + 1, st));
    }
    const uint64_t* K = dk.Current();
    const double* V = dv.Current();

    // the run numbering goes into the sort's other key buffer, free now (a 64-bit scan: CUB's 32-bit one spills)
    unsigned long long* slot = reinterpret_cast<unsigned long long*>(dk.Alternate());
    unsigned long long nnz = 0;
    if (m) {
        k_run_heads<<<blocks_for(m), kThreads, 0, st>>>(m, K, slot);
        HRAG_CUDA(cudaGetLastError());
        size_t tb = 0;
        HRAG_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb, slot, slot, (int)m, st));
        HRAG_TRY(tmp.ensure(tb));
        HRAG_CUDA(cub::DeviceScan::InclusiveSum(tmp.p, tb, slot, slot, (int)m, st));
        HRAG_TRY(read_back(&nnz, slot + (m - 1), st));
    }
    out->nnz = (int64_t)nnz;
    HRAG_TRY(out->row_ptr.ensure((size_t)(n + 1) * sizeof(int64_t)));
    HRAG_TRY(out->col.ensure((size_t)std::max(nnz, 1ull) * sizeof(int32_t)));
    HRAG_TRY(out->val.ensure((size_t)std::max(nnz, 1ull) * sizeof(double)));
    HRAG_TRY(strength.ensure((size_t)n * sizeof(double)));
    int32_t* col = out->col.as<int32_t>();
    double* val = out->val.as<double>();
    int64_t* row_ptr = out->row_ptr.as<int64_t>();
    if (m)
        k_merge_runs<<<blocks_for(m), kThreads, 0, st>>>(m, K, V, slot, ((uint64_t)1 << bits) - 1, col, val);
    k_merged_row_ptr<<<blocks_for(n + 1), kThreads, 0, st>>>(n, m, K, slot, bits, row_ptr);
    k_strength<<<blocks_for(n), kThreads, 0, st>>>(n, row_ptr, val, strength.as<double>());
    if (nnz) k_normalise<<<blocks_for(nnz), kThreads, 0, st>>>(nnz, col, strength.as<double>(), val);
    HRAG_CUDA(cudaGetLastError());
    HRAG_CUDA(cudaStreamSynchronize(st));   // the scratch is freed on return
    return 0;
}

int install_graph(hrag_t* h, int64_t n_nodes, int64_t row_lo, int64_t row_hi, int64_t nnz, const int64_t* row_ptr,
                  int64_t base, const int32_t* col, const float* val, const double* val64,
                  const std::vector<int64_t>& bounds) {
    cudaStream_t st = h->stream;
    PprGraph g;
    g.num_sms = h->num_sms;
    g.n_global = (int)n_nodes;
    g.row_lo = (int)row_lo;
    g.n_rows = (int)(row_hi - row_lo);
    g.nnz = nnz;
    g.long_thresh = kSegLen;
    g.max_batch = 64;
    const int n_rows = g.n_rows;

    // every input is valid: the old graph, the fp32 state sized for it, the slot maps and the captured solves go first
    // (a reload never holds two graphs); the new graph becomes the handle's
    // only once all of it is built (a failure leaves no graph; the next load frees what was allocated)
    HRAG_TRY(invalidate_solves(h));
    h->graph = GraphMem{};
    h->g = PprGraph();
    h->V.reset(); h->XA.reset(); h->XC.reset(); h->partials.reset();
    h->row_bounds = bounds;
    h->chunk_rows = h->world > 1 ? ceil_div(n_nodes, h->world) : n_nodes;
    GraphMem& m = h->graph;
    HRAG_TRY(m.row_ptr.ensure((size_t)(n_rows + 1) * sizeof(int)));
    g.row_ptr = m.row_ptr.as<int>();
    k_local_row_ptr<<<blocks_for(n_rows + 1), kThreads, 0, st>>>(n_rows, row_ptr, base, g.row_ptr);
    HRAG_TRY(m.cv.ensure(nnz ? (size_t)nnz * sizeof(int2) : 1));       // non-null: marks a loaded graph
    g.cv = m.cv.as<int2>();
    if (val64) {                                                        // non-null: marks an fp64 operator
        HRAG_TRY(m.val_lo.ensure(nnz ? (size_t)nnz * sizeof(float) : 1));
        g.val_lo = m.val_lo.as<float>();
    }
    if (nnz) k_pack<<<blocks_for(nnz), kThreads, 0, st>>>(nnz, col, val, val64, g.cv, g.val_lo);
    HRAG_TRY(m.row_order.ensure(n_rows ? (size_t)n_rows * sizeof(int) : 1));
    g.row_order = m.row_order.as<int>();
    if (n_rows) k_row_order<<<(unsigned)ceil_div(n_rows, 64), 64, 0, st>>>(n_rows, g.row_ptr, g.row_order);

    Buf scan, tmp;
    HRAG_TRY(scan.ensure((size_t)(n_rows + 1) * sizeof(unsigned long long)));
    auto* cnt = scan.as<unsigned long long>();
    k_long_count<<<blocks_for(n_rows + 1), kThreads, 0, st>>>(n_rows, g.row_ptr, cnt);
    HRAG_CUDA(cudaGetLastError());
    size_t tb = 0;
    HRAG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, cnt, n_rows + 1, st));
    HRAG_TRY(tmp.ensure(tb));
    HRAG_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, cnt, cnt, n_rows + 1, st));
    unsigned long long total = 0;
    HRAG_TRY(read_back(&total, cnt + n_rows, st));
    g.n_long = (int)(total >> 32);
    g.n_seg = (int)(total & 0xffffffffu);
    if (g.n_long) {
        HRAG_TRY(m.long_rows.ensure((size_t)g.n_long * sizeof(int)));
        HRAG_TRY(m.long_seg_ptr.ensure((size_t)(g.n_long + 1) * sizeof(int)));
        HRAG_TRY(m.segs.ensure((size_t)g.n_seg * sizeof(int4)));
        g.long_rows = m.long_rows.as<int>();
        g.long_seg_ptr = m.long_seg_ptr.as<int>();
        g.segs = m.segs.as<int4>();
        k_long_fill<<<blocks_for(n_rows), kThreads, 0, st>>>(n_rows, g.n_long, g.row_ptr, cnt, g.long_rows,
                                                               g.long_seg_ptr, g.segs);
        HRAG_TRY(m.seg_partial.ensure((size_t)g.n_seg * g.max_batch * sizeof(float)));
        g.seg_partial = m.seg_partial.as<float>();
    }
    HRAG_CUDA(cudaGetLastError());
    HRAG_CUDA(cudaStreamSynchronize(st));
    h->g = g;
    return 0;
}

}  // namespace hrag
