// K1 -- batched CSR SpMM sweep of the Personalized-PageRank iteration (sm_90a).
//
// Replaces the numeric core of HippoRAG.run_ppr (reference HippoRAG.py:1736-1743, which
// hands one reset vector at a time to igraph/PRPACK) with a batched fixed-point sweep
//     y[i,:] = w * (alpha * sum_j P[i,j] x[j,:] + v[i,:]) + (1 - w) * prev[i,:]
// over B right-hand sides at once.  w == 1 is the plain Neumann/power sweep
// z <- alpha P z + v; w != 1 is one Chebyshev semi-iteration step on the same fixed point.
// The L1 normalisation of the result (pi = z / sum z) needs only the column sums of the
// last iterate, which the last sweep's epilogue produces with warp-level reductions.
//
// Data layout: state matrices are [N, B] row-major fp32 (node-major, batch contiguous), so
// the gather of x[j,:] for a non-zero (i, j) is one contiguous 4B-byte segment (>= one
// 32-byte sector for B >= 8) and a group of B/4 lanes moves it with one 16-byte load per
// lane.  The matrix is CSR with (col, val) packed in 8 bytes so one load fetches both.
//
// Mapping: a group of LPR = B/4 lanes owns one row (a float4 each, sweep.cuh LaneF32);
// 256/LPR rows per CTA.  The row walk (4 gathers in flight per lane), the long-row segments
// and their fixed-order finalize sum, and the column sums are the shared skeleton of
// sweep.cuh; this file holds the sweep's epilogue and its kernels.
//
// Roofline (DESIGN.md): HBM-bound; algorithmic bytes per sweep =
//     nnz * 8 + (n_rows + 1) * 4 + 3 * n_rows * B * 4.
#include "sweep.cuh"

namespace hrag {

static int64_t g_launches = 0;
int64_t launches_since_reset() { return g_launches; }
void reset_launch_counter() { g_launches = 0; }
void count_launch(int n) { g_launches += n; }

namespace {

template <int LPR, bool CHEB>
__device__ __forceinline__ float4 row_epilogue(float4 acc, size_t o, const float4* __restrict__ v4,
                                               const float4* prev4, float4* y4, float alpha, float w) {
    const float4 vv = ld_stream_f4(v4 + o);
    float4 out;
    out.x = fmaf(alpha, acc.x, vv.x);
    out.y = fmaf(alpha, acc.y, vv.y);
    out.z = fmaf(alpha, acc.z, vv.z);
    out.w = fmaf(alpha, acc.w, vv.w);
    if (CHEB) {
        const float4 p = prev4[o];
        const float w1 = 1.f - w;
        out.x = fmaf(w, out.x, w1 * p.x);
        out.y = fmaf(w, out.y, w1 * p.y);
        out.z = fmaf(w, out.z, w1 * p.z);
        out.w = fmaf(w, out.w, w1 * p.w);
    }
    y4[o] = out;
    return out;
}

// ---- short rows: one group of LPR lanes per row ------------------------------------------
template <int LPR, bool CHEB, bool FINAL>
__global__ void __launch_bounds__(kThreads, 6)
k_sweep_rows(int n_rows, int row_base, int long_thresh, const int* __restrict__ row_ptr,
             const int2* __restrict__ cv, const float4* __restrict__ x4, const float4* __restrict__ v4,
             const float4* prev4, float4* y4, float alpha, float w, float* __restrict__ partials) {
    constexpr int GPB = kThreads / LPR;
    const int g = threadIdx.x / LPR, l = threadIdx.x % LPR;
    const int r = blockIdx.x * GPB + g;
    float4 out = f4_zero();
    if (r < n_rows) {
        const int s = __ldg(row_ptr + r), e = __ldg(row_ptr + r + 1);
        if (e - s <= long_thresh) {
            const float4 acc = row_walk<LaneF32, LPR, 1>(cv, nullptr, s, e, x4 + l);
            out = row_epilogue<LPR, CHEB>(acc, (size_t)(row_base + r) * LPR + l, v4, prev4, y4, alpha, w);
        }
    }
    if (FINAL) block_colsum<LaneF32, LPR>(out, partials + (size_t)blockIdx.x * (LPR * 4));
}

// ---- long rows: one warp per segment, then one group per row sums its segments -------------
template <int LPR>
__global__ void __launch_bounds__(kThreads)
k_sweep_long_segments(int n_seg, const int4* __restrict__ segs, const int2* __restrict__ cv,
                      const float4* __restrict__ x4, float4* __restrict__ seg_partial4) {
    segment_partial<LaneF32, LPR>(n_seg, segs, cv, nullptr, x4, seg_partial4);
}

template <int LPR, bool CHEB, bool FINAL>
__global__ void __launch_bounds__(kThreads)
k_sweep_long_finalize(int n_long, int row_base, const int* __restrict__ long_rows,
                      const int* __restrict__ long_seg_ptr, const float4* __restrict__ seg_partial4,
                      const float4* __restrict__ v4, const float4* prev4, float4* y4, float alpha, float w,
                      float* __restrict__ partials) {
    constexpr int GPB = kThreads / LPR;
    const int g = threadIdx.x / LPR, l = threadIdx.x % LPR;
    const int k = blockIdx.x * GPB + g;
    float4 out = f4_zero();
    if (k < n_long) {
        const int r = __ldg(long_rows + k);
        const float4 acc = segment_sum<LaneF32, LPR>(long_seg_ptr, k, seg_partial4 + l);
        out = row_epilogue<LPR, CHEB>(acc, (size_t)(row_base + r) * LPR + l, v4, prev4, y4, alpha, w);
    }
    if (FINAL) block_colsum<LaneF32, LPR>(out, partials + (size_t)blockIdx.x * (LPR * 4));
}

template <int LPR>
int launch_sweep(const PprGraph& g, const float* x, const float* v, const float* prev, float* y, float alpha,
                 float w, float* partials, int* n_partials, cudaStream_t st) {
    const SweepGrid grid(g, kThreads / LPR);
    const float4* x4 = reinterpret_cast<const float4*>(x);
    const float4* v4 = reinterpret_cast<const float4*>(v);
    const float4* p4 = reinterpret_cast<const float4*>(prev);
    float4* y4 = reinterpret_cast<float4*>(y);
    float4* segp = reinterpret_cast<float4*>(g.seg_partial);
    if (g.n_long) {
        k_sweep_long_segments<LPR><<<grid.nb_seg, kThreads, 0, st>>>(g.n_seg, g.segs, g.cv, x4, segp);
        count_launch();
    }
    float* part_long = partials ? partials + (size_t)grid.nb_rows * LPR * 4 : nullptr;
    with_bools([&](auto cheb, auto fin) {
        if (grid.nb_rows) {
            k_sweep_rows<LPR, cheb, fin><<<grid.nb_rows, kThreads, 0, st>>>(
                g.n_rows, g.row_lo, g.long_thresh, g.row_ptr, g.cv, x4, v4, p4, y4, alpha, w, partials);
            count_launch();
        }
        if (grid.nb_long) {
            k_sweep_long_finalize<LPR, cheb, fin><<<grid.nb_long, kThreads, 0, st>>>(
                g.n_long, g.row_lo, g.long_rows, g.long_seg_ptr, segp, v4, p4, y4, alpha, w, part_long);
            count_launch();
        }
    }, prev != nullptr, partials != nullptr);
    if (n_partials) *n_partials = grid.nb_rows + grid.nb_long;
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

int ppr_sweep_partial_rows(const PprGraph& g, int B) { return sweep_partial_rows(g, kThreads / (B / 4)); }

int ppr_sweep(const PprGraph& g, int B, const float* x, const float* v, const float* prev, float* y,
              float alpha, float w, float* colsum_partials, int* n_partials, cudaStream_t stream) {
    HRAG_CHECK(g.row_ptr && g.cv, "ppr_sweep: graph not loaded");
    HRAG_CHECK(B <= g.max_batch, "ppr_sweep: batch wider than the graph was prepared for");
    switch (B) {
        case 4:  return launch_sweep<1>(g, x, v, prev, y, alpha, w, colsum_partials, n_partials, stream);
        case 8:  return launch_sweep<2>(g, x, v, prev, y, alpha, w, colsum_partials, n_partials, stream);
        case 16: return launch_sweep<4>(g, x, v, prev, y, alpha, w, colsum_partials, n_partials, stream);
        case 32: return launch_sweep<8>(g, x, v, prev, y, alpha, w, colsum_partials, n_partials, stream);
        case 64: return launch_sweep<16>(g, x, v, prev, y, alpha, w, colsum_partials, n_partials, stream);
        default: break;
    }
    set_error("ppr_sweep: batch width must be one of 4, 8, 16, 32, 64");
    return 2;
}

int colsum_reduce(const float* partials, int n_partials, int B, double* sums, cudaStream_t stream) {
    k_colsum_reduce<float><<<B, 256, 0, stream>>>(partials, n_partials, B, sums);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace hrag
