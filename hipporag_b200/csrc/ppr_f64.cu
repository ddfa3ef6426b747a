// Residual sweep of the float64 PPR solver (hrag_ppr_f64, sm_90a).
//
// The fp64 solver is iterative refinement one level above the mixed solver (DESIGN.md section 2): K1's fp32
// sweeps solve the correction equation, and this file computes the residual of the accumulated fp64 iterate
// against the fp64 operator P = hi + lo (hi = the fp32 value in cv, lo = fp32(P64 - hi), ~2^-48 relative):
//     r[i,:] = v[i,:] - x[i,:] + alpha * sum_j (hi[i,j] + lo[i,j]) x[j,:]          (all in fp64)
// State is [N, B] row-major fp64; a group of LPR = B/2 lanes owns one row and each lane one double2 of it (sweep.cuh
// LaneF64), so the gather of x[j,:] is 8B bytes (128 B at B = 16).  The row walk, the long-row segments and their
// finalize sum, and the column sums are K1's, from sweep.cuh; the segment partials reuse K1's seg_partial buffer
// (every sweep of a handle runs on its one stream).  The fused epilogue writes only fp32(r) -- the right-hand side of
// the next correction solve -- and per-CTA fp64 partials of sum |r| and of sum x (the normalisation of the final
// iterate).  Deterministic: every sum runs in a fixed order, no atomics, so two calls give identical bytes.
//
// Bytes per sweep (algorithmic): nnz * (8 + 4) + (n_rows + 1) * 4 + n_rows * B * (8 + 8 + 4)  (cv, lo, row_ptr;
// x and v read once, fp32 r written); the gathers add nnz * 8B bytes of L2 -> SM traffic.
#include "sweep.cuh"

namespace hrag {

namespace {

// r = v - x + alpha * acc on one double2 of a row; stores fp32(r), returns |r| and x for the column sums
__device__ __forceinline__ void resid_epilogue(double2 acc, size_t o, const double2* __restrict__ v2,
                                               const double2* __restrict__ x2, float2* __restrict__ r32, double alpha,
                                               double2& abs_r, double2& xv) {
    const double2 v = v2[o], x = x2[o];
    const double rx = fma(alpha, acc.x, v.x - x.x), ry = fma(alpha, acc.y, v.y - x.y);
    r32[o] = make_float2(__double2float_rn(rx), __double2float_rn(ry));
    abs_r = make_double2(fabs(rx), fabs(ry));
    xv = x;
}

// Column sums of |r| and x over the whole CTA -> part_r / part_x [blockIdx, B]
template <int LPR>
__device__ __forceinline__ void resid_colsums(double2 abs_r, double2 xv, double* __restrict__ part_r,
                                              double* __restrict__ part_x) {
    const size_t o = (size_t)blockIdx.x * (LPR * 2);
    double2 v[2] = {abs_r, xv};
    double* const rows[2] = {part_r + o, part_x + o};
    block_colsum<LaneF64, LPR>(v, rows);
}

// ---- short rows: one group of LPR lanes per row ------------------------------------------
template <int LPR>
__global__ void __launch_bounds__(kThreads)
k_resid_f64(int n_rows, int long_thresh, const int* __restrict__ row_ptr, const int2* __restrict__ cv,
            const float* __restrict__ lo, const double2* __restrict__ x2, const double2* __restrict__ v2,
            float2* __restrict__ r32, double alpha, double* __restrict__ part_r, double* __restrict__ part_x) {
    constexpr int GPB = kThreads / LPR;
    const int g = threadIdx.x / LPR, l = threadIdx.x % LPR;
    const int r = blockIdx.x * GPB + g;
    double2 abs_r = make_double2(0.0, 0.0), xv = make_double2(0.0, 0.0);
    if (r < n_rows) {
        const int s = __ldg(row_ptr + r), e = __ldg(row_ptr + r + 1);
        if (e - s <= long_thresh) {
            const double2 acc = row_walk<LaneF64, LPR, 1>(cv, lo, s, e, x2 + l);
            resid_epilogue(acc, (size_t)r * LPR + l, v2, x2, r32, alpha, abs_r, xv);
        }
    }
    resid_colsums<LPR>(abs_r, xv, part_r, part_x);
}

// ---- long rows: one warp per segment, then one group per row sums its segments -------------
template <int LPR>
__global__ void __launch_bounds__(kThreads)
k_resid_long_segments_f64(int n_seg, const int4* __restrict__ segs, const int2* __restrict__ cv,
                          const float* __restrict__ lo, const double2* __restrict__ x2,
                          double2* __restrict__ seg_partial2) {
    segment_partial<LaneF64, LPR>(n_seg, segs, cv, lo, x2, seg_partial2);
}

template <int LPR>
__global__ void __launch_bounds__(kThreads)
k_resid_long_finalize_f64(int n_long, const int* __restrict__ long_rows, const int* __restrict__ long_seg_ptr,
                          const double2* __restrict__ seg_partial2, const double2* __restrict__ x2,
                          const double2* __restrict__ v2, float2* __restrict__ r32, double alpha,
                          double* __restrict__ part_r, double* __restrict__ part_x) {
    constexpr int GPB = kThreads / LPR;
    const int g = threadIdx.x / LPR, l = threadIdx.x % LPR;
    const int k = blockIdx.x * GPB + g;
    double2 abs_r = make_double2(0.0, 0.0), xv = make_double2(0.0, 0.0);
    if (k < n_long) {
        const int r = __ldg(long_rows + k);
        const double2 acc = segment_sum<LaneF64, LPR>(long_seg_ptr, k, seg_partial2 + l);
        resid_epilogue(acc, (size_t)r * LPR + l, v2, x2, r32, alpha, abs_r, xv);
    }
    resid_colsums<LPR>(abs_r, xv, part_r, part_x);
}

template <int LPR>
int launch_resid(const PprGraph& g, const double* x, const double* v, float* r32, double alpha, double* part_r,
                 double* part_x, int* n_partials, cudaStream_t st) {
    const SweepGrid grid(g, kThreads / LPR);
    const double2* x2 = reinterpret_cast<const double2*>(x);
    const double2* v2 = reinterpret_cast<const double2*>(v);
    float2* r2 = reinterpret_cast<float2*>(r32);
    double2* segp = reinterpret_cast<double2*>(g.seg_partial);
    if (g.n_long) {
        k_resid_long_segments_f64<LPR><<<grid.nb_seg, kThreads, 0, st>>>(g.n_seg, g.segs, g.cv, g.val_lo, x2, segp);
        count_launch();
    }
    if (grid.nb_rows) {
        k_resid_f64<LPR><<<grid.nb_rows, kThreads, 0, st>>>(g.n_rows, g.long_thresh, g.row_ptr, g.cv, g.val_lo, x2, v2,
                                                            r2, alpha, part_r, part_x);
        count_launch();
    }
    if (grid.nb_long) {
        const size_t off = (size_t)grid.nb_rows * LPR * 2;
        k_resid_long_finalize_f64<LPR><<<grid.nb_long, kThreads, 0, st>>>(g.n_long, g.long_rows, g.long_seg_ptr, segp,
                                                                          x2, v2, r2, alpha, part_r + off,
                                                                          part_x + off);
        count_launch();
    }
    *n_partials = grid.nb_rows + grid.nb_long;
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

// V[n, b] = sanitised R[b, n] (NaN / negative -> 0, run_ppr HippoRAG.py:1735), V32 = fp32(V), X = 0, and per-CTA
// column sums of V -> part_v [blockIdx, B].  256 % B == 0, so every thread of a CTA stays on column tid % B.
__global__ void __launch_bounds__(256)
k_reset_to_state_f64(const double* __restrict__ R, int nb, int N, int B, double* __restrict__ V,
                     float* __restrict__ V32, double* __restrict__ X, double* __restrict__ part_v) {
    __shared__ double s[256];
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t n = t / B;
    const int b = (int)(t % B);
    double r = 0.0;
    if (n < N) {
        if (b < nb) {
            r = R[(size_t)b * N + n];
            if (!(r >= 0.0)) r = 0.0;
        }
        V[t] = r;
        V32[t] = __double2float_rn(r);
        X[t] = 0.0;
    }
    s[threadIdx.x] = r;
    __syncthreads();
    if (threadIdx.x < B) {
        double acc = 0.0;
        for (int k = threadIdx.x; k < 256; k += B) acc += s[k];
        part_v[(size_t)blockIdx.x * B + threadIdx.x] = acc;
    }
}

// X += D on the columns whose bit is set in `active` (a converged column keeps its iterate, so its result does not
// depend on the other columns of the sub-batch)
__global__ void __launch_bounds__(256)
k_add_correction_f64(double* __restrict__ X, const float* __restrict__ D, int64_t n, int B, unsigned active) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n && ((active >> (int)(i % B)) & 1u)) X[i] += (double)D[i];
}

__global__ void __launch_bounds__(256)
k_state_to_scores_f64(const double* __restrict__ X, int nb, int N, int B, const double* __restrict__ sums,
                      double* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t n = t / nb;
    const int b = (int)(t % nb);
    if (n >= N) return;
    out[(size_t)b * N + n] = X[(size_t)n * B + b] / sums[b];
}

}  // namespace

int resid_f64_partial_rows(const PprGraph& g, int B) { return sweep_partial_rows(g, kThreads / (B / 2)); }

int resid_sweep_f64(const PprGraph& g, int B, const double* x, const double* v, float* r32, double alpha,
                    double* part_r, double* part_x, int* n_partials, cudaStream_t stream) {
    HRAG_CHECK(g.row_ptr && g.cv && g.val_lo, "resid_sweep_f64: graph not loaded with an fp64 operator");
    // the fp64 segment partials (B doubles per segment) live in seg_partial (max_batch floats per segment)
    HRAG_CHECK((size_t)B * sizeof(double) <= (size_t)g.max_batch * sizeof(float),
               "resid_sweep_f64: segment partials too small for an fp64 batch this wide");
    switch (B) {
        case 4:  return launch_resid<2>(g, x, v, r32, alpha, part_r, part_x, n_partials, stream);
        case 8:  return launch_resid<4>(g, x, v, r32, alpha, part_r, part_x, n_partials, stream);
        case 16: return launch_resid<8>(g, x, v, r32, alpha, part_r, part_x, n_partials, stream);
        default: break;
    }
    set_error("resid_sweep_f64: batch width must be one of 4, 8, 16");
    return 2;
}

int reset_to_state_f64(const double* R, int nb, int N, int B, double* V, float* V32, double* X, double* part_v,
                       int* n_partials, cudaStream_t stream) {
    HRAG_CHECK(256 % B == 0, "reset_to_state_f64: B must divide 256");
    const int64_t blocks = ceil_div((int64_t)N * B, 256);
    k_reset_to_state_f64<<<(unsigned)blocks, 256, 0, stream>>>(R, nb, N, B, V, V32, X, part_v);
    count_launch();
    *n_partials = (int)blocks;
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int add_correction_f64(double* X, const float* D, int64_t n, int B, unsigned active, cudaStream_t stream) {
    k_add_correction_f64<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(X, D, n, B, active);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int colsum_reduce_f64(const double* partials, int n_partials, int B, double* sums, cudaStream_t stream) {
    k_colsum_reduce<double><<<B, 256, 0, stream>>>(partials, n_partials, B, sums);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int state_to_scores_f64(const double* X, int nb, int N, int B, const double* sums, double* out, cudaStream_t stream) {
    const int64_t total = (int64_t)N * nb;
    k_state_to_scores_f64<<<(unsigned)ceil_div(total, 256), 256, 0, stream>>>(X, nb, N, B, sums, out);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace hrag
