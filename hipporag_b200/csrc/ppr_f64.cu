// Residual sweep of the float64 PPR solver (hrag_ppr_f64, sm_90a).
//
// The fp64 solver is iterative refinement one level above the mixed solver (DESIGN.md section 2): K1's fp32
// sweeps solve the correction equation, and this file computes the residual of the accumulated fp64 iterate
// against the fp64 operator P = hi + lo (hi = the fp32 value in cv, lo = fp32(P64 - hi), ~2^-48 relative):
//     r[i,:] = v[i,:] - x[i,:] + alpha * sum_j (hi[i,j] + lo[i,j]) x[j,:]          (all in fp64)
// State is [N, B] row-major fp64; a group of LPR = B/2 lanes owns one row and each lane one double2 of it, so the
// gather of x[j,:] is 8B bytes (128 B at B = 16).  Four non-zeros are in flight per lane, as in K1.  The fused
// epilogue writes only fp32(r) -- the right-hand side of the next correction solve -- and per-CTA fp64 partials of
// sum |r| and of sum x (the normalisation of the final iterate).  Rows longer than long_thresh go through the
// segment / finalize pair of K1 with fp64 segment partials.  Deterministic: every sum runs in a fixed order, no
// atomics, so two calls give identical bytes.
//
// Bytes per sweep (algorithmic): nnz * (8 + 4) + (n_rows + 1) * 4 + n_rows * B * (8 + 8 + 4)  (cv, lo, row_ptr;
// x and v read once, fp32 r written); the gathers add nnz * 8B bytes of L2 -> SM traffic.
#include "common.cuh"
#include "kernels.h"

namespace hrag {

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ void d2_fma(double2& acc, double a, const double2& x) {
    acc.x = fma(a, x.x, acc.x);
    acc.y = fma(a, x.y, acc.y);
}
__device__ __forceinline__ double p64(int2 c, float lo) { return (double)__int_as_float(c.y) + (double)lo; }

template <int LPR>
__device__ __forceinline__ double2 group_row_dot_f64(const int2* __restrict__ cv, const float* __restrict__ lo, int s,
                                                     int e, const double2* __restrict__ x2 /* already + lane */) {
    double2 acc = make_double2(0.0, 0.0);
    int i = s;
    for (; i + 4 <= e; i += 4) {
        const int2 c0 = __ldg(cv + i), c1 = __ldg(cv + i + 1), c2 = __ldg(cv + i + 2), c3 = __ldg(cv + i + 3);
        const float l0 = __ldg(lo + i), l1 = __ldg(lo + i + 1), l2 = __ldg(lo + i + 2), l3 = __ldg(lo + i + 3);
        const double2 a0 = __ldg(x2 + (size_t)c0.x * LPR);
        const double2 a1 = __ldg(x2 + (size_t)c1.x * LPR);
        const double2 a2 = __ldg(x2 + (size_t)c2.x * LPR);
        const double2 a3 = __ldg(x2 + (size_t)c3.x * LPR);
        d2_fma(acc, p64(c0, l0), a0);
        d2_fma(acc, p64(c1, l1), a1);
        d2_fma(acc, p64(c2, l2), a2);
        d2_fma(acc, p64(c3, l3), a3);
    }
    for (; i < e; ++i) {
        const int2 c = __ldg(cv + i);
        d2_fma(acc, p64(c, __ldg(lo + i)), __ldg(x2 + (size_t)c.x * LPR));
    }
    return acc;
}

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

// Column sums of |r| and x over the whole CTA -> part_r / part_x [blockIdx, B] (fixed order: lanes, then warps).
template <int LPR>
__device__ __forceinline__ void block_colsum2_f64(double2 a, double2 b, double* __restrict__ part_r_row,
                                                  double* __restrict__ part_x_row) {
    constexpr int B = LPR * 2;
    __shared__ double s_r[kThreads / 32][B], s_x[kThreads / 32][B];
#pragma unroll
    for (int off = LPR; off < 32; off <<= 1) {
        a.x += __shfl_xor_sync(0xffffffffu, a.x, off);
        a.y += __shfl_xor_sync(0xffffffffu, a.y, off);
        b.x += __shfl_xor_sync(0xffffffffu, b.x, off);
        b.y += __shfl_xor_sync(0xffffffffu, b.y, off);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane < LPR) {
        s_r[warp][lane * 2] = a.x;
        s_r[warp][lane * 2 + 1] = a.y;
        s_x[warp][lane * 2] = b.x;
        s_x[warp][lane * 2 + 1] = b.y;
    }
    __syncthreads();
    if (threadIdx.x < B) {
        double sr = 0.0, sx = 0.0;
#pragma unroll
        for (int wi = 0; wi < kThreads / 32; ++wi) {
            sr += s_r[wi][threadIdx.x];
            sx += s_x[wi][threadIdx.x];
        }
        part_r_row[threadIdx.x] = sr;
        part_x_row[threadIdx.x] = sx;
    }
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
            const double2 acc = group_row_dot_f64<LPR>(cv, lo, s, e, x2 + l);
            resid_epilogue(acc, (size_t)r * LPR + l, v2, x2, r32, alpha, abs_r, xv);
        }
    }
    block_colsum2_f64<LPR>(abs_r, xv, part_r + (size_t)blockIdx.x * (LPR * 2), part_x + (size_t)blockIdx.x * (LPR * 2));
}

// ---- long rows: one warp per segment, groups stride through it ----------------------------
template <int LPR>
__global__ void __launch_bounds__(kThreads)
k_resid_long_segments_f64(int n_seg, const int4* __restrict__ segs, const int2* __restrict__ cv,
                          const float* __restrict__ lo, const double2* __restrict__ x2,
                          double2* __restrict__ seg_partial2) {
    constexpr int G = 32 / LPR;
    const int warp = (blockIdx.x * kThreads + threadIdx.x) >> 5;
    if (warp >= n_seg) return;
    const int lane = threadIdx.x & 31;
    const int g = lane / LPR, l = lane % LPR;
    const int4 sg = __ldg(segs + warp);
    double2 acc = make_double2(0.0, 0.0);
    int i = sg.y + g;
    for (; i + 3 * G < sg.z; i += 4 * G) {
        const int2 c0 = __ldg(cv + i), c1 = __ldg(cv + i + G), c2 = __ldg(cv + i + 2 * G), c3 = __ldg(cv + i + 3 * G);
        const float l0 = __ldg(lo + i), l1 = __ldg(lo + i + G), l2 = __ldg(lo + i + 2 * G), l3 = __ldg(lo + i + 3 * G);
        const double2 a0 = __ldg(x2 + (size_t)c0.x * LPR + l);
        const double2 a1 = __ldg(x2 + (size_t)c1.x * LPR + l);
        const double2 a2 = __ldg(x2 + (size_t)c2.x * LPR + l);
        const double2 a3 = __ldg(x2 + (size_t)c3.x * LPR + l);
        d2_fma(acc, p64(c0, l0), a0);
        d2_fma(acc, p64(c1, l1), a1);
        d2_fma(acc, p64(c2, l2), a2);
        d2_fma(acc, p64(c3, l3), a3);
    }
    for (; i < sg.z; i += G) {
        const int2 c = __ldg(cv + i);
        d2_fma(acc, p64(c, __ldg(lo + i)), __ldg(x2 + (size_t)c.x * LPR + l));
    }
#pragma unroll
    for (int off = LPR; off < 32; off <<= 1) {
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, off);
        acc.y += __shfl_xor_sync(0xffffffffu, acc.y, off);
    }
    if (lane < LPR) seg_partial2[(size_t)warp * LPR + lane] = acc;
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
        double2 acc = make_double2(0.0, 0.0);
        for (int s = __ldg(long_seg_ptr + k); s < __ldg(long_seg_ptr + k + 1); ++s) {
            const double2 p = seg_partial2[(size_t)s * LPR + l];
            acc.x += p.x;
            acc.y += p.y;
        }
        resid_epilogue(acc, (size_t)r * LPR + l, v2, x2, r32, alpha, abs_r, xv);
    }
    block_colsum2_f64<LPR>(abs_r, xv, part_r + (size_t)blockIdx.x * (LPR * 2), part_x + (size_t)blockIdx.x * (LPR * 2));
}

template <int LPR>
int launch_resid(const PprGraph& g, const double* x, const double* v, float* r32, double alpha, double* part_r,
                 double* part_x, int* n_partials, cudaStream_t st) {
    constexpr int GPB = kThreads / LPR;
    const int nb_rows = (int)ceil_div(g.n_rows, GPB);
    const int nb_long = g.n_long ? (int)ceil_div(g.n_long, GPB) : 0;
    const double2* x2 = reinterpret_cast<const double2*>(x);
    const double2* v2 = reinterpret_cast<const double2*>(v);
    float2* r2 = reinterpret_cast<float2*>(r32);
    double2* segp = reinterpret_cast<double2*>(g.seg_partial64);
    if (g.n_long) {
        k_resid_long_segments_f64<LPR><<<(unsigned)ceil_div((int64_t)g.n_seg * 32, kThreads), kThreads, 0, st>>>(
            g.n_seg, g.segs, g.cv, g.val_lo, x2, segp);
        count_launch();
    }
    if (nb_rows) {
        k_resid_f64<LPR><<<nb_rows, kThreads, 0, st>>>(g.n_rows, g.long_thresh, g.row_ptr, g.cv, g.val_lo, x2, v2, r2,
                                                       alpha, part_r, part_x);
        count_launch();
    }
    if (nb_long) {
        const size_t off = (size_t)nb_rows * LPR * 2;
        k_resid_long_finalize_f64<LPR><<<nb_long, kThreads, 0, st>>>(g.n_long, g.long_rows, g.long_seg_ptr, segp, x2,
                                                                     v2, r2, alpha, part_r + off, part_x + off);
        count_launch();
    }
    *n_partials = nb_rows + nb_long;
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
k_colsum_reduce_f64(const double* __restrict__ partials, int n_partials, int B, double* __restrict__ sums) {
    // one CTA per column, same fixed-order tree as k_colsum_reduce
    __shared__ double s[256];
    const int b = blockIdx.x;
    double acc = 0.0;
    for (int r = threadIdx.x; r < n_partials; r += 256) acc += partials[(size_t)r * B + b];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off) s[threadIdx.x] += s[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) sums[b] = s[0];
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

int resid_f64_partial_rows(const PprGraph& g, int B) {
    const int GPB = kThreads / (B / 2);
    return (int)ceil_div(g.n_rows, GPB) + (g.n_long ? (int)ceil_div(g.n_long, GPB) : 0);
}

int resid_sweep_f64(const PprGraph& g, int B, const double* x, const double* v, float* r32, double alpha,
                    double* part_r, double* part_x, int* n_partials, cudaStream_t stream) {
    HRAG_CHECK(g.row_ptr && g.cv && g.val_lo, "resid_sweep_f64: graph not loaded with an fp64 operator");
    HRAG_CHECK(g.n_long == 0 || g.seg_partial64, "resid_sweep_f64: fp64 segment partials missing");
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
    k_colsum_reduce_f64<<<B, 256, 0, stream>>>(partials, n_partials, B, sums);
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
