// CSR sweep skeleton shared by the PPR kernels: K1 (fp32 state, ppr_spmm.cu), K1m (fp16 state, ppr_mixed.cu) and
// K1d (fp64 state, ppr_f64.cu).
//
// A group of LPR lanes owns one row of the [N, B] node-major state and each lane one fixed slice of its columns.  The
// precisions differ only in what a lane holds (a float4, 8 halves widened to fp32, a double2) and in the coefficient of
// a non-zero (the fp32 value, or hi + lo for the fp64 operator); a lane policy below states exactly that, and the walk,
// the long-row segments, their fixed-order sum and the CTA column sums are written once over it.  (K1m's short-row
// kernels k_sweep_h / k_sweep_h_push keep their own walk and column sums, ppr_mixed.cu.)
//
// Rows longer than long_thresh are cut into segments, one warp each (its groups stride through the segment), summed in
// a fixed order by a finalize kernel.  Every sum has a fixed order -- per lane in non-zero order, lanes by butterfly,
// warps by index, segments by index -- so a sweep gives the same bytes every time; no atomics.
//
// One launch sequence for every precision, all on one stream: the segment kernel, the short-row kernel, the finalize
// kernel, whose column-sum partials follow the short-row kernel's at row nb_rows.  The segment partials of all three
// live in PprGraph::seg_partial (64 floats = 256 B per segment; fp16 and fp64 use 128 B of it).
#pragma once
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace hrag {

namespace {

constexpr int kThreads = 256;

// ---- lane policies: one lane's slice of a row ----------------------------------------------------
// T: scalar of the accumulator and the column sums; X: the lane's slice of a gathered row; Acc: its fp32/fp64 sum.

// fp32 state (K1): 4 columns per lane
struct LaneF32 {
    using T = float; using X = float4; using Acc = float4;
    static __device__ __forceinline__ Acc zero() { return f4_zero(); }
    static __device__ __forceinline__ T coef(int2 c, const float*, int) { return __int_as_float(c.y); }
    static __device__ __forceinline__ void fma(Acc& a, T k, const X& x) { f4_fma(a, k, x); }
    static __device__ __forceinline__ void add(Acc& a, const Acc& b) { f4_add(a, b); }
    static __device__ __forceinline__ void shfl_xor_add(Acc& a, int off) {
        a.x += __shfl_xor_sync(0xffffffffu, a.x, off);
        a.y += __shfl_xor_sync(0xffffffffu, a.y, off);
        a.z += __shfl_xor_sync(0xffffffffu, a.z, off);
        a.w += __shfl_xor_sync(0xffffffffu, a.w, off);
    }
};

// fp16 state (K1m): 8 columns per lane, widened to fp32
__device__ __forceinline__ void h8_to_f(const uint4& u, float (&f)[8]) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 a = __half22float2(h[j]);
        f[2 * j] = a.x;
        f[2 * j + 1] = a.y;
    }
}
__device__ __forceinline__ void fma8(float (&acc)[8], float a, const uint4& u) {
    float f[8];
    h8_to_f(u, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = fmaf(a, f[j], acc[j]);
}
struct F8 { float v[8]; };
struct LaneF16 {
    using T = float; using X = uint4; using Acc = F8;
    static __device__ __forceinline__ Acc zero() {
        Acc a;
#pragma unroll
        for (int j = 0; j < 8; ++j) a.v[j] = 0.f;
        return a;
    }
    static __device__ __forceinline__ T coef(int2 c, const float*, int) { return __int_as_float(c.y); }
    static __device__ __forceinline__ void fma(Acc& a, T k, const X& x) { fma8(a.v, k, x); }
    static __device__ __forceinline__ void add(Acc& a, const Acc& b) {
#pragma unroll
        for (int j = 0; j < 8; ++j) a.v[j] += b.v[j];
    }
    static __device__ __forceinline__ void shfl_xor_add(Acc& a, int off) {
#pragma unroll
        for (int j = 0; j < 8; ++j) a.v[j] += __shfl_xor_sync(0xffffffffu, a.v[j], off);
    }
};

// fp64 state (K1d): 2 columns per lane; the coefficient is hi (cv) + lo (val_lo), P64 to ~2^-48 relative
struct LaneF64 {
    using T = double; using X = double2; using Acc = double2;
    static __device__ __forceinline__ Acc zero() { return make_double2(0.0, 0.0); }
    static __device__ __forceinline__ T coef(int2 c, const float* lo, int i) {
        return (double)__int_as_float(c.y) + (double)__ldg(lo + i);
    }
    static __device__ __forceinline__ void fma(Acc& a, T k, const X& x) {
        a.x = ::fma(k, x.x, a.x);
        a.y = ::fma(k, x.y, a.y);
    }
    static __device__ __forceinline__ void add(Acc& a, const Acc& b) { a.x += b.x; a.y += b.y; }
    static __device__ __forceinline__ void shfl_xor_add(Acc& a, int off) {
        a.x += __shfl_xor_sync(0xffffffffu, a.x, off);
        a.y += __shfl_xor_sync(0xffffffffu, a.y, off);
    }
};

// ---- device skeleton ------------------------------------------------------------------------------
// Non-zeros i, i + S, i + 2S, ... below e of one row, four at a time so four independent gathers are in flight per
// lane (the sweep is bound by gather latency x bandwidth, not by FMA issue); each lane sums in non-zero order.
// S = 1 walks a whole short row; S = 32 / LPR is one group's share of a long-row segment.  x is already + lane.
// (The bound is written `+ 1 <=`: nvcc unrolls the `i + 3 * S < e` form 4x more at S = 1, a larger k_sweep_rows.)
// RS: the state's row stride in X units (LPR unless two states are interleaved row by row).  x is the state itself, or
// any source with a gather_row overload (ppr_mixed.cu reads a compact first iterate through its slot map).
template <int RS, class X>
__device__ __forceinline__ X gather_row(const X* __restrict__ x, int col) { return __ldg(x + (size_t)col * RS); }

template <class L, int LPR, int S, int RS = LPR, class Src = const typename L::X*>
__device__ __forceinline__ typename L::Acc row_walk(const int2* __restrict__ cv, const float* __restrict__ lo, int i,
                                                    int e, const Src x) {
    typename L::Acc acc = L::zero();
    for (; i + 3 * S + 1 <= e; i += 4 * S) {
        const int2 c0 = __ldg(cv + i), c1 = __ldg(cv + i + S), c2 = __ldg(cv + i + 2 * S), c3 = __ldg(cv + i + 3 * S);
        const auto a0 = gather_row<RS>(x, c0.x);
        const auto a1 = gather_row<RS>(x, c1.x);
        const auto a2 = gather_row<RS>(x, c2.x);
        const auto a3 = gather_row<RS>(x, c3.x);
        L::fma(acc, L::coef(c0, lo, i), a0);
        L::fma(acc, L::coef(c1, lo, i + S), a1);
        L::fma(acc, L::coef(c2, lo, i + 2 * S), a2);
        L::fma(acc, L::coef(c3, lo, i + 3 * S), a3);
    }
    for (; i < e; i += S) {
        const int2 c = __ldg(cv + i);
        L::fma(acc, L::coef(c, lo, i), gather_row<RS>(x, c.x));
    }
    return acc;
}

// Body of the segment kernels: warp w of the grid sums segment w of the long rows; the groups of the warp are then
// added by butterfly and the warp's LPR lane slices go to seg_partial[w].
template <class L, int LPR, int RS = LPR, class Src = const typename L::X*>
__device__ __forceinline__ void segment_partial(int n_seg, const int4* __restrict__ segs, const int2* __restrict__ cv,
                                                const float* __restrict__ lo, const Src x,
                                                typename L::Acc* __restrict__ seg_partial) {
    const int warp = (blockIdx.x * kThreads + threadIdx.x) >> 5;
    if (warp >= n_seg) return;
    const int lane = threadIdx.x & 31;
    const int4 sg = __ldg(segs + warp);
    typename L::Acc acc = row_walk<L, LPR, 32 / LPR, RS, Src>(cv, lo, sg.y + lane / LPR, sg.z, x + lane % LPR);
#pragma unroll
    for (int off = LPR; off < 32; off <<= 1) L::shfl_xor_add(acc, off);
    if (lane < LPR) seg_partial[(size_t)warp * LPR + lane] = acc;
}

// Long row k's sum: its segment partials added in segment order.  seg_partial is already + lane.
template <class L, int LPR>
__device__ __forceinline__ typename L::Acc segment_sum(const int* __restrict__ long_seg_ptr, int k,
                                                       const typename L::Acc* __restrict__ seg_partial) {
    typename L::Acc acc = L::zero();
    for (int s = __ldg(long_seg_ptr + k); s < __ldg(long_seg_ptr + k + 1); ++s) L::add(acc, seg_partial[(size_t)s * LPR]);
    return acc;
}

// Column sums over the whole CTA of each thread's N slices v[n] -> rows[n][0, B): lanes by butterfly, then warps in
// index order, one barrier for all N.  Its shared scratch is reused by the next call, so two calls in a row need a
// __syncthreads() between them.
template <class L, int LPR, int N>
__device__ __forceinline__ void block_colsum(typename L::Acc (&v)[N], typename L::T* const (&rows)[N]) {
    static_assert(N == 1 || N == 2, "one or two slices per thread");
    using T = typename L::T;
    constexpr int W = sizeof(v[0]) / sizeof(T), B = LPR * W;   // columns per lane, per row
    __shared__ T s_sum[N][kThreads / 32][B];
#pragma unroll
    for (int off = LPR; off < 32; off <<= 1)
#pragma unroll
        for (int n = 0; n < N; ++n) L::shfl_xor_add(v[n], off);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane < LPR) {
#pragma unroll
        for (int n = 0; n < N; ++n)
#pragma unroll
            for (int j = 0; j < W; ++j) s_sum[n][warp][lane * W + j] = reinterpret_cast<const T*>(&v[n])[j];
    }
    __syncthreads();
    if (threadIdx.x < N * B) {                       // one thread per column of each slice
        const unsigned n = N == 1 ? 0u : threadIdx.x / B, c = N == 1 ? threadIdx.x : threadIdx.x % B;
        T s = 0;
#pragma unroll
        for (int wi = 0; wi < kThreads / 32; ++wi) s += s_sum[n][wi][c];
        (n == 0 ? rows[0] : rows[N - 1])[c] = s;     // constant indices: rows stays in registers
    }
}
// one slice per thread
template <class L, int LPR>
__device__ __forceinline__ void block_colsum(typename L::Acc v, typename L::T* partial_row) {
    typename L::Acc vs[1] = {v};
    typename L::T* const rows[1] = {partial_row};
    block_colsum<L, LPR, 1>(vs, rows);
}

// sums[b] = sum over the rows of partials[r, b]; one CTA per column, fp64 accumulation (an fp32 running sum over 10^4
// partials costs ~1e-6), each thread striding over the rows and then a fixed-order tree
template <class T>
__global__ void __launch_bounds__(256)
k_colsum_reduce(const T* __restrict__ partials, int n_partials, int B, double* __restrict__ sums) {
    __shared__ double s[256];
    const int b = blockIdx.x;
    double acc = 0.0;
    for (int r = threadIdx.x; r < n_partials; r += 256) acc += (double)partials[(size_t)r * B + b];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off) s[threadIdx.x] += s[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) sums[b] = s[0];
}

// ---- host side -------------------------------------------------------------------------------------
// CTAs of a sweep's three launches: one warp per segment; rows_per_cta rows per CTA for the short rows and for the
// long-row finalize (0 when the graph has no long rows).
struct SweepGrid {
    unsigned nb_seg;
    int nb_rows, nb_long;
    SweepGrid(const PprGraph& g, int rows_per_cta)
        : nb_seg((unsigned)ceil_div((int64_t)g.n_seg * 32, kThreads)),
          nb_rows((int)ceil_div(g.n_rows, rows_per_cta)),
          nb_long(g.n_long ? (int)ceil_div(g.n_long, rows_per_cta) : 0) {}
};

// rows of column-sum partials one sweep writes
inline int sweep_partial_rows(const PprGraph& g, int rows_per_cta) {
    const SweepGrid s(g, rows_per_cta);
    return s.nb_rows + s.nb_long;
}

// f(std::bool_constant<b0>{}, std::bool_constant<b1>{}, ...) for the runtime flags b0, b1, ...: turns the flags of a
// launch into template arguments, one instantiation per combination that f's body does not discard
template <class F>
void with_bools(F&& f) { f(); }
template <class F, class... Bs>
void with_bools(F&& f, bool b, Bs... bs) {
    if (b) with_bools([&](auto... c) { f(std::true_type{}, c...); }, bs...);
    else with_bools([&](auto... c) { f(std::false_type{}, c...); }, bs...);
}

}  // namespace

}  // namespace hrag
