// K2 (exact-fp32 variant) -- batched query x embedding similarity on the fp32 FMA pipe.
//
// Replaces the per-query sgemv of get_fact_scores / dense_passage_retrieval (reference
// HippoRAG.py:1459, :1496: np.dot(E, q)) with one batched contraction S = Q E^T.  This is the
// HRAG_SIM_FP32 mode: every product is an exact fp32 FMA, so it is the in-library reference
// the wgmma split-bf16 kernel (sim_tc.cu) is checked against, and the mode of choice for
// tiny corpora.  Register-tiled 64x64x16, 4x4 outputs per thread, operands staged K-major in
// shared memory.
#include "common.cuh"
#include "kernels.h"

namespace hrag {

namespace {

constexpr int BM = 64, BN = 64, BK = 16, PAD = 4;

__global__ void __launch_bounds__(256)
k_sim_fp32(const float* __restrict__ Q, int Bq, const float* __restrict__ E, int64_t M, int dim,
           float* __restrict__ S, int64_t ldS) {
    __shared__ __align__(16) float As[BK][BM + PAD];   // queries, K-major
    __shared__ __align__(16) float Bs[BK][BN + PAD];   // embeddings, K-major
    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;
    const int64_t m0 = (int64_t)blockIdx.x * BN;
    const int b0 = blockIdx.y * BM;
    const int lrow = tid / 4, lk = (tid % 4) * 4;      // loader: one float4 of one row per thread
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < dim; k0 += BK) {
        float4 qa = f4_zero(), eb = f4_zero();
        if (b0 + lrow < Bq && k0 + lk < dim)
            qa = __ldg(reinterpret_cast<const float4*>(Q + (size_t)(b0 + lrow) * dim + k0 + lk));
        if (m0 + lrow < M && k0 + lk < dim)
            eb = __ldg(reinterpret_cast<const float4*>(E + (size_t)(m0 + lrow) * dim + k0 + lk));
        __syncthreads();
        As[lk + 0][lrow] = qa.x; As[lk + 1][lrow] = qa.y; As[lk + 2][lrow] = qa.z; As[lk + 3][lrow] = qa.w;
        Bs[lk + 0][lrow] = eb.x; Bs[lk + 1][lrow] = eb.y; Bs[lk + 2][lrow] = eb.z; Bs[lk + 3][lrow] = eb.w;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w};
            const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int b = b0 + ty * 4 + i;
        if (b >= Bq) continue;
        const int64_t m = m0 + tx * 4;
        float* dst = S + (size_t)b * ldS + m;
        if (m + 3 < M && (ldS % 4 == 0)) {
            *reinterpret_cast<float4*>(dst) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (m + j < M) dst[j] = acc[i][j];
        }
    }
}

}  // namespace

int sim_fp32(const float* Q, int Bq, const float* E, int64_t M, int dim, float* S, int64_t ldS,
             cudaStream_t stream) {
    HRAG_CHECK(dim % 4 == 0, "sim_fp32: embedding dim must be a multiple of 4");
    if (Bq == 0 || M == 0) return 0;
    dim3 grid((unsigned)ceil_div(M, BN), (unsigned)ceil_div(Bq, BM));
    k_sim_fp32<<<grid, 256, 0, stream>>>(Q, Bq, E, M, dim, S, ldS);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace hrag
