// K1t -- the fp16-state PPR sweep with the gathered state rows fetched by the TMA unit (sm_90a).
// (A variant of K1m; like it, one sweep of the iteration that stands in for igraph's personalized_pagerank call in
// HippoRAG.run_ppr, reference HippoRAG.py:1736-1743.)
//
// Same arithmetic as k_sweep_h (ppr_mixed.cu), different data path for the operand that bounds
// the sweep: the rows x[j, :] named by the non-zeros of a row block.  Producer warps read the
// block's (col, val) stream once (coalesced) and issue one bulk asynchronous copy
// (`cp.async.bulk.shared::cluster.global`) per non-zero: the TMA unit fetches the 64-byte state row
// into a shared-memory stage and signals an mbarrier (complete_tx); the values go to the same stage
// with plain shared stores.  Consumer groups (4 lanes per row, as in k_sweep_h) then take their
// row's operands from shared memory.  Loads in flight are bounded by the ring (3 stages x 1024
// rows x 64 B = 192 KB per SM), not by registers x resident warps.
//
// Row blocks: <= 64 rows and <= 1024 non-zeros, contiguous in the CSR (built at graph load);
// rows longer than long_thresh keep the segment path of ppr_mixed.cu and are skipped here.
// Selected with HRAG_MIXED_TMA=1; k_sweep_h stays the default.
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace hrag {

namespace {

constexpr int kLPR = 4;
constexpr int kBlkRows = 64;                  // rows per block = consumer groups per CTA
constexpr int kBlkNnz = 1024;                 // non-zeros per block (one stage)
constexpr int kStages = 3;
constexpr int kProdWarps = 4;
constexpr int kConsWarps = kBlkRows * kLPR / 32;                 // 8
constexpr int kTmaThreads = 32 * (kProdWarps + kConsWarps);      // 384
constexpr int kStageXBytes = kBlkNnz * 64;                       // 64 KB of gathered rows
constexpr int kStageBytes = kStageXBytes + kBlkNnz * 4;          // + the values
constexpr size_t kSmemBytes = (size_t)kStages * kStageBytes + 1024 + 128;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
// tx-count only (no arrival): the producer warp arrives after its shared stores
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(bar), "r"(parity) : "memory");
}
// one 64-byte state row global -> shared, completion counted on bar (complete_tx)
__device__ __forceinline__ void bulk_row64(uint32_t dst, const void* src, uint32_t bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], 64, [%2], %3;"
        ::"r"(dst), "l"(src), "r"(bar), "l"(policy) : "memory");
}

__device__ __forceinline__ void h8_to_f(const uint4& u, float (&f)[8]) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 a = __half22float2(h[j]);
        f[2 * j] = a.x;
        f[2 * j + 1] = a.y;
    }
}
__device__ __forceinline__ float sat_h(float x) { return fminf(fmaxf(x, -65504.f), 65504.f); }
__device__ __forceinline__ uint4 f_to_h8(const float (&f)[8]) {
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(sat_h(f[2 * j]), sat_h(f[2 * j + 1]));
    return u;
}

struct TmaSweepArgs {
    int n_blk;
    const uint4* xh;           // [rows, 32] fp16 state: 4 x 16 bytes per row
    const int* blk_row;        // [n_blk + 1] first local row of each block; bit 31 = a long row (skipped here)
    int row_base;
    const int* row_ptr;
    const int2* cv;
    const int* slot_map;
    const uint4* rhs_h;
    const uint4* prevh;
    uint4* yh;
    float alpha, w;
};

template <bool CHEB>
__global__ void __launch_bounds__(kTmaThreads, 1)
k_sweep_h_tma(const TmaSweepArgs a, const PeerOut peers) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)kStages * kStageBytes);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(smem_u32(bars + s), kProdWarps);              // full: one arrival per producer warp (+ tx bytes)
            mbar_init(smem_u32(bars + kStages + s), kConsWarps);    // empty: one arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < kProdWarps) {
        // ------------------------------------------------------------------ producers
        uint64_t keep;
        asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(keep));
        int it = 0;
        for (int blk = blockIdx.x; blk < a.n_blk; blk += gridDim.x, ++it) {
            const int st = it % kStages;
            const uint32_t full = smem_u32(bars + st), empty = smem_u32(bars + kStages + st);
            if (it >= kStages) mbar_wait(empty, ((it / kStages) - 1) & 1);
            const int r0raw = __ldg(a.blk_row + blk);
            int n_q = 0, s0 = 0, e0 = 0;
            if (r0raw >= 0) {                                       // not a long row
                const int r1 = __ldg(a.blk_row + blk + 1) & 0x7fffffff;
                s0 = __ldg(a.row_ptr + r0raw);
                e0 = __ldg(a.row_ptr + r1);
                n_q = (e0 - s0 + 3) >> 2;
            }
            uint8_t* xs = smem + (size_t)st * kStageBytes;
            float* vs = reinterpret_cast<float*>(xs + kStageXBytes);
            if (warp == 0 && lane == 0) mbar_expect_tx(full, (uint32_t)n_q * 256u);
            for (int q = warp * 32 + lane; q < n_q; q += kProdWarps * 32) {
                const int i = s0 + 4 * q;
                int2 c[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    c[j] = __ldg(a.cv + min(i + j, e0 - 1));   // tail: repeat the last entry
                    bulk_row64(smem_u32(xs + (size_t)q * 256 + 64 * j), a.xh + (size_t)c[j].x * 4, full, keep);
                }
                *reinterpret_cast<float4*>(vs + 4 * q) =
                    make_float4(__int_as_float(c[0].y), __int_as_float(c[1].y), __int_as_float(c[2].y),
                                __int_as_float(c[3].y));
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(full);
        }
    } else {
        // ------------------------------------------------------------------ consumers
        const int ct = threadIdx.x - kProdWarps * 32;
        const int g = ct / kLPR, l = ct % kLPR;
        int it = 0;
        for (int blk = blockIdx.x; blk < a.n_blk; blk += gridDim.x, ++it) {
            const int st = it % kStages;
            const uint32_t full = smem_u32(bars + st), empty = smem_u32(bars + kStages + st);
            const int r0raw = __ldg(a.blk_row + blk);
            const int r1 = __ldg(a.blk_row + blk + 1) & 0x7fffffff;
            mbar_wait(full, (it / kStages) & 1);
            const uint8_t* xs = smem + (size_t)st * kStageBytes;
            const float* vs = reinterpret_cast<const float*>(xs + kStageXBytes);
            const int row = r0raw + g;
            if (r0raw >= 0 && row < r1) {
                const int s0 = __ldg(a.row_ptr + r0raw);
                const int s = __ldg(a.row_ptr + row) - s0, e = __ldg(a.row_ptr + row + 1) - s0;
                float acc[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] = 0.f;
                int i = s;
                for (; i + 4 <= e; i += 4) {
                    uint4 x[4];
                    float v[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        x[j] = *reinterpret_cast<const uint4*>(xs + (size_t)(i + j) * 64 + l * 16);
                        v[j] = vs[i + j];
                    }
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        float f[8];
                        h8_to_f(x[j], f);
#pragma unroll
                        for (int k = 0; k < 8; ++k) acc[k] = fmaf(v[j], f[k], acc[k]);
                    }
                }
                for (; i < e; ++i) {
                    float f[8];
                    h8_to_f(*reinterpret_cast<const uint4*>(xs + (size_t)i * 64 + l * 16), f);
                    const float v = vs[i];
#pragma unroll
                    for (int k = 0; k < 8; ++k) acc[k] = fmaf(v, f[k], acc[k]);
                }
                // epilogue (as row_epilogue_h, MODE 0)
                const int grow = a.row_base + row;
                const size_t o = (size_t)grow * kLPR + l;
                const int slot = a.slot_map ? __ldg(a.slot_map + grow) : grow;
                float out[8];
                if (slot >= 0) {
                    float r[8];
                    h8_to_f(__ldcs(a.rhs_h + (size_t)slot * kLPR + l), r);
#pragma unroll
                    for (int j = 0; j < 8; ++j) out[j] = fmaf(a.alpha, acc[j], r[j]);
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) out[j] = a.alpha * acc[j];
                }
                if (CHEB) {
                    float p[8];
                    h8_to_f(a.prevh[o], p);
                    const float w1 = 1.f - a.w;
#pragma unroll
                    for (int j = 0; j < 8; ++j) out[j] = fmaf(a.w, out[j], w1 * p[j]);
                }
                const uint4 packed = f_to_h8(out);
                a.yh[o] = packed;
#pragma unroll
                for (int pi = 0; pi < 7; ++pi)
                    if (pi < peers.n) reinterpret_cast<uint4*>(peers.y[pi])[o] = packed;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty);
        }
    }
}

}  // namespace

// Row blocks of the TMA sweep for local rows [0, n_rows): <= 64 rows, <= 1024 non-zeros; a long row is a block of
// its own with bit 31 set.  Host helper (called at graph load).
void tma_build_blocks(const int* row_ptr, int n_rows, int long_thresh, std::vector<int>& blk) {
    blk.clear();
    int r = 0;
    while (r < n_rows) {
        const int deg = row_ptr[r + 1] - row_ptr[r];
        if (deg > long_thresh) { blk.push_back(r | (int)0x80000000); ++r; continue; }
        const int start = r;
        int cnt = 0;
        while (r < n_rows && r - start < kBlkRows) {
            const int d = row_ptr[r + 1] - row_ptr[r];
            if (d > long_thresh || cnt + d > kBlkNnz) break;
            cnt += d;
            ++r;
        }
        blk.push_back(start);
    }
    blk.push_back(n_rows);
}

// MODE 0, non-final sweep over the short rows through the TMA gather; long rows are NOT handled here.
int mixed_sweep_tma(const PprGraph& g, const void* xh, const int* slot_map, const void* rhs_h, const void* prevh,
                    void* yh, float alpha, float w, const PeerOut& peers, cudaStream_t st) {
    HRAG_CHECK(g.tma_blk_row != nullptr && g.n_tma_blk > 0, "mixed_sweep_tma: row blocks not built");
    static bool attr_set = false;
    if (!attr_set) {
        HRAG_CUDA(cudaFuncSetAttribute(k_sweep_h_tma<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
        HRAG_CUDA(cudaFuncSetAttribute(k_sweep_h_tma<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
        attr_set = true;
    }
    TmaSweepArgs a;
    a.n_blk = g.n_tma_blk;
    a.xh = reinterpret_cast<const uint4*>(xh);
    a.blk_row = g.tma_blk_row;
    a.row_base = g.row_lo;
    a.row_ptr = g.row_ptr;
    a.cv = g.cv;
    a.slot_map = slot_map;
    a.rhs_h = reinterpret_cast<const uint4*>(rhs_h);
    a.prevh = reinterpret_cast<const uint4*>(prevh);
    a.yh = reinterpret_cast<uint4*>(yh);
    a.alpha = alpha;
    a.w = w;
    const int grid = std::min(g.n_tma_blk, g.num_sms);
    if (prevh) k_sweep_h_tma<true><<<grid, kTmaThreads, kSmemBytes, st>>>(a, peers);
    else k_sweep_h_tma<false><<<grid, kTmaThreads, kSmemBytes, st>>>(a, peers);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace hrag
