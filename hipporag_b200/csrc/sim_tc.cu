// K2 -- batched query x embedding similarity on the Hopper tensor cores (wgmma, sm_90a).
//
// Replaces the per-query fp32 sgemv of get_fact_scores / dense_passage_retrieval (reference
// HippoRAG.py:1459, :1496: np.dot(E, q)) with one batched contraction S = Q E^T:
//   D[128 queries, 256 embeddings] (fp32, registers) += A[128, BK] (bf16, smem) * B[256, BK]^T (bf16, smem)
// Both operands are K-major (a row = one embedding), staged by TMA (swizzled) into a 4-stage
// shared-memory ring of 48-KB stages (192 KB of the 227 KB a block may use).  Warpgroup 2 issues the
// TMA loads (one thread); warpgroups 0 and 1 each own 64 of the tile's 128 query rows, issue wgmma.m64n256k16 straight
// from shared memory and keep their 64 x 256 fp32 accumulator in registers (128 per thread).
//
// Precision (SURVEY.md 7, hard part 3): a single bf16 pass flips top-k membership, so the parity
// mode is the fp32-faithful split  x = hi + lo (both bf16, 16 mantissa bits together):
//     q.e ~= q_lo.e_lo + q_hi.e_lo + q_lo.e_hi + q_hi.e_hi      (fp32 accumulate)
// All four products are issued per k-block from ONE stage holding {q_hi, q_lo, e_hi, e_lo}:
// 4 products per byte-set of operand traffic, where three separate K-passes would move 1.5x the
// bytes for 3.  Split stages are 32 K-columns wide (64-byte swizzle), so three TMA batches are in
// flight while one is consumed.  The lo.lo term is kept because it is systematic (always positive)
// exactly for the highly correlated query/fact pairs that end up in the top-k.
// HRAG_SIM_BF16 = hi.hi only (64 K-columns a stage, 128-byte swizzle).
#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace hrag {

namespace {

constexpr int BM = 128;          // queries per tile (two warpgroups x wgmma M = 64)
constexpr int BN = 256;          // embeddings per tile (wgmma N)
constexpr int BK = 64;           // bf16 elements per k-block = one 128-byte swizzle row
constexpr int UK = 16;           // wgmma K for 16-bit inputs
constexpr int STAGES = 4;
constexpr int RING_BYTES = STAGES * (BM + BN) * BK * 2;   // 192 KB = 4 stages of 48 KB in both modes
constexpr int CONSUMER_WARPS = 8;                          // warpgroups 0 and 1
constexpr int PRODUCER_WARP = CONSUMER_WARPS;              // first warp of warpgroup 2: TMA
constexpr int TC_THREADS = 32 * (CONSUMER_WARPS + 4);      // 384
// register budget per thread: the producer warpgroup gives up what the consumers' 128-register accumulators need
// (128 x 40 + 256 x 232 <= 64 K registers of the SM)
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr size_t SMEM_BYTES = (size_t)RING_BYTES + 1024 /*align*/ + 256 /*barriers*/;

// ---- PTX wrappers ------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
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
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* map, int c0, int c1) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global [%0, {%1, %2}];" ::"l"(map), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulator registers are written asynchronously by wgmma: pin every read after wgmma_wait
__device__ __forceinline__ void acc_fence(float (&d)[128]) {
#pragma unroll
    for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define HRAG_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                   "+f"(d[i + 6]), "+f"(d[i + 7])
// D[64, 256] (fp32, 128 registers per thread of the warpgroup) (+)= A[64, 16] * B[256, 16]^T, both bf16 K-major in smem
__device__ __forceinline__ void wgmma_bf16(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
        "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
        "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
        "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
        "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, "
        "%128, %129, p, 1, 1, 0, 0;\n\t"
        "}"
        : HRAG_D8(0), HRAG_D8(8), HRAG_D8(16), HRAG_D8(24), HRAG_D8(32), HRAG_D8(40), HRAG_D8(48), HRAG_D8(56),
          HRAG_D8(64), HRAG_D8(72), HRAG_D8(80), HRAG_D8(88), HRAG_D8(96), HRAG_D8(104), HRAG_D8(112), HRAG_D8(120)
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}
#undef HRAG_D8

// wgmma shared-memory descriptor of a K-major operand tile whose rows are ROW_BYTES wide
// (128 -> SWIZZLE_128B, 64 -> SWIZZLE_64B): 8-row swizzle atoms 8*ROW_BYTES apart (SBO); LBO is
// unused by these layouts.
template <int ROW_BYTES>
__device__ __forceinline__ uint64_t gmma_desc_kmajor(uint32_t smem_addr) {
    static_assert(ROW_BYTES == 128 || ROW_BYTES == 64, "row = one swizzle span");
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);        // start address, 16-byte units
    d |= (uint64_t)1 << 16;                              // leading byte offset (ignored)
    d |= (uint64_t)((8u * ROW_BYTES) >> 4) << 32;        // stride byte offset
    d |= (uint64_t)(ROW_BYTES == 128 ? 1 : 2) << 62;     // layout: SWIZZLE_128B = 1, SWIZZLE_64B = 2
    return d;
}

struct TcParams {
    int Bq;            // valid query rows
    int64_t M;         // valid embedding rows
    int dim;
    float* S;
    int64_t ldS;
    int num_m_tiles, num_n_tiles;
    // fused epilogue (FUSE): per (query, n-tile) min/max and the 8 best rank keys instead of scores
    float2* part_mm;          // [Bq, num_n_tiles]
    uint64_t* part_keys;      // [Bq, num_n_tiles, 8]
    uint64_t* bound;          // [Bq] zeroed per launch: the largest 8th-best key of any tile list written so far
    // threshold epilogue (FUSE == 2, index-time synonymy KNN): every score >= thr is appended to its query's
    // candidate list as a rank key; cand_count keeps counting past cand_cap so overflow is detectable
    float thr;
    uint64_t* cand_keys;      // [Bq, cand_cap]
    int* cand_count;          // [Bq]
    int cand_cap;
    // fused epilogue of the exact fallback (FUSE == 1): with gate != null the kernel runs only when *gate != 0
    const int* gate;
    // screen epilogue (FUSE == 4, hi planes only): per (query, tile) the 8 best keys of s1 = hi.hi into part_keys and
    // the two smallest s1 with their rows into part_low {s1 bits, row, s1 bits, row}; err [Bq] = the per-query bound
    // E_q on |s4 - s1|, so the tile lists may drop only keys below the running bound minus 2 E_q
    const float* err;
    uint4* part_low;          // [Bq, num_n_tiles]
    // staged rescore (FUSE == 3): the B rows of m-tile mt are its own stage_tiles staged tiles, of which the first
    // stage_count[mt] are live; scores are stored as in FUSE 0 into S [Bq, stage_tiles * 256]
    int stage_tiles;
    const int* stage_count;   // [num_m_tiles]
};

constexpr int kFuseK = 8;

__device__ __forceinline__ void insert_best(uint64_t (&best)[kFuseK], uint64_t key) {
    if (key > best[kFuseK - 1]) {
#pragma unroll
        for (int k = 0; k < kFuseK; ++k)
            if (key > best[k]) { const uint64_t tmp = best[k]; best[k] = key; key = tmp; }
    }
}
// rank_key of an accumulator register read under a branch.  The bits are taken by an opaque move: a plain bitcast there
// makes the compiler carry the accumulator across the tile loop in integer registers and copy it back before every
// wgmma, which serialises the MMAs (ptxas C7511).
__device__ __forceinline__ uint64_t acc_rank_key(float f, uint32_t idx) {
    uint32_t u;
    asm("mov.b32 %0, %1;" : "=r"(u) : "f"(f));
    return rank_key(__uint_as_float(u), idx);
}
// The accumulator register of bit b of a row half's pass mask (bit 2 j + c = register 4 j + 2 h + c, column
// 8 j + 2 (lane % 4) + c), picked by a switch so that the rare insert path below is compiled once, not once per column.
__device__ __forceinline__ float acc_at(const float (&d)[128], int h, int b) {
    switch (b) {
#define HRAG_ACC_CASE(i) case i: return d[4 * ((i) >> 1) + 2 * h + ((i) & 1)];
#define HRAG_ACC_CASE8(i) HRAG_ACC_CASE(i) HRAG_ACC_CASE(i + 1) HRAG_ACC_CASE(i + 2) HRAG_ACC_CASE(i + 3) \
                          HRAG_ACC_CASE(i + 4) HRAG_ACC_CASE(i + 5) HRAG_ACC_CASE(i + 6) HRAG_ACC_CASE(i + 7)
        HRAG_ACC_CASE8(0) HRAG_ACC_CASE8(8) HRAG_ACC_CASE8(16) HRAG_ACC_CASE8(24)
        HRAG_ACC_CASE8(32) HRAG_ACC_CASE8(40) HRAG_ACC_CASE8(48) HRAG_ACC_CASE8(56)
#undef HRAG_ACC_CASE8
#undef HRAG_ACC_CASE
        default: return 0.f;
    }
}
// best <- the 8 best of best and the keys of the columns set in `pass` (column of bit b: col0 + 8 (b >> 1) + (b & 1)).
// The 8 best of a set of keys do not depend on the order they are inserted in, so the epilogues first mark the
// columns that pass their gate and insert them afterwards in one loop: inserting under each column, unrolled over the
// tile, made the epilogue too large for the instruction cache.
__device__ __forceinline__ void insert_passing(const float (&d)[128], int h, uint64_t pass, uint32_t col0,
                                               uint64_t (&best)[kFuseK]) {
#pragma unroll 1
    while (pass != 0ull) {
        const int b = __ffsll((long long)pass) - 1;
        pass &= pass - 1ull;
        insert_best(best, acc_rank_key(acc_at(d, h, b), col0 + 8u * (uint32_t)(b >> 1) + (uint32_t)(b & 1)));
    }
}
__device__ __forceinline__ void cmp_swap_desc(uint64_t& a, uint64_t& b) {
    const uint64_t hi = a > b ? a : b, lo = a > b ? b : a;
    a = hi;
    b = lo;
}
// best <- the 8 largest of best and lane (lane ^ off)'s best, both sorted descending: max(best[k], other[7 - k])
// holds exactly those 8 as a bitonic sequence, which three compare-exchange rounds sort.  Pairs (k, 7 - k) are
// exchanged together so neither lane reads an entry its partner has already replaced.
__device__ __forceinline__ void merge_best_xor(uint64_t (&best)[kFuseK], int off) {
#pragma unroll
    for (int k = 0; k < kFuseK / 2; ++k) {
        const uint64_t o_hi = __shfl_xor_sync(0xffffffffu, best[kFuseK - 1 - k], off);
        const uint64_t o_lo = __shfl_xor_sync(0xffffffffu, best[k], off);
        best[k] = best[k] > o_hi ? best[k] : o_hi;
        best[kFuseK - 1 - k] = best[kFuseK - 1 - k] > o_lo ? best[kFuseK - 1 - k] : o_lo;
    }
#pragma unroll
    for (int stride = kFuseK / 2; stride >= 1; stride >>= 1)
#pragma unroll
        for (int k = 0; k < kFuseK; ++k)
            if ((k & stride) == 0) cmp_swap_desc(best[k], best[k + stride]);
}

// FUSE: 0 = store scores, 1 = min/max + 8 best per tile, 2 = threshold append, 3 = store scores of staged tiles,
// 4 = screen (8 best and 2 smallest per tile, bound gate widened by 2 E_q)
template <bool SPLIT, int FUSE>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_sim_tc(const __grid_constant__ CUtensorMap map_q_hi, const __grid_constant__ CUtensorMap map_q_lo,
         const __grid_constant__ CUtensorMap map_e_hi, const __grid_constant__ CUtensorMap map_e_lo, TcParams p) {
    constexpr int BKs = SPLIT ? BK / 2 : BK;                 // K-columns per stage
    constexpr int ROW_BYTES = BKs * 2;                       // = the TMA / wgmma swizzle span
    constexpr int A_BYTES = BM * ROW_BYTES, B_BYTES = BN * ROW_BYTES;
    constexpr int STAGE_BYTES = (SPLIT ? 2 : 1) * (A_BYTES + B_BYTES);   // 48 KB either way
    // stage layout: [A_hi | B_hi] or [A_hi | A_lo | B_hi | B_lo]
    constexpr int OFF_A_LO = A_BYTES, OFF_B_HI = SPLIT ? 2 * A_BYTES : A_BYTES, OFF_B_LO = 2 * A_BYTES + B_BYTES;
    constexpr int WG_A_OFF = 64 * ROW_BYTES;                 // a warpgroup's 64 query rows inside an A tile
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;                 // SWIZZLE_128B tiles need 1024-B alignment
    const uint32_t bars = base + RING_BYTES;                      // barrier block
    auto full_bar = [&](int s) { return bars + 8u * s; };
    auto empty_bar = [&](int s) { return bars + 64u + 8u * s; };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nkb = (p.dim + BKs - 1) / BKs;
    const int total_tiles = p.num_m_tiles * p.num_n_tiles;
    if (FUSE == 1 && p.gate != nullptr && *reinterpret_cast<const volatile int*>(p.gate) == 0) return;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (warp == PRODUCER_WARP && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_q_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_e_hi) : "memory");
        if (SPLIT) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_q_lo) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_e_lo) : "memory");
        }
    }
    __syncthreads();

    if (warp >= PRODUCER_WARP) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
        if (warp != PRODUCER_WARP) return;
        // ===== TMA producer =====
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
                const int mt = t % p.num_m_tiles, nt = t / p.num_m_tiles;
                if (FUSE == 3 && nt >= __ldg(p.stage_count + mt)) continue;
                const int brow = FUSE == 3 ? (mt * p.stage_tiles + nt) * BN : nt * BN;
                // L2 prefetch of this CTA's share of the NEXT embedding tile: the num_m_tiles CTAs that
                // will work on it each pull every num_m_tiles-th k-block, a whole tile ahead, so the
                // later TMA loads of all of them are L2 hits instead of num_m_tiles DRAM reads
                const int tn = t + gridDim.x;
                if (FUSE != 3 && tn < total_tiles) {
                    const int mtn = tn % p.num_m_tiles, ntn = tn / p.num_m_tiles;
                    for (int kb = mtn; kb < nkb; kb += p.num_m_tiles) {
                        tma_prefetch_l2_2d(&map_e_hi, kb * BKs, ntn * BN);
                        if (SPLIT) tma_prefetch_l2_2d(&map_e_lo, kb * BKs, ntn * BN);
                    }
                }
                for (int kb = 0; kb < nkb; ++kb) {
                    mbar_wait(empty_bar(stage), phase ^ 1u);
                    mbar_expect_tx(full_bar(stage), STAGE_BYTES);
                    const uint32_t sa = base + stage * STAGE_BYTES;
                    tma_load_2d(sa, &map_q_hi, full_bar(stage), kb * BKs, mt * BM);
                    tma_load_2d(sa + OFF_B_HI, &map_e_hi, full_bar(stage), kb * BKs, brow);
                    if (SPLIT) {
                        tma_load_2d(sa + OFF_A_LO, &map_q_lo, full_bar(stage), kb * BKs, mt * BM);
                        tma_load_2d(sa + OFF_B_LO, &map_e_lo, full_bar(stage), kb * BKs, brow);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1u; }
                }
            }
        }
        return;
    }

    // ===== consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) of each tile =====
    const int wg = warp >> 2;
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
    float d[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) d[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int mt = t % p.num_m_tiles, nt = t / p.num_m_tiles;
        if (FUSE == 3 && nt >= __ldg(p.stage_count + mt)) continue;
        int prev_stage = -1;
        for (int kb = 0; kb < nkb; ++kb) {
            mbar_wait(full_bar(stage), phase);
            const uint32_t sa = base + stage * STAGE_BYTES;
            const uint64_t a_hi = gmma_desc_kmajor<ROW_BYTES>(sa + wg * WG_A_OFF);
            const uint64_t b_hi = gmma_desc_kmajor<ROW_BYTES>(sa + OFF_B_HI);
            wgmma_fence();
            if (SPLIT) {
                const uint64_t a_lo = gmma_desc_kmajor<ROW_BYTES>(sa + OFF_A_LO + wg * WG_A_OFF);
                const uint64_t b_lo = gmma_desc_kmajor<ROW_BYTES>(sa + OFF_B_LO);
                // smallest terms first: lo.lo, hi.lo, lo.hi, then hi.hi; +32 bytes (2 x 16-byte units) along K per step
#pragma unroll
                for (int k = 0; k < BKs / UK; ++k)
                    wgmma_bf16(d, a_lo + (uint64_t)(2 * k), b_lo + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1u : 0u);
#pragma unroll
                for (int k = 0; k < BKs / UK; ++k) wgmma_bf16(d, a_hi + (uint64_t)(2 * k), b_lo + (uint64_t)(2 * k), 1u);
#pragma unroll
                for (int k = 0; k < BKs / UK; ++k) wgmma_bf16(d, a_lo + (uint64_t)(2 * k), b_hi + (uint64_t)(2 * k), 1u);
#pragma unroll
                for (int k = 0; k < BKs / UK; ++k) wgmma_bf16(d, a_hi + (uint64_t)(2 * k), b_hi + (uint64_t)(2 * k), 1u);
            } else {
#pragma unroll
                for (int k = 0; k < BKs / UK; ++k)
                    wgmma_bf16(d, a_hi + (uint64_t)(2 * k), b_hi + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1u : 0u);
            }
            wgmma_commit();
            // at most this k-block's MMAs are still in flight: the previous stage can be refilled
            wgmma_wait<1>();
            if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));
            prev_stage = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        acc_fence(d);
        if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));

        // ===== epilogue from the wgmma accumulator layout: register 4j + 2h + c of this thread holds
        // row 16 (warp % 4) + lane / 4 + 8h, column 8j + 2 (lane % 4) + c of the warpgroup's 64 x 256 block;
        // the four lanes of a quad share a row and hold 64 of its 256 columns each
        const int64_t n0 = (int64_t)nt * BN;
        const int c0 = 2 * (lane & 3);
        const int n_valid = p.M - n0 < BN ? (int)(p.M - n0) : BN;     // columns of this tile below M
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int q = mt * BM + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
            if (FUSE == 2) {
                if (q < p.Bq) {
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                        for (int c = 0; c < 2; ++c) {
                            const int col = 8 * j + c0 + c;
                            const float f = d[4 * j + 2 * h + c];
                            if (col < n_valid && f >= p.thr) {
                                const int pos = atomicAdd(p.cand_count + q, 1);
                                if (pos < p.cand_cap) p.cand_keys[(size_t)q * p.cand_cap + pos] = rank_key(f, (uint32_t)(n0 + col));
                            }
                        }
                }
            } else if (FUSE == 1) {
                // The query's bound is the 8th best key of some set of its scores, so it is at most its global 8th
                // best: a key below it is in no top-k (k <= 8), and the tile's list may drop it.  Only columns whose
                // score is not below `cut`, the score of the bound, are marked and then inserted (few, once the bound
                // has risen); insert_best keeps the lane's 8 best of them.  min / max still see every valid column.
                // !(f < cut) keeps every key >= the bound, ties, -0.0 and NaNs included (the empty
                // bound 0 decodes to a NaN cut, which passes everything).
                const bool live = q < p.Bq;
                const uint64_t thr = live ? __ldcg(reinterpret_cast<const unsigned long long*>(p.bound + q)) : 0ull;
                const float cut = key_score(thr);
                float mn = INFINITY, mx = -INFINITY;
                uint64_t best[kFuseK];
#pragma unroll
                for (int k = 0; k < kFuseK; ++k) best[k] = 0ull;
                uint64_t pass = 0ull;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int col = 8 * j + c0 + c;
                        const float f = d[4 * j + 2 * h + c];
                        const bool valid = col < n_valid;
                        mn = valid ? fminf(mn, f) : mn;
                        mx = valid ? fmaxf(mx, f) : mx;
                        if (live && valid && !(f < cut)) pass |= 1ull << (2 * j + c);
                    }
                }
                insert_passing(d, h, pass, (uint32_t)(n0 + c0), best);
                // merge the quad's four partial results: after two butterfly rounds every lane holds the row's
                // min / max and its 8 best keys
#pragma unroll
                for (int off = 1; off <= 2; off <<= 1) {
                    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, off));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
                    merge_best_xor(best, off);
                }
                if (q < p.Bq && (lane & 3) == 0) {
                    const size_t o = (size_t)q * p.num_n_tiles + nt;
                    p.part_mm[o] = make_float2(mn, mx);
#pragma unroll
                    for (int k = 0; k < kFuseK; k += 2)
                        *reinterpret_cast<ulonglong2*>(p.part_keys + o * kFuseK + k) = make_ulonglong2(best[k], best[k + 1]);
                    // a full list's 8th key is the 8th best of a subset of the query's scores: a valid bound in any
                    // order of tiles and CTAs
                    if (best[kFuseK - 1] > thr)
                        atomicMax(reinterpret_cast<unsigned long long*>(p.bound + q), (unsigned long long)best[kFuseK - 1]);
                }
            } else if (FUSE == 4) {
                // As FUSE 1, in s1 space, with the bound's cut lowered by 2 E_q: a key the gate drops is below every
                // key the candidate band of its query can hold (select.cu: screen_select).  Among the marked keys
                // insert_best keeps the lane's 8 best: a list that drops keys that way is full, and a full list whose
                // 8th key lies in the band marks its tile saturated.  The two smallest valid scores per row are kept
                // beside the list.
                const bool live = q < p.Bq;
                const uint64_t thr = live ? __ldcg(reinterpret_cast<const unsigned long long*>(p.bound + q)) : 0ull;
                const float cut_thr = __fsub_rd(key_score(thr), live ? 2.f * __ldg(p.err + q) : 0.f);
                float m1 = INFINITY, m2 = INFINITY;
                uint32_t i1 = 0xffffffffu, i2 = 0xffffffffu;
                uint64_t best[kFuseK];
#pragma unroll
                for (int k = 0; k < kFuseK; ++k) best[k] = 0ull;
                uint64_t pass = 0ull;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int col = 8 * j + c0 + c;
                        const float f = d[4 * j + 2 * h + c];
                        const bool valid = col < n_valid;
                        if (valid && f < m2) {
                            const uint32_t idx = (uint32_t)(n0 + col);
                            if (f < m1) { m2 = m1; i2 = i1; m1 = f; i1 = idx; }
                            else { m2 = f; i2 = idx; }
                        }
                        if (live && valid && !(f < cut_thr)) pass |= 1ull << (2 * j + c);
                    }
                }
                insert_passing(d, h, pass, (uint32_t)(n0 + c0), best);
#pragma unroll
                for (int off = 1; off <= 2; off <<= 1) {
                    const float o1 = __shfl_xor_sync(0xffffffffu, m1, off), o2 = __shfl_xor_sync(0xffffffffu, m2, off);
                    const uint32_t oi1 = __shfl_xor_sync(0xffffffffu, i1, off), oi2 = __shfl_xor_sync(0xffffffffu, i2, off);
                    // the two smallest of two sorted pairs: the smaller head, then the smaller of the other head and
                    // the winner's second
                    const bool ofirst = o1 < m1 || (o1 == m1 && oi1 < i1);
                    const float l = ofirst ? m1 : o1, w2 = ofirst ? o2 : m2;
                    const uint32_t li = ofirst ? i1 : oi1, w2i = ofirst ? oi2 : i2;
                    m1 = ofirst ? o1 : m1;
                    i1 = ofirst ? oi1 : i1;
                    const bool lfirst = l < w2 || (l == w2 && li < w2i);
                    m2 = lfirst ? l : w2;
                    i2 = lfirst ? li : w2i;
                    merge_best_xor(best, off);
                }
                if (q < p.Bq && (lane & 3) == 0) {
                    const size_t o = (size_t)q * p.num_n_tiles + nt;
                    p.part_low[o] = make_uint4(__float_as_uint(m1), i1, __float_as_uint(m2), i2);
#pragma unroll
                    for (int k = 0; k < kFuseK; k += 2)
                        *reinterpret_cast<ulonglong2*>(p.part_keys + o * kFuseK + k) = make_ulonglong2(best[k], best[k + 1]);
                    if (best[kFuseK - 1] > thr)
                        atomicMax(reinterpret_cast<unsigned long long*>(p.bound + q), (unsigned long long)best[kFuseK - 1]);
                }
            } else {
                if (q < p.Bq) {
                    float* row = p.S + (size_t)q * p.ldS + n0;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j)
                        if (n0 + 8 * j + c0 < p.ldS)     // ldS is a multiple of 4: the whole float2 is in range
                            *reinterpret_cast<float2*>(row + 8 * j + c0) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
                }
            }
        }
    }
}

// x = hi + lo with hi = bf16(x), lo = bf16(x - hi)
__global__ void __launch_bounds__(256)
k_split_bf16(const float* __restrict__ x, int64_t n, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const int64_t i = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 4;
    if (i >= n) return;
    if (i + 3 < n) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(x + i));
        const float f[4] = {v.x, v.y, v.z, v.w};
        __nv_bfloat16 h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            h[j] = __float2bfloat16_rn(f[j]);
            l[j] = __float2bfloat16_rn(f[j] - __bfloat162float(h[j]));
        }
        *reinterpret_cast<uint2*>(hi + i) = *reinterpret_cast<uint2*>(h);
        *reinterpret_cast<uint2*>(lo + i) = *reinterpret_cast<uint2*>(l);
    } else {
        for (int64_t j = i; j < n; ++j) {
            const __nv_bfloat16 h = __float2bfloat16_rn(x[j]);
            hi[j] = h;
            lo[j] = __float2bfloat16_rn(x[j] - __bfloat162float(h));
        }
    }
}

// Upper bounds on the L2 norms of bf16 rows: one warp per row, fp32 sums of squares.  A non-finite norm becomes +inf,
// so a NaN or an infinity in a plane turns every bound built on it into +inf (the screen then falls back).
__device__ __forceinline__ float warp_row_norm(const __nv_bfloat16* __restrict__ x, int dim, int lane) {
    float s = 0.f;
    for (int i = 2 * lane; i < dim; i += 64) {
        const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + i));
        s = fmaf(v.x, v.x, fmaf(v.y, v.y, s));
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    const float n = sqrtf(s);
    return n <= 3.0e38f ? n : INFINITY;
}

// nmax[0] / nmax[1] = max(themselves, the largest row norm of hi / lo over `rows` rows): float bits of non-negative
// values order as unsigned integers
__global__ void __launch_bounds__(256)
k_plane_norm_max(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, int64_t rows, int dim,
                 unsigned int* __restrict__ nmax) {
    const int64_t r = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;
    const float nh = warp_row_norm(hi + (size_t)r * dim, dim, lane), nl = warp_row_norm(lo + (size_t)r * dim, dim, lane);
    if (lane == 0) {
        atomicMax(nmax, __float_as_uint(nh));
        atomicMax(nmax + 1, __float_as_uint(nl));
    }
}

// E_q >= |s4 - s1| for query row q against any fact row, s4 / s1 the split / hi-only K2 accumulators (DESIGN.md
// section 4, the stage-A screen): the three dropped products by Cauchy-Schwarz with the fact planes' largest row norms
// Hf / Lf, plus the fp32 accumulation of both GEMMs at a relative error of 2^-20 per k16 step (dim / 16 steps for s1,
// 4 dim / 16 for s4) on the sum of |products| <= (|qh| + |ql|)(Hf + Lf); the whole raised by 2^-10 for the rounding of
// the norms and of this sum.  2^-20 covers what the H100's wgmma was measured to lose per step: it truncates each of
// the 17 addends two bits below the last place of the largest and truncates their sum, up to 20 2^-25 in all
// (tests/test_gpu_split_exact.py reached 1.18 times the 2^-21 this term used to assume).
__global__ void __launch_bounds__(256)
k_query_err(const __nv_bfloat16* __restrict__ q_hi, const __nv_bfloat16* __restrict__ q_lo, int Bq, int dim,
            const unsigned int* __restrict__ nmax, float* __restrict__ err) {
    const int q = (blockIdx.x * 256 + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q >= Bq) return;
    const float nh = warp_row_norm(q_hi + (size_t)q * dim, dim, lane), nl = warp_row_norm(q_lo + (size_t)q * dim, dim, lane);
    if (lane == 0) {
        const float Hf = __uint_as_float(nmax[0]), Lf = __uint_as_float(nmax[1]);
        const float steps = 5.f * (float)((dim + 15) / 16);
        const float e = nh * Lf + nl * Hf + nl * Lf + steps * 0x1p-20f * (nh + nl) * (Hf + Lf);
        err[q] = e * (1.f + 0x1p-10f);
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

int get_encoder() {
    if (g_encode) return 0;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    HRAG_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    HRAG_CHECK(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    return 0;
}

// [rows, dim] bf16 row-major -> 2-D tensor map with a {box_cols x box_rows} box whose row is one
// swizzle span (64 columns -> 128-byte swizzle, 32 -> 64-byte swizzle).
int make_map(CUtensorMap* map, const void* ptr, int64_t rows, int dim, int box_cols, int box_rows) {
    HRAG_TRY(get_encoder());
    cuuint64_t gdim[2] = {(cuuint64_t)dim, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)dim * 2};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estride[2] = {1, 1};
    CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box,
                          estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    HRAG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return 0;
}

}  // namespace

int split_bf16(const float* x, int64_t n, void* hi, void* lo, cudaStream_t stream) {
    if (n == 0) return 0;
    k_split_bf16<<<(unsigned)ceil_div(ceil_div(n, 4), 256), 256, 0, stream>>>(
        x, n, reinterpret_cast<__nv_bfloat16*>(hi), reinterpret_cast<__nv_bfloat16*>(lo));
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int sim_tc_n_tiles(int64_t M) { return (int)ceil_div(M, BN); }

int sim_tc_threshold(const void* q_hi, const void* q_lo, int Bq, const void* e_hi, const void* e_lo, int64_t M, int dim,
                     int n_seg, float thr, uint64_t* cand_keys, int* cand_count, int cand_cap, int num_sms,
                     cudaStream_t stream) {
    HRAG_CHECK(dim % 8 == 0, "sim_tc: embedding dim must be a multiple of 8 (TMA row pitch)");
    HRAG_CHECK(n_seg == 1 || n_seg == 4, "sim_tc: n_seg must be 1 (bf16) or 4 (split)");
    HRAG_CHECK(cand_keys && cand_count && cand_cap > 0, "sim_tc_threshold: candidate buffers missing");
    if (Bq == 0 || M == 0) return 0;
    static bool attr_set = false;
    if (!attr_set) {
        HRAG_CUDA(cudaFuncSetAttribute(k_sim_tc<true, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        HRAG_CUDA(cudaFuncSetAttribute(k_sim_tc<false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        attr_set = true;
    }
    CUtensorMap mqh, mql, meh, mel;
    const int bkc = n_seg == 4 ? BK / 2 : BK;
    HRAG_TRY(make_map(&mqh, q_hi, Bq, dim, bkc, BM));
    HRAG_TRY(make_map(&mql, q_lo, Bq, dim, bkc, BM));
    HRAG_TRY(make_map(&meh, e_hi, M, dim, bkc, BN));
    HRAG_TRY(make_map(&mel, e_lo, M, dim, bkc, BN));
    TcParams p;
    p.Bq = Bq; p.M = M; p.dim = dim; p.S = nullptr; p.ldS = 0; p.part_mm = nullptr; p.part_keys = nullptr;
    p.bound = nullptr; p.thr = thr; p.cand_keys = cand_keys; p.cand_count = cand_count; p.cand_cap = cand_cap;
    p.gate = nullptr; p.err = nullptr; p.part_low = nullptr; p.stage_tiles = 0; p.stage_count = nullptr;
    p.num_m_tiles = (int)ceil_div(Bq, BM);
    p.num_n_tiles = (int)ceil_div(M, BN);
    const int grid = (int)std::min<int64_t>((int64_t)p.num_m_tiles * p.num_n_tiles, num_sms);
    if (n_seg == 4) k_sim_tc<true, 2><<<grid, TC_THREADS, SMEM_BYTES, stream>>>(mqh, mql, meh, mel, p);
    else k_sim_tc<false, 2><<<grid, TC_THREADS, SMEM_BYTES, stream>>>(mqh, mql, meh, mel, p);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int sim_tc(const void* q_hi, const void* q_lo, int Bq, const void* e_hi, const void* e_lo, int64_t M, int dim,
           int n_seg, float* S, int64_t ldS, float2* part_mm, uint64_t* part_keys, uint64_t* part_bound, int n_ctas,
           cudaStream_t stream, const int* gate) {
    HRAG_CHECK(dim % 8 == 0, "sim_tc: embedding dim must be a multiple of 8 (TMA row pitch)");
    HRAG_CHECK(n_seg == 1 || n_seg == 4, "sim_tc: n_seg must be 1 (bf16) or 4 (split)");
    HRAG_CHECK(part_mm == nullptr || (part_keys != nullptr && part_bound != nullptr), "sim_tc: fused buffers missing");
    if (Bq == 0 || M == 0) return 0;
    static bool attr_set = false;
    if (!attr_set) {
        HRAG_CUDA(cudaFuncSetAttribute(k_sim_tc<true, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        HRAG_CUDA(cudaFuncSetAttribute(k_sim_tc<false, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        HRAG_CUDA(cudaFuncSetAttribute(k_sim_tc<true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        HRAG_CUDA(cudaFuncSetAttribute(k_sim_tc<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        attr_set = true;
    }
    CUtensorMap mqh, mql, meh, mel;
    const int bkc = n_seg == 4 ? BK / 2 : BK;
    HRAG_TRY(make_map(&mqh, q_hi, Bq, dim, bkc, BM));
    HRAG_TRY(make_map(&mql, q_lo, Bq, dim, bkc, BM));
    HRAG_TRY(make_map(&meh, e_hi, M, dim, bkc, BN));
    HRAG_TRY(make_map(&mel, e_lo, M, dim, bkc, BN));
    TcParams p;
    p.Bq = Bq; p.M = M; p.dim = dim; p.S = S; p.ldS = ldS; p.part_mm = part_mm; p.part_keys = part_keys;
    p.bound = part_bound;
    const bool fuse = part_mm != nullptr;
    if (fuse) HRAG_CUDA(cudaMemsetAsync(part_bound, 0, (size_t)Bq * sizeof(uint64_t), stream));
    p.thr = 0.f; p.cand_keys = nullptr; p.cand_count = nullptr; p.cand_cap = 0;
    p.gate = gate; p.err = nullptr; p.part_low = nullptr; p.stage_tiles = 0; p.stage_count = nullptr;
    HRAG_CHECK(fuse || (S != nullptr && ldS % 4 == 0), "sim_tc: score buffer missing");
    p.num_m_tiles = (int)ceil_div(Bq, BM);
    p.num_n_tiles = (int)ceil_div(M, BN);
    const int64_t tiles = (int64_t)p.num_m_tiles * p.num_n_tiles;
    const int grid = (int)std::min<int64_t>(tiles, std::max(n_ctas, 1));
    if (n_seg == 4 && fuse) k_sim_tc<true, 1><<<grid, TC_THREADS, SMEM_BYTES, stream>>>(mqh, mql, meh, mel, p);
    else if (n_seg == 4) k_sim_tc<true, 0><<<grid, TC_THREADS, SMEM_BYTES, stream>>>(mqh, mql, meh, mel, p);
    else if (fuse) k_sim_tc<false, 1><<<grid, TC_THREADS, SMEM_BYTES, stream>>>(mqh, mql, meh, mel, p);
    else k_sim_tc<false, 0><<<grid, TC_THREADS, SMEM_BYTES, stream>>>(mqh, mql, meh, mel, p);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int sim_tc_screen(const void* q_hi, int Bq, const void* e_hi, int64_t M, int dim, const float* err,
                  uint64_t* part_keys, uint4* part_low, uint64_t* part_bound, int n_ctas, cudaStream_t stream) {
    HRAG_CHECK(dim % 8 == 0, "sim_tc_screen: embedding dim must be a multiple of 8 (TMA row pitch)");
    if (Bq == 0 || M == 0) return 0;
    static bool attr_set = false;
    if (!attr_set) {
        HRAG_CUDA(cudaFuncSetAttribute(k_sim_tc<false, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        attr_set = true;
    }
    CUtensorMap mq, me;
    HRAG_TRY(make_map(&mq, q_hi, Bq, dim, BK, BM));
    HRAG_TRY(make_map(&me, e_hi, M, dim, BK, BN));
    TcParams p{};
    p.Bq = Bq; p.M = M; p.dim = dim; p.part_keys = part_keys; p.bound = part_bound; p.err = err; p.part_low = part_low;
    p.num_m_tiles = (int)ceil_div(Bq, BM);
    p.num_n_tiles = (int)ceil_div(M, BN);
    HRAG_CUDA(cudaMemsetAsync(part_bound, 0, (size_t)Bq * sizeof(uint64_t), stream));
    const int64_t tiles = (int64_t)p.num_m_tiles * p.num_n_tiles;
    const int grid = (int)std::min<int64_t>(tiles, std::max(n_ctas, 1));
    k_sim_tc<false, 4><<<grid, TC_THREADS, SMEM_BYTES, stream>>>(mq, mq, me, me, p);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int sim_tc_staged(const void* q_hi, const void* q_lo, int Bq, const void* st_hi, const void* st_lo, int stage_tiles,
                  const int* stage_count, int dim, float* S, int n_ctas, cudaStream_t stream) {
    HRAG_CHECK(dim % 8 == 0, "sim_tc_staged: embedding dim must be a multiple of 8 (TMA row pitch)");
    if (Bq == 0) return 0;
    static bool attr_set = false;
    if (!attr_set) {
        HRAG_CUDA(cudaFuncSetAttribute(k_sim_tc<true, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        attr_set = true;
    }
    TcParams p{};
    p.Bq = Bq; p.dim = dim; p.S = S;
    p.num_m_tiles = (int)ceil_div(Bq, BM);
    p.num_n_tiles = stage_tiles;
    p.stage_tiles = stage_tiles; p.stage_count = stage_count;
    p.M = (int64_t)stage_tiles * BN;          // every staged tile is 256 columns wide (empty slots masked later)
    p.ldS = (int64_t)stage_tiles * BN;
    CUtensorMap mqh, mql, meh, mel;
    const int64_t rows = (int64_t)p.num_m_tiles * stage_tiles * BN;
    HRAG_TRY(make_map(&mqh, q_hi, Bq, dim, BK / 2, BM));
    HRAG_TRY(make_map(&mql, q_lo, Bq, dim, BK / 2, BM));
    HRAG_TRY(make_map(&meh, st_hi, rows, dim, BK / 2, BN));
    HRAG_TRY(make_map(&mel, st_lo, rows, dim, BK / 2, BN));
    const int64_t tiles = (int64_t)p.num_m_tiles * stage_tiles;
    const int grid = (int)std::min<int64_t>(tiles, std::max(n_ctas, 1));
    k_sim_tc<true, 3><<<grid, TC_THREADS, SMEM_BYTES, stream>>>(mqh, mql, meh, mel, p);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int plane_norm_max(const void* hi, const void* lo, int64_t rows, int dim, unsigned int* nmax, cudaStream_t stream) {
    if (rows <= 0) return 0;
    k_plane_norm_max<<<(unsigned)ceil_div(rows * 32, 256), 256, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(hi), reinterpret_cast<const __nv_bfloat16*>(lo), rows, dim, nmax);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int query_err(const void* q_hi, const void* q_lo, int Bq, int dim, const unsigned int* nmax, float* err,
              cudaStream_t stream) {
    if (Bq <= 0) return 0;
    k_query_err<<<(unsigned)ceil_div((int64_t)Bq * 32, 256), 256, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(q_hi), reinterpret_cast<const __nv_bfloat16*>(q_lo), Bq, dim, nmax, err);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace hrag
