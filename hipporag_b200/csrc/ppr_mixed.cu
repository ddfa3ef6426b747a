// K1m -- mixed-precision PPR: fp16 state, fp32 arithmetic, iterative refinement.
//
// K1 (ppr_spmm.cu) is bound by the rate at which the SMs can pull gathered rows of the state
// matrix out of L2 (DESIGN.md section 4), i.e. by bytes per gathered row.  Storing the iterate
// in fp16 halves those bytes: a [N, 32] fp16 state has the same 64-byte rows as the [N, 16]
// fp32 state, so one sweep costs the same and serves twice the queries.  fp32-level accuracy is
// recovered by classical iterative refinement on the linear system (I - aP) x = v:
//     1. x0  ~ solve(v)          m1 Chebyshev sweeps, state + rhs in fp16 (scaled per column)
//     2. r   = v - x0 + aP x0    ONE sweep, fp32 arithmetic on the exact fp32 v and the fp16 x0
//     3. d   ~ solve(r)          m2 Chebyshev sweeps in fp16 (r scaled by t)
//     4. x   = x0 + d            only where it is consumed (passage rows) + the column sums
// (when one round cannot reach the requested tolerance -- large damping -- the caller takes the fp32
// solver instead, solve.cu plan_sweeps).  Every product is accumulated in fp32; only the STORED
// iterate is rounded, and step 2 measures exactly what that rounding (and the truncated step 1)
// left behind: its column sums give the residual check of the solve for free.
//
// Layout: half state [N, 32] row-major (64 B per row); a group of 4 lanes owns a row, each lane
// 8 columns (one 16-byte load per gathered row per lane; sweep.cuh LaneF16).  Rows > long_thresh
// go through K1's segment kernel body and fixed-order finalize sum (sweep.cuh), 4 gathers in flight.
//
// Right-hand side.  The reset vector of graph_search_with_fact_entities (HippoRAG.py:1544-1656)
// is non-zero only on the P passage vertices and on <= link_top_k phrase vertices per query, so
// it is kept COMPACT: `slot_map[node]` (-1 = the row has no rhs) points into `[n_slots, 32]`
// arrays (fp32 exact v, fp16 scaled rhs).  The 90 % of rows that are neither passages nor seeds
// read 4 bytes instead of 64, and building the rhs of a sub-batch touches P x 32 values instead
// of three passes over [N, 32] fp32.  slot_map == nullptr means "dense": slot = row (hrag_ppr's
// arbitrary reset vectors, and the residual rhs of the correction solve).
//
// First iterate.  The first solve starts from x = rhs, so on a single GPU its first two sweeps read that iterate where
// it already is, compactly (template argument X0C): sweep 1 gathers row c as rhs[slot_map[c]] and skips the load of a
// row without a slot (about 3 in 4 of the gathers of a sweep over the whole graph, and those would miss L2), sweep 2's
// Chebyshev epilogue takes prev = its rhs row.  No dense [N, 32] copy of the rhs is built.  Every skipped gather is a
// zero operand of the same fma sequence, so the sums are bit for bit those of the dense first iterate.
//
// Row walk: 4 gathers in flight per lane, the ragged end of a row is one PREDICATED batch (not a
// serial tail), and the 64 rows of a CTA are handed to the groups by length (row_order) so the 8
// rows that share a warp finish together.
//
// K5 (node-range sharding, k_sweep_h_push): each CTA stages its 64 output rows in shared memory
// and pushes the 4-KB block into every peer GPU's copy of y with one TMA bulk copy per peer over
// NVLink; the epoch handshake that replaces a collective is folded into the sweep itself: every
// CTA starts by polling the local flag words (ld.relaxed.sys), the last CTA of the persistent
// grid to finish publishes this rank's epoch to the peers (st.release.sys) -- no extra launches.
#include <algorithm>

#include "sweep.cuh"

namespace hrag {

namespace {

constexpr int kLPR = 4;                 // lanes per row
constexpr int kGPB = kThreads / kLPR;   // rows per CTA
constexpr int kB = 32;                  // batch width of the mixed solver

__device__ __forceinline__ float sat_h(float x) { return fminf(fmaxf(x, -65504.f), 65504.f); }
__device__ __forceinline__ uint4 f_to_h8(const float (&f)[8]) {
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(sat_h(f[2 * j]), sat_h(f[2 * j + 1]));
    return u;
}

// predicated forms: `ok == false` yields zeros without touching memory (the ragged end of a row is a predicated batch)
__device__ __forceinline__ uint4 ld_gather(const uint4* p, bool ok) {
    return ok ? __ldg(p) : make_uint4(0u, 0u, 0u, 0u);
}
__device__ __forceinline__ int2 ld_cv(const int2* p, bool ok) { return ok ? __ldg(p) : make_int2(0, 0); }
// read-once operand of the epilogue (rhs, exact v): no L1 allocation, first out of L2
__device__ __forceinline__ uint4 ld_stream16(const void* p) { return __ldcs(reinterpret_cast<const uint4*>(p)); }
// prev may alias y (in-place Chebyshev): a coherent load, no .nc
__device__ __forceinline__ uint4 ld_prev(const uint4* p) { return *p; }
__device__ __forceinline__ void st_y(uint4* p, const uint4& v) { *p = v; }

constexpr int kU = 4;                   // independent gathers in flight per lane

// Where the first iterate x0 = rhs of a solve is read from (template argument X0C of the sweep kernels): kX0Dense, a
// dense state like every other iterate; kX0AsX, sweep 1 gathers it through the slot map (RhsRows); kX0AsPrev, sweep
// 2's Chebyshev epilogue takes prev = the rhs row it already reads.
constexpr int kX0Dense = 0, kX0AsX = 1, kX0AsPrev = 2;

// The compact first iterate as a gathered operand: row c = rhs[slot_map[c]] (rows kLPR uint4 apart, rhs already
// + lane), zeros when c has no slot -- without a load.
struct RhsRows {
    const int* slot_map;
    const uint4* rhs;
    __device__ __forceinline__ RhsRows operator+(int lane) const { return {slot_map, rhs + lane}; }
};
template <int RS>
__device__ __forceinline__ uint4 gather_row(const RhsRows& x, int col) {
    const int slot = __ldg(x.slot_map + col);
    return slot >= 0 ? __ldg(x.rhs + (size_t)slot * kLPR) : make_uint4(0u, 0u, 0u, 0u);
}
// predicated gather of row c of the state (rows RS uint4 apart) or of the compact first iterate
__device__ __forceinline__ uint4 ld_gather_row(const uint4* x, int rs, int c, bool ok) {
    return ld_gather(x + (size_t)c * rs, ok);
}
__device__ __forceinline__ uint4 ld_gather_row(const RhsRows& x, int, int c, bool ok) {
    const int slot = ok ? __ldg(x.slot_map + c) : -1;
    return ld_gather(x.rhs + slot * kLPR, slot >= 0);
}

template <class Src>
__device__ __forceinline__ void group_row_dot_h(const int2* __restrict__ cv, int s, int e, const Src xh /* + lane */,
                                                float (&acc)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // kU independent 16-byte gathers in flight per lane; the ragged end of the row is a PREDICATED batch, not a
    // serial one-at-a-time loop (a row of 14 non-zeros costs 4 round trips to L2, not 3 + 2)
    for (int i = s; i < e; i += kU) {
        int2 c[kU];
        uint4 a[kU];
#pragma unroll
        for (int j = 0; j < kU; ++j) c[j] = ld_cv(cv + i + j, i + j < e);
#pragma unroll
        for (int j = 0; j < kU; ++j) a[j] = ld_gather_row(xh, kLPR, c[j].x, i + j < e);
#pragma unroll
        for (int j = 0; j < kU; ++j) fma8(acc, __int_as_float(c[j].y), a[j]);
    }
}

// ---- K5 epoch handshake, folded into the sweep kernels ---------------------------------------
__device__ __forceinline__ void sync_wait(const SweepSync& sy) {
    if (sy.flags == nullptr) return;                 // single GPU (uniform branch)
    const int r = threadIdx.x;
    if (r < sy.world && r != sy.rank) {
        unsigned long long v = 0;
        long long spin = 0;
#pragma unroll 1
        for (; spin < (1ll << 24); ++spin) {         // bounded (~seconds): a lost peer must not hang the GPU
            // relaxed, not acquire: an acquire load at system scope is followed by CCTL.IVALL, i.e. every poll of every
            // CTA would flush the SM's L1 under the CTAs already gathering.  Nothing stale can be in L1: it is
            // invalidated at kernel launch and no row of x is loaded before this wait has passed.
            asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(sy.flags + r) : "memory");
            if (v >= sy.need) break;
            __nanosleep(32);
        }
        if (v < sy.need) *sy.error_flag = 1;
    }
    __syncthreads();
}
__device__ __forceinline__ void sync_signal(const SweepSync& sy) {
    if (sy.flags == nullptr || sy.done_ctr == nullptr) return;
    __syncthreads();                                 // every thread's (peer) stores are issued
    if (threadIdx.x == 0) {
        __threadfence_system();
        const unsigned int prev = atomicAdd(sy.done_ctr, 1u);
        if (prev + 1 == sy.total_ctas) {             // last CTA of the sweep: publish this rank's epoch
            *sy.done_ctr = 0;
            __threadfence_system();
#pragma unroll
            for (int i = 0; i < 7; ++i)                  // static indices: kernel parameters stay in the constant bank
                if (i < sy.n_remote)
                    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(sy.remote[i]), "l"(sy.epoch) : "memory");
        }
    }
}

// MODE 0: y = w * (alpha * acc + rhs) + (1 - w) * prev        (all fp16 in memory)
// MODE 1: y = t * (scale * v32 - x0 + alpha * acc)            (the refinement residual)
// rhs / v32 are addressed through slot_map (null = dense).  Returns (in out[]) the value as
// STORED (after fp16 rounding) so column sums match memory; MODE 1 + FINAL returns |value|.  RS: row stride in uint4 of
// x0h / prevh / yh and of a dense rhs_h (kLPR; 2 kLPR when two states are interleaved row by row); compact rhs_h and v32
// are per state.  PREV_RHS: prev is the rhs row itself (kX0AsPrev), zeros where the row has no slot.
template <bool CHEB, int MODE, int RS = kLPR, bool PREV_RHS = false>
__device__ __forceinline__ void row_epilogue_h(float (&acc)[8], int row, int lane, const int* __restrict__ slot_map,
                                               const uint4* __restrict__ rhs_h, const float4* __restrict__ v32,
                                               const float* __restrict__ col_scale, const uint4* x0h,
                                               const uint4* prevh, uint4* yh, float alpha, float w, float t,
                                               const PeerOut& peers, int* overflow, float (&out)[8], uint4& packed_out) {
    const size_t o = (size_t)row * RS + lane;
    const int slot = slot_map ? __ldg(slot_map + row) : row;
    if (MODE == 0) {
        float r[8];
        if (slot >= 0) {
            h8_to_f(ld_stream16(rhs_h + (size_t)slot * (slot_map ? kLPR : RS) + lane), r);
#pragma unroll
            for (int j = 0; j < 8; ++j) out[j] = fmaf(alpha, acc[j], r[j]);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) out[j] = alpha * acc[j];
        }
        if (CHEB) {
            float p[8];
            if (PREV_RHS) {
#pragma unroll
                for (int j = 0; j < 8; ++j) p[j] = slot >= 0 ? r[j] : 0.f;
            } else {
                h8_to_f(ld_prev(prevh + o), p);
            }
            const float w1 = 1.f - w;
#pragma unroll
            for (int j = 0; j < 8; ++j) out[j] = fmaf(w, out[j], w1 * p[j]);
        }
    } else {
        float x0[8];
        h8_to_f(__ldg(x0h + o), x0);
        float v[8];
        if (slot >= 0) {
            const float4* vp = v32 + ((size_t)slot * kLPR + lane) * 2;
            const uint4 ua = ld_stream16(vp), ub = ld_stream16(vp + 1);
            v[0] = __uint_as_float(ua.x); v[1] = __uint_as_float(ua.y); v[2] = __uint_as_float(ua.z); v[3] = __uint_as_float(ua.w);
            v[4] = __uint_as_float(ub.x); v[5] = __uint_as_float(ub.y); v[6] = __uint_as_float(ub.z); v[7] = __uint_as_float(ub.w);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float sc = __ldg(col_scale + lane * 8 + j);
            out[j] = t * (fmaf(alpha, acc[j], fmaf(sc, v[j], -x0[j])));
        }
    }
    // fp16 rounds |x| >= 65520 to inf, so sat_h would clamp such a value and change the answer: flag it (pinned small
    // sweep counts on a concentrated seed can push the scaled residual that far; the host turns the flag into an error)
    float mx = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fabsf(out[j]));
    if (mx >= 65520.f && overflow) *overflow = 1;
    const uint4 packed = f_to_h8(out);
    packed_out = packed;
    st_y(yh + o, packed);
    // K5, direct form (long rows only): the same 16 bytes go into every peer GPU's copy of y.  The main kernel passes
    // no peers here and pushes its whole 4-KB row block at once (below)
#pragma unroll
    for (int i = 0; i < 7; ++i)
        if (i < peers.n) reinterpret_cast<uint4*>(peers.y[i])[o] = packed;
    h8_to_f(packed, out);
    if (MODE == 1) {
#pragma unroll
        for (int j = 0; j < 8; ++j) out[j] = fabsf(out[j]);
    }
}

// The same sums as sweep.cuh's block_colsum<LaneF16, 4>, kept here because nvcc schedules k_sweep_h / k_sweep_h_push
// differently through the shared one; their code stays as it is measured.
__device__ __forceinline__ void block_colsum_h(float (&v)[8], float* __restrict__ partial_row) {
    __shared__ float s_sum[kThreads / 32][kB];
#pragma unroll
    for (int off = kLPR; off < 32; off <<= 1)
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += __shfl_xor_sync(0xffffffffu, v[j], off);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane < kLPR)
#pragma unroll
        for (int j = 0; j < 8; ++j) s_sum[warp][lane * 8 + j] = v[j];
    __syncthreads();
    if (threadIdx.x < kB) {
        float s = 0.f;
#pragma unroll
        for (int wi = 0; wi < kThreads / 32; ++wi) s += s_sum[wi][threadIdx.x];
        partial_row[threadIdx.x] = s;
    }
}

struct SweepArgs {
    int n_rows, row_base, long_thresh;
    const int* row_order;      // null = identity; else the local row handled by slot (cta * 64 + group): the 64 rows
                               // of a CTA sorted by length, so the 8 rows that share a warp finish together
    const int* row_ptr;
    const int2* cv;
    const uint4* xh;
    const int* slot_map;
    const uint4* rhs_h;
    const float4* v32;
    const float* col_scale;
    const uint4* prevh;
    uint4* yh;
    float alpha, w, t;
    float* partials;
    int* overflow;             // set to 1 when a stored value would leave fp16's range (null = not reported)
};

// Single-GPU sweep: one block of 64 rows per CTA.  (Kept free of the exchange code of k_sweep_h_push below: a block
// loop with the staging / bulk-copy code behind a uniform branch slows the plain sweep down.)
template <bool CHEB, int MODE, bool FINAL, int X0C = kX0Dense>
__global__ void __launch_bounds__(kThreads, 6)
k_sweep_h(const SweepArgs a) {
    const int g = threadIdx.x / kLPR, l = threadIdx.x % kLPR;
    const int slot_r = blockIdx.x * kGPB + g;
    float out[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) out[j] = 0.f;
    if (slot_r < a.n_rows) {
        const int r = a.row_order ? __ldg(a.row_order + slot_r) : slot_r;
        const int s = __ldg(a.row_ptr + r), e = __ldg(a.row_ptr + r + 1);
        if (e - s <= a.long_thresh) {
            float acc[8];
            uint4 packed;
            if (X0C == kX0AsX) group_row_dot_h(a.cv, s, e, RhsRows{a.slot_map, a.rhs_h + l}, acc);
            else group_row_dot_h(a.cv, s, e, a.xh + l, acc);
            row_epilogue_h<CHEB, MODE, kLPR, X0C == kX0AsPrev>(acc, a.row_base + r, l, a.slot_map, a.rhs_h, a.v32,
                                                               a.col_scale, a.xh, a.prevh, a.yh, a.alpha, a.w, a.t,
                                                               PeerOut(), a.overflow, out, packed);
        }
    }
    if (FINAL) block_colsum_h(out, a.partials + (size_t)blockIdx.x * kB);
}

// Paired sweep: one walk of a row's non-zeros serves two states A and B (two sub-batches of 32 columns) stored
// interleaved, [N, 2, 32]: each cv entry is loaded once and its two 16-byte gathers per lane fall in one 128-byte line,
// and the column-independent bytes (cv, row_ptr, row_order) are paid once per 64 columns.  Each state's sums keep
// k_sweep_h's order: the same fma sequence per lane, the same epilogue and the same column-sum partials.
constexpr int kRS2 = 2 * kLPR;          // row stride of the interleaved pair in uint4
template <class Src>
__device__ __forceinline__ void group_row_dot_h2(const int2* __restrict__ cv, int s, int e, const Src xa, const Src xb,
                                                 float (&acc_a)[8], float (&acc_b)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) acc_a[j] = acc_b[j] = 0.f;
    for (int i = s; i < e; i += kU) {
        int2 c[kU];
        uint4 a[kU], b[kU];
#pragma unroll
        for (int j = 0; j < kU; ++j) c[j] = ld_cv(cv + i + j, i + j < e);
#pragma unroll
        for (int j = 0; j < kU; ++j) {
            a[j] = ld_gather_row(xa, kRS2, c[j].x, i + j < e);
            b[j] = ld_gather_row(xb, kRS2, c[j].x, i + j < e);
        }
#pragma unroll
        for (int j = 0; j < kU; ++j) {
            fma8(acc_a, __int_as_float(c[j].y), a[j]);
            fma8(acc_b, __int_as_float(c[j].y), b[j]);
        }
    }
}

// 64 registers (4 CTAs per SM: 8 gathers in flight per lane, 8 K per SM against k_sweep_h's 6 K); FINAL keeps both
// states' stored values for the column sums and takes 72 registers (3 CTAs per SM) rather than spill.  With X0C ==
// kX0AsX each state gathers its own compact first iterate: the passage slots are shared, the seed slots are not.
template <bool CHEB, int MODE, bool FINAL, int X0C = kX0Dense>
__global__ void __launch_bounds__(kThreads, FINAL ? 3 : 4)
k_sweep_h2(const SweepArgs a, const SweepArgs b) {
    const int g = threadIdx.x / kLPR, l = threadIdx.x % kLPR;
    const int slot_r = blockIdx.x * kGPB + g;
    float out_a[8], out_b[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) out_a[j] = out_b[j] = 0.f;
    if (slot_r < a.n_rows) {
        const int r = a.row_order ? __ldg(a.row_order + slot_r) : slot_r;
        const int s = __ldg(a.row_ptr + r), e = __ldg(a.row_ptr + r + 1);
        if (e - s <= a.long_thresh) {
            float acc_a[8], acc_b[8];
            uint4 packed;
            if (X0C == kX0AsX)
                group_row_dot_h2(a.cv, s, e, RhsRows{a.slot_map, a.rhs_h + l}, RhsRows{b.slot_map, b.rhs_h + l}, acc_a,
                                 acc_b);
            else group_row_dot_h2(a.cv, s, e, a.xh + l, b.xh + l, acc_a, acc_b);
            constexpr bool PR = X0C == kX0AsPrev;
            row_epilogue_h<CHEB, MODE, kRS2, PR>(acc_a, a.row_base + r, l, a.slot_map, a.rhs_h, a.v32, a.col_scale,
                                                 a.xh, a.prevh, a.yh, a.alpha, a.w, a.t, PeerOut(), a.overflow, out_a,
                                                 packed);
            row_epilogue_h<CHEB, MODE, kRS2, PR>(acc_b, a.row_base + r, l, b.slot_map, b.rhs_h, b.v32, b.col_scale,
                                                 b.xh, b.prevh, b.yh, a.alpha, a.w, a.t, PeerOut(), a.overflow, out_b,
                                                 packed);
        }
    }
    if (FINAL) {
        block_colsum_h(out_a, a.partials + (size_t)blockIdx.x * kB);
        __syncthreads();                             // block_colsum_h's shared scratch is reused
        block_colsum_h(out_b, b.partials + (size_t)blockIdx.x * kB);
    }
}

// K5, the sharded sweep: the same row computation with the exchange fused in.
template <bool CHEB, int MODE, bool FINAL>
__global__ void __launch_bounds__(kThreads, 6)
k_sweep_h_push(const SweepArgs a, const PeerOut peers, const SweepSync sy) {
    // K5 staging: a block's 64 output rows are one contiguous 4-KB piece of y.  They are collected in shared memory and
    // pushed to every peer as ONE bulk copy per peer by the TMA engine (cp.async.bulk shared -> peer global over NVLink,
    // SASS UBLKCP): full-size NVLink packets, no store instructions on the SMs' LSUs, double-buffered so the copy of block
    // k overlaps the gathers of block k + 1.  Blocks that are not whole (ragged end, a long row inside) fall back to
    // coalesced 16-byte stores (thread t -> bytes [16 t, 16 t + 16)).
    __shared__ __align__(128) uint4 s_out[2][kThreads];
    __shared__ unsigned char s_valid[kGPB];
    sync_wait(sy);
    const int g = threadIdx.x / kLPR, l = threadIdx.x % kLPR;
    const bool push = peers.n > 0;                       // uniform
    const int n_blocks = (a.n_rows + kGPB - 1) / kGPB;
    int buf = 0;
    // a persistent grid strides over the blocks, so the system-scope fence that must follow the peer writes (and waits
    // for their acknowledgements) is paid once per CTA at the end of the sweep, not once per 64 rows
    for (int blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        const int slot_r = blk * kGPB + g;
        if (push) {
            // the bulk copies that read s_out[buf] two blocks ago must have finished reading it
            if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            if (l == 0) s_valid[g] = 0;
            __syncthreads();
        }
        float out[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) out[j] = 0.f;
        if (slot_r < a.n_rows) {
            const int r = a.row_order ? __ldg(a.row_order + slot_r) : slot_r;
            const int s = __ldg(a.row_ptr + r), e = __ldg(a.row_ptr + r + 1);
            if (e - s <= a.long_thresh) {
                float acc[8];
                uint4 packed;
                group_row_dot_h(a.cv, s, e, a.xh + l, acc);
                row_epilogue_h<CHEB, MODE>(acc, a.row_base + r, l, a.slot_map, a.rhs_h, a.v32, a.col_scale, a.xh,
                                           a.prevh, a.yh, a.alpha, a.w, a.t, PeerOut(), a.overflow, out, packed);
                if (push) {
                    const int rl = r - blk * kGPB;       // row_order permutes rows inside their own 64-row block only
                    s_out[buf][rl * kLPR + l] = packed;
                    if (l == 0) s_valid[rl] = 1;
                }
            }
        }
        if (push) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the TMA engine
            const int whole = __syncthreads_and(s_valid[threadIdx.x / kLPR] != 0);
            const size_t o0 = (size_t)(a.row_base + blk * kGPB) * kLPR;
            if (whole) {
                if (threadIdx.x == 0) {
                    const uint32_t src = (uint32_t)__cvta_generic_to_shared(&s_out[buf][0]);
#pragma unroll
                    for (int i = 0; i < 7; ++i)
                        if (i < peers.n)
                            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                                         ::"l"(reinterpret_cast<uint4*>(peers.y[i]) + o0), "r"(src), "r"((uint32_t)(kThreads * 16))
                                         : "memory");
                }
            } else if (s_valid[threadIdx.x / kLPR]) {
                const uint4 v = s_out[buf][threadIdx.x];
#pragma unroll
                for (int i = 0; i < 7; ++i)
                    if (i < peers.n) reinterpret_cast<uint4*>(peers.y[i])[o0 + threadIdx.x] = v;
            }
            if (threadIdx.x == 0) asm volatile("cp.async.bulk.commit_group;" ::: "memory");   // one group per block, empty or not
            buf ^= 1;
        }
        if (FINAL) {
            block_colsum_h(out, a.partials + (size_t)blk * kB);
            if (blk + (int)gridDim.x < n_blocks) __syncthreads();     // its shared scratch is reused by the next block
        }
    }
    if (push && threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all peer writes performed
    sync_signal(sy);
}

// Src: the state (const uint4*), or RhsRows for the compact first iterate
template <int RS = kLPR, class Src = const uint4*>
__global__ void __launch_bounds__(kThreads)
k_sweep_long_segments_h(int n_seg, const int4* __restrict__ segs, const int2* __restrict__ cv, const Src xh,
                        F8* __restrict__ seg_partial, const SweepSync sy) {
    sync_wait(sy);
    segment_partial<LaneF16, kLPR, RS, Src>(n_seg, segs, cv, nullptr, xh, seg_partial);
}

template <bool CHEB, int MODE, bool FINAL, int RS = kLPR, bool PREV_RHS = false>
__global__ void __launch_bounds__(kThreads)
k_sweep_long_finalize_h(int n_long, const int* __restrict__ long_rows, const int* __restrict__ long_seg_ptr,
                        const F8* __restrict__ seg_partial, const SweepArgs a, const PeerOut peers,
                        const SweepSync sy) {
    const int g = threadIdx.x / kLPR, l = threadIdx.x % kLPR;
    const int k = blockIdx.x * kGPB + g;
    float out[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) out[j] = 0.f;
    if (k < n_long) {
        const int r = __ldg(long_rows + k);
        F8 acc = segment_sum<LaneF16, kLPR>(long_seg_ptr, k, seg_partial + l);
        uint4 packed;
        row_epilogue_h<CHEB, MODE, RS, PREV_RHS>(acc.v, a.row_base + r, l, a.slot_map, a.rhs_h, a.v32, a.col_scale,
                                                 a.xh, a.prevh, a.yh, a.alpha, a.w, a.t, peers, a.overflow, out, packed);
    }
    if (FINAL) block_colsum_h(out, a.partials + (size_t)blockIdx.x * kB);
    sync_signal(sy);
}

// stand-alone halves of the handshake, for the exchange points that are not sweeps (see comm.cu)
__global__ void k_epoch_wait(const SweepSync sy) { sync_wait(sy); }
__global__ void k_epoch_signal(const SweepSync sy) { sync_signal(sy); }

// ---- dense prepare path (hrag_ppr: arbitrary reset vectors) ------------------------------------
// per-CTA column sums of a non-negative fp32 [N, 32] matrix -> partial[blockIdx, 32]
__global__ void __launch_bounds__(256)
k_colsum32_partial(const float* __restrict__ V, int64_t n_elems, float* __restrict__ partial) {
    float m = 0.f;                                   // thread's column = threadIdx.x % 32 (strides are multiples of 32)
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n_elems; i += (int64_t)gridDim.x * 256) m += V[i];
    __shared__ float s[256];
    s[threadIdx.x] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        for (int k = 1; k < 8; ++k) m += s[threadIdx.x + 32 * k];
        partial[(size_t)blockIdx.x * 32 + threadIdx.x] = m;
    }
}
// All entries of x = (I - aP)^-1 v are >= 0 and sum to <= sum(v) / (1 - a), so no entry of the
// scaled iterate can exceed fp16's range when  scale * sum(v) / (1 - a) <= 32768:
// scale[b] = 2^floor(log2(32768 (1 - a) / sum_b))      (sum == 0: an unused column -> 1)
__device__ __forceinline__ float column_scale(float sv, float one_minus_alpha) {
    return sv > 0.f ? exp2f(floorf(log2f(32768.f * one_minus_alpha / sv))) : 1.f;
}
__global__ void k_scales32(const double* __restrict__ vsum, float one_minus_alpha, float* __restrict__ scale) {
    scale[threadIdx.x] = column_scale((float)vsum[threadIdx.x], one_minus_alpha);
}
// V16[n, b] = fp16(scale[b] * V32[n, b])
__global__ void __launch_bounds__(256)
k_scale_to_half(const float4* __restrict__ V, int64_t n_vec8, const float* __restrict__ scale, uint4* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;       // one 8-column group
    if (i >= n_vec8) return;
    const int c0 = (int)(i & 3) * 8;
    const float4 a = __ldcs(V + 2 * i), b = __ldcs(V + 2 * i + 1);
    float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= __ldg(scale + c0 + j);
    out[i] = f_to_h8(f);
}

// ---- compact prepare path (stage B: passage weights + phrase seeds) ----------------------------
// Vc[p, b] = fp32(minmax(S[q0+b, p])) * fp32(pnw) for the P passage slots (HippoRAG.py:1626-1633; the
// product is formed in fp32 as numpy does for float32 * python float); columns b >= nb are 0.
// 32 passages x 32 queries per CTA through a shared-memory transpose: S is read along passages
// (coalesced), Vc written along queries.  partial[blockIdx, b] = the CTA's column sums.
__global__ void __launch_bounds__(256)
k_rhs_passages(int P, int nb, const float* __restrict__ S, int64_t ldS, int q0, const float2* __restrict__ minmax,
               float pnw, float* __restrict__ Vc, float* __restrict__ partial) {
    __shared__ float tile[32][33];
    __shared__ float red[8][32];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int p0 = blockIdx.x * 32;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int b = ty + 8 * k, p = p0 + tx;
        float v = 0.f;
        if (b < nb && p < P) {
            const float2 mm = __ldg(minmax + q0 + b);
            const float range = mm.y - mm.x;
            const float s = __ldcs(S + (size_t)(q0 + b) * ldS + p);
            const float nrm = range == 0.f ? 1.f : __fdiv_rn(s - mm.x, range);   // misc_utils.py:130-139
            v = nrm * pnw;
        }
        tile[b][tx] = v;
    }
    __syncthreads();
    float csum = 0.f;                                   // column tx over this thread's 4 passages
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int pl = ty + 8 * k;
        const float v = tile[tx][pl];
        if (p0 + pl < P) Vc[(size_t)(p0 + pl) * kB + tx] = v;
        csum += v;
    }
    red[ty][tx] = csum;
    __syncthreads();
    if (ty == 0) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += red[k][tx];
        partial[(size_t)blockIdx.x * kB + tx] = s;
    }
}

// One CTA: gives every distinct seed vertex of the sub-batch a slot (passage vertices keep theirs), adds the
// phrase weights (HippoRAG.py:1638 phrase + passage weights), finishes the column sums of v and derives the
// fp16 column scales.  Item i = (query b = i / slots_per_query, seed r = i % slots_per_query) owns slot P + i.
__global__ void __launch_bounds__(1024)
k_rhs_seeds(int P, int nb, int q0, int slots_per_query, const int* __restrict__ seed_vid,
            const double* __restrict__ seed_w, int* __restrict__ slot_map, int* __restrict__ slot_vid,
            float* __restrict__ Vc, const float* __restrict__ partial, int n_partial, float one_minus_alpha,
            double* __restrict__ vsum, float* __restrict__ scale) {
    __shared__ double s_sum[32][33];
    __shared__ double s_seed[32];
    const int t = threadIdx.x;
    if (t < 32) s_seed[t] = 0.0;
    __syncthreads();
    const int n_items = kB * slots_per_query;
    for (int i = t; i < n_items; i += 1024) {
        const int b = i / slots_per_query, r = i % slots_per_query;
        int created = -1;
        if (b < nb) {
            const int v = seed_vid[(size_t)(q0 + b) * slots_per_query + r];
            if (v >= 0) {
                const float w = (float)seed_w[(size_t)(q0 + b) * slots_per_query + r];
                const int old = atomicCAS(slot_map + v, -1, P + i);
                const int slot = old < 0 ? P + i : old;
                if (old < 0) created = v;
                // (vertex, query) pairs are distinct; seed rows were zeroed by the caller, passage rows hold the
                // passage weight written by k_rhs_passages (stream order)
                atomicAdd(Vc + (size_t)slot * kB + b, w);
                atomicAdd(&s_seed[b], (double)w);
            }
        }
        slot_vid[P + i] = created;
    }
    const int col = t & 31, part = t >> 5;           // 32 columns x 32 partial lanes
    double acc = 0.0;
    for (int i = part; i < n_partial; i += 32) acc += (double)partial[(size_t)i * kB + col];
    s_sum[part][col] = acc;
    __syncthreads();
    if (t < 32) {
        double s = s_seed[t];
        for (int i = 0; i < 32; ++i) s += s_sum[i][t];
        vsum[t] = s;
        scale[t] = column_scale((float)s, one_minus_alpha);
    }
}

// rhs16[slot, :] = fp16(scale * Vc[slot, :]) for every slot, and (x0 not null) the same row scattered into the dense
// first iterate x0 (zeroed by the caller): x0[vertex(slot), :], rows x0_stride uint4 apart
__global__ void __launch_bounds__(256)
k_rhs_convert(int P, int n_slots, const int* __restrict__ passage_vid, const int* __restrict__ slot_vid,
              const float4* __restrict__ Vc, const float* __restrict__ scale, uint4* __restrict__ rhs16,
              uint4* __restrict__ x0, int x0_stride) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;       // one 8-column group
    const int slot = (int)(i >> 2), l = (int)(i & 3);
    if (slot >= n_slots) return;
    const float4 a = __ldcs(Vc + 2 * i), b = __ldcs(Vc + 2 * i + 1);
    float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= __ldg(scale + l * 8 + j);
    const uint4 h = f_to_h8(f);
    rhs16[i] = h;
    if (x0 == nullptr) return;
    const int vid = slot < P ? __ldg(passage_vid + slot) : __ldg(slot_vid + slot);
    if (vid >= 0) x0[(size_t)vid * x0_stride + l] = h;
}

// undo k_rhs_seeds: seed vertices that were given a slot of their own go back to "no rhs"
__global__ void __launch_bounds__(1024)
k_slot_clear(int P, int nb, int q0, int slots_per_query, const int* __restrict__ seed_vid, int* __restrict__ slot_map) {
    const int n_items = kB * slots_per_query;
    for (int i = threadIdx.x; i < n_items; i += 1024) {
        const int b = i / slots_per_query, r = i % slots_per_query;
        if (b >= nb) continue;
        const int v = seed_vid[(size_t)(q0 + b) * slots_per_query + r];
        if (v >= 0 && slot_map[v] >= P) slot_map[v] = -1;
    }
}

__global__ void __launch_bounds__(256)
k_slot_map_init(int N, int* __restrict__ slot_map) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < N) slot_map[i] = -1;
}
__global__ void __launch_bounds__(256)
k_slot_map_passages(int P, const int* __restrict__ passage_vid, int* __restrict__ slot_map) {
    const int p = blockIdx.x * 256 + threadIdx.x;
    if (p < P) slot_map[passage_vid[p]] = p;
}

// relative L1 size of the refinement residual per column: rho[b] = (sum_i |r_i| / t) / (scale[b] * sum v);
// keeps the running maximum over every solve since the last reset (checked on the host, solve.cu)
__global__ void k_residual_check(const double* __restrict__ rsum, const double* __restrict__ vsum,
                                 const float* __restrict__ scale, float inv_t, float* __restrict__ rho_max) {
    const int b = threadIdx.x;
    const double den = (double)scale[b] * vsum[b];
    float rho = den > 0.0 ? (float)(rsum[b] * (double)inv_t / den) : 0.f;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) rho = fmaxf(rho, __shfl_xor_sync(0xffffffffu, rho, off));
    if (b == 0 && rho > *rho_max) *rho_max = rho;
}

__global__ void __launch_bounds__(256)
k_gather_passage_scores_mixed(int P, int nb, int q0, const int* __restrict__ passage_vid,
                              const __half* __restrict__ X0, const __half* __restrict__ D, float inv_t,
                              const double* __restrict__ sum0, const double* __restrict__ sum1,
                              const int* __restrict__ mode, const float2* __restrict__ minmax, float* S, int64_t ldS,
                              int ldx) {
    const int64_t tI = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int p = (int)(tI / nb), b = (int)(tI % nb);
    if (p >= P) return;
    float* dst = S + (size_t)(q0 + b) * ldS + p;
    if (mode[q0 + b]) {
        const size_t o = (size_t)__ldg(passage_vid + p) * ldx + b;
        const float z = __half2float(X0[o]) + inv_t * __half2float(D[o]);        // x = x0 + d
        const float tot = (float)(sum0[b] + (double)inv_t * sum1[b]);
        *dst = __fdiv_rn(z, tot);
    } else {
        const float2 mm = __ldg(minmax + q0 + b);
        const float range = mm.y - mm.x;
        *dst = range == 0.f ? 1.f : __fdiv_rn(*dst - mm.x, range);
    }
}

__global__ void __launch_bounds__(256)
k_state_to_scores_mixed(const __half* __restrict__ X0, const __half* __restrict__ D, float inv_t, int nb, int N,
                        const double* __restrict__ sum0, const double* __restrict__ sum1, float* __restrict__ out) {
    const int64_t tI = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int n = (int)(tI / nb), b = (int)(tI % nb);
    if (n >= N) return;
    const size_t o = (size_t)n * kB + b;
    const float z = __half2float(X0[o]) + inv_t * __half2float(D[o]);
    out[(size_t)b * N + n] = __fdiv_rn(z, (float)(sum0[b] + (double)inv_t * sum1[b]));
}

}  // namespace

int mixed_partial_rows(const PprGraph& g) { return sweep_partial_rows(g, kGPB); }

int epoch_wait(const SweepSync& sync, cudaStream_t st) {
    k_epoch_wait<<<1, 32, 0, st>>>(sync);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}
int epoch_signal(const SweepSync& sync, cudaStream_t st) {
    SweepSync sy = sync;
    sy.total_ctas = 1;
    k_epoch_signal<<<1, 32, 0, st>>>(sy);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

// The kernels' arguments for one state's sweep
static SweepArgs sweep_args(const PprGraph& g, const MixedSweepIO& io, float alpha, float w, float t, int* overflow) {
    SweepArgs a;
    a.n_rows = g.n_rows; a.row_base = g.row_lo; a.long_thresh = g.long_thresh;
    a.row_order = g.row_order;
    a.row_ptr = g.row_ptr; a.cv = g.cv;
    a.xh = reinterpret_cast<const uint4*>(io.xh);
    a.slot_map = io.slot_map;
    a.rhs_h = reinterpret_cast<const uint4*>(io.rhs_h);
    a.v32 = reinterpret_cast<const float4*>(io.v32);
    a.col_scale = io.col_scale;
    a.prevh = reinterpret_cast<const uint4*>(io.prevh);
    a.yh = reinterpret_cast<uint4*>(io.yh);
    a.alpha = alpha; a.w = w; a.t = t;
    a.partials = io.partials;
    a.overflow = overflow;
    return a;
}

// One fp16 sweep (mode 0) or the residual sweep (mode 1) of n = 1 or 2 states over the owned rows.
int mixed_sweep(const PprGraph& g, int mode, const MixedSweepIO* io, int n, float alpha, float w, float t,
                int* n_partials, int* overflow, const PeerOut& peers, const SweepSync& sync, cudaStream_t st) {
    HRAG_CHECK(g.row_ptr && g.cv, "mixed_sweep: graph not loaded");
    HRAG_CHECK(kB <= g.max_batch, "mixed_sweep: segment partials too small for 32 columns");
    const bool sharded = sync.flags != nullptr;
    HRAG_CHECK(n == 1 || (n == 2 && !sharded && peers.n == 0), "mixed_sweep: the paired sweep runs on a single GPU");
    for (int k = 1; k < n; ++k)
        HRAG_CHECK((io[k].partials == nullptr) == (io[0].partials == nullptr),
                   "mixed_sweep: partials for all states or none");
    for (int k = 0; k < n; ++k)
        HRAG_CHECK(io[k].x0c == io[0].x0c && (io[k].x0c == kX0Dense || (io[k].slot_map && !sharded && mode == 0)),
                   "mixed_sweep: the compact first iterate needs a compact rhs for every state on a single GPU");
    const SweepGrid grid(g, kGPB);
    SweepSync sy = sync;
    // sharded (fused exchange): a persistent grid of 6 CTAs per SM, so each CTA pays one system-scope fence per sweep
    // and the epoch is published by the last CTA of the sweep itself, with no extra launch (see k_sweep_h_push).  The
    // staging ring is double-buffered so a block's bulk copies overlap the next block's gathers: without the second
    // buffer a CTA would sit on its slot until the TMA engine has drained its copies into a congested link.
    const int grid_rows = sharded ? std::min(grid.nb_rows, g.num_sms * 6) : grid.nb_rows;
    sy.total_ctas = (unsigned)(grid_rows + grid.nb_long);
    F8* segp = reinterpret_cast<F8*>(g.seg_partial);
    const int x0c = io[0].x0c;
    with_bools([&](auto cheb, auto resid, auto fin, auto x0x, auto x0p, auto pair) {
        // the residual (mode 1) has no Chebyshev form; sweep 1 (x0 as x) is a plain sweep, sweep 2 (x0 as prev) a
        // Chebyshev one
        if constexpr (!(cheb && resid) && !(x0x && (cheb || resid)) && !(x0p && (!cheb || resid))) {
            constexpr int NS = pair ? 2 : 1, M = resid ? 1 : 0;
            constexpr int X0C = x0x ? kX0AsX : x0p ? kX0AsPrev : kX0Dense;
            SweepArgs a[NS];
            for (int k = 0; k < NS; ++k) a[k] = sweep_args(g, io[k], alpha, w, t, overflow);
            // the long rows of state k: the single-state segment and finalize kernels on the state's rows (NS * kLPR
            // uint4 apart); seg_partial is reused in stream order.  The segment kernel only waits: it writes no
            // exchanged rows.
            auto segments = [&](int k) {
                if constexpr (X0C == kX0AsX)
                    k_sweep_long_segments_h<kLPR, RhsRows><<<grid.nb_seg, kThreads, 0, st>>>(
                        g.n_seg, g.segs, g.cv, RhsRows{a[k].slot_map, a[k].rhs_h}, segp, sy);
                else k_sweep_long_segments_h<NS * kLPR><<<grid.nb_seg, kThreads, 0, st>>>(g.n_seg, g.segs, g.cv,
                                                                                            a[k].xh, segp, sy);
                count_launch();
            };
            auto finalize = [&](int k) {
                SweepArgs al = a[k];
                al.partials = al.partials ? al.partials + (size_t)grid.nb_rows * kB : nullptr;
                k_sweep_long_finalize_h<cheb, M, fin, NS * kLPR, X0C == kX0AsPrev><<<grid.nb_long, kThreads, 0, st>>>(
                    g.n_long, g.long_rows, g.long_seg_ptr, segp, al, peers, sy);
                count_launch();
            };
            // one state: the segments first, so the finalize follows the short rows directly
            if (NS == 1 && grid.nb_long) segments(0);
            if (grid.nb_rows) {
                if (sharded) {               // one state with a dense first iterate (checked above)
                    if constexpr (NS == 1 && X0C == kX0Dense)
                        k_sweep_h_push<cheb, M, fin><<<grid_rows, kThreads, 0, st>>>(a[0], peers, sy);
                } else {
                    if constexpr (NS == 1) k_sweep_h<cheb, M, fin, X0C><<<grid_rows, kThreads, 0, st>>>(a[0]);
                    else k_sweep_h2<cheb, M, fin, X0C><<<grid_rows, kThreads, 0, st>>>(a[0], a[1]);
                }
                count_launch();
            }
            for (int k = 0; k < NS && grid.nb_long; ++k) {
                if (NS == 2) segments(k);
                finalize(k);
            }
        }
    }, mode == 0 && (io[0].prevh != nullptr || x0c == kX0AsPrev), mode == 1, io[0].partials != nullptr,
       x0c == kX0AsX, x0c == kX0AsPrev, n == 2);
    if (grid.nb_rows + grid.nb_long == 0 && sharded) HRAG_TRY(epoch_signal(sy, st));
    if (n_partials) *n_partials = grid.nb_rows + grid.nb_long;
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int mixed_prepare_rhs(const float* V32, int64_t n_rows, float alpha, float* partials, double* vsum, float* scale,
                      void* V16, cudaStream_t st) {
    const int64_t n_elems = n_rows * kB;
    const int nblk = (int)std::min<int64_t>(ceil_div(n_elems, 256), 1024);
    k_colsum32_partial<<<nblk, 256, 0, st>>>(V32, n_elems, partials);
    HRAG_TRY(colsum_reduce(partials, nblk, kB, vsum, st));
    k_scales32<<<1, kB, 0, st>>>(vsum, 1.f - alpha, scale);
    k_scale_to_half<<<(unsigned)ceil_div(n_elems / 8, 256), 256, 0, st>>>(reinterpret_cast<const float4*>(V32),
                                                                          n_elems / 8, scale,
                                                                          reinterpret_cast<uint4*>(V16));
    count_launch(3);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int slot_map_build(int N, int P, const int* passage_vid, int* slot_map, cudaStream_t st) {
    k_slot_map_init<<<(unsigned)ceil_div(N, 256), 256, 0, st>>>(N, slot_map);
    if (P) k_slot_map_passages<<<(unsigned)ceil_div(P, 256), 256, 0, st>>>(P, passage_vid, slot_map);
    count_launch(2);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int compact_rhs_partial_rows(int P) { return (int)ceil_div(std::max(P, 1), 32); }

int compact_prepare_rhs(const SeedTables& t, int nb, int q0, const float* S, int64_t ldS, const float2* minmax,
                        float pnw, int slots_per_query, const int* seed_vid, const double* seed_w, float alpha,
                        int* slot_map, int* slot_vid, float* Vc, void* rhs16, void* x0_dense, int x0_ld, int64_t n_nodes,
                        float* partials, double* vsum, float* scale, cudaStream_t st) {
    const int P = t.n_passages;
    const int n_seed_slots = kB * slots_per_query;
    HRAG_CHECK(slots_per_query > 0, "compact_prepare_rhs: slots_per_query must be positive");
    const int nblk = compact_rhs_partial_rows(P);
    if (x0_dense) {
        HRAG_CHECK(x0_ld == kB || x0_ld == 2 * kB, "compact_prepare_rhs: x0 rows are 32 or 64 halves apart");
        if (x0_ld == kB) HRAG_CUDA(cudaMemsetAsync(x0_dense, 0, (size_t)n_nodes * kB * 2, st));
        else HRAG_CUDA(cudaMemset2DAsync(x0_dense, (size_t)x0_ld * 2, 0, kB * 2, (size_t)n_nodes, st));
    }
    HRAG_CUDA(cudaMemsetAsync(Vc + (size_t)P * kB, 0, (size_t)n_seed_slots * kB * sizeof(float), st));
    k_rhs_passages<<<nblk, 256, 0, st>>>(P, nb, S, ldS, q0, minmax, pnw, Vc, partials);
    k_rhs_seeds<<<1, 1024, 0, st>>>(P, nb, q0, slots_per_query, seed_vid, seed_w, slot_map, slot_vid, Vc,
                                            partials, nblk, 1.f - alpha, vsum, scale);
    const int n_slots = P + n_seed_slots;
    k_rhs_convert<<<(unsigned)ceil_div((int64_t)n_slots * kLPR, 256), 256, 0, st>>>(
        P, n_slots, t.passage_vid, slot_vid, reinterpret_cast<const float4*>(Vc), scale,
        reinterpret_cast<uint4*>(rhs16), reinterpret_cast<uint4*>(x0_dense), x0_ld / 8);
    count_launch(3);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int compact_release_slots(int P, int nb, int q0, int slots_per_query, const int* seed_vid, int* slot_map,
                          cudaStream_t st) {
    k_slot_clear<<<1, 1024, 0, st>>>(P, nb, q0, slots_per_query, seed_vid, slot_map);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int residual_check(const double* rsum, const double* vsum, const float* scale, float inv_t, float* rho_max,
                   cudaStream_t st) {
    k_residual_check<<<1, kB, 0, st>>>(rsum, vsum, scale, inv_t, rho_max);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int gather_passage_scores_mixed(const SeedTables& t, int nb, int q0, const void* X0, const void* D, int ldx,
                                float inv_t, const double* sum0, const double* sum1, const int* mode,
                                const float2* minmax, float* S, int64_t ldS, cudaStream_t st) {
    if (t.n_passages == 0 || nb == 0) return 0;
    const int64_t total = (int64_t)t.n_passages * nb;
    k_gather_passage_scores_mixed<<<(unsigned)ceil_div(total, 256), 256, 0, st>>>(
        t.n_passages, nb, q0, t.passage_vid, reinterpret_cast<const __half*>(X0), reinterpret_cast<const __half*>(D),
        inv_t, sum0, sum1, mode, minmax, S, ldS, ldx);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int state_to_scores_mixed(const void* X0, const void* D, float inv_t, int nb, int N, const double* sum0,
                          const double* sum1, float* out, cudaStream_t st) {
    const int64_t total = (int64_t)N * nb;
    k_state_to_scores_mixed<<<(unsigned)ceil_div(total, 256), 256, 0, st>>>(
        reinterpret_cast<const __half*>(X0), reinterpret_cast<const __half*>(D), inv_t, nb, N, sum0, sum1, out);
    count_launch();
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace hrag
