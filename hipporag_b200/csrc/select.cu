// Selection kernels (sm_90a): per-query min/max + small top-k of the fact scores (the
// argsort of rerank_facts, reference HippoRAG.py:1683-1688, and min_max_normalize,
// misc_utils.py:130-139) and the exact top-k of the passage scores (the argsort + slice of
// run_ppr / _build_retrieval_result, HippoRAG.py:1746-1747, 501-507).
//
// Tie policy everywhere: score descending, then index ascending -- encoded in one 64-bit
// key (common.cuh: rank_key) so "top-k" is a total order and the result is unique.
#include "common.cuh"
#include "kernels.h"

namespace hrag {

namespace {

constexpr int kSelThreads = 256;
constexpr int kMaxSmallK = 8;
constexpr int kScreenCand = kScreenCandidates, kScreenSat = kScreenSatTiles;

__device__ __forceinline__ uint64_t shfl_xor_u64(uint64_t v, int off) {
    uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
    lo = __shfl_xor_sync(0xffffffffu, lo, off);
    hi = __shfl_xor_sync(0xffffffffu, hi, off);
    return ((uint64_t)hi << 32) | lo;
}

// One CTA per row: min, max and the K best keys.
template <int K>
__global__ void __launch_bounds__(kSelThreads)
k_row_minmax_topk(const float* __restrict__ S, int64_t M, int64_t ld, int k, float2* __restrict__ minmax,
                  int* __restrict__ top_idx, float* __restrict__ top_score, int* __restrict__ n_valid) {
    const int row = blockIdx.x;
    const float* s = S + (size_t)row * ld;
    float mn = INFINITY, mx = -INFINITY;
    uint64_t best[K > 0 ? K : 1];
#pragma unroll
    for (int j = 0; j < (K > 0 ? K : 1); ++j) best[j] = 0ull;  // 0 is below every real key
    for (int64_t i = threadIdx.x; i < M; i += kSelThreads) {
        const float f = __ldg(s + i);
        mn = fminf(mn, f);
        mx = fmaxf(mx, f);
        if (K > 0) {
            uint64_t key = rank_key(f, (uint32_t)i);
            if (key > best[K - 1]) {
#pragma unroll
                for (int j = 0; j < K; ++j) {   // sorted insertion, best[0] largest
                    if (key > best[j]) { const uint64_t t = best[j]; best[j] = key; key = t; }
                }
            }
        }
    }
    // block min / max
    __shared__ float s_mn[kSelThreads / 32], s_mx[kSelThreads / 32];
    __shared__ uint64_t s_key[kSelThreads / 32];
    __shared__ uint64_t s_pick;
    for (int off = 16; off > 0; off >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, off));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_mn[warp] = mn; s_mx[warp] = mx; }
    __syncthreads();
    mn = s_mn[0]; mx = s_mx[0];
#pragma unroll
    for (int wi = 1; wi < kSelThreads / 32; ++wi) { mn = fminf(mn, s_mn[wi]); mx = fmaxf(mx, s_mx[wi]); }
    if (threadIdx.x == 0 && minmax) minmax[row] = make_float2(mn, mx);
    if (K == 0) return;
    // k rounds of "pop the global best head"
    const float range = mx - mn;
    int head = 0;
    const int kk = (int)((int64_t)k < M ? k : M);
    for (int round = 0; round < k; ++round) {
        uint64_t cand = 0ull;
#pragma unroll
        for (int j = 0; j < K; ++j) if (j == head) cand = best[j];
        uint64_t m = cand;
        for (int off = 16; off > 0; off >>= 1) { const uint64_t o = shfl_xor_u64(m, off); m = o > m ? o : m; }
        if (lane == 0) s_key[warp] = m;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint64_t b = s_key[0];
#pragma unroll
            for (int wi = 1; wi < kSelThreads / 32; ++wi) b = s_key[wi] > b ? s_key[wi] : b;
            s_pick = b;
            if (round < kk) {
                const float f = key_score(b);
                top_idx[(size_t)row * k + round] = (int)key_index(b);
                top_score[(size_t)row * k + round] = range == 0.f ? 1.f : __fdiv_rn(f - mn, range);
            } else {
                top_idx[(size_t)row * k + round] = -1;
                top_score[(size_t)row * k + round] = 0.f;
            }
        }
        __syncthreads();
        if (cand != 0ull && cand == s_pick) ++head;   // keys are unique: exactly one thread pops
        __syncthreads();
    }
    if (threadIdx.x == 0) n_valid[row] = kk;
}

// The end of a row's merge, one CTA per row: each thread holds min / max and its K best keys of part of the row; the
// block reduces min / max into minmax[row] and pops the k best keys (K = kMaxSmallK) into top_idx / top_score
// (normalised) or raw_keys, n_valid[row] = min(k, M).
__device__ __forceinline__ void finish_minmax_topk(int row, float mn, float mx, uint64_t (&best)[kMaxSmallK], int64_t M,
                                                   int k, float2* __restrict__ minmax, int* __restrict__ top_idx,
                                                   float* __restrict__ top_score, int* __restrict__ n_valid,
                                                   uint64_t* __restrict__ raw_keys) {
    constexpr int K = kMaxSmallK;
    __shared__ float s_mn[kSelThreads / 32], s_mx[kSelThreads / 32];
    __shared__ uint64_t s_key[kSelThreads / 32];
    __shared__ uint64_t s_pick;
    for (int off = 16; off > 0; off >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, off));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_mn[warp] = mn; s_mx[warp] = mx; }
    __syncthreads();
    mn = s_mn[0]; mx = s_mx[0];
#pragma unroll
    for (int wi = 1; wi < kSelThreads / 32; ++wi) { mn = fminf(mn, s_mn[wi]); mx = fmaxf(mx, s_mx[wi]); }
    if (threadIdx.x == 0 && minmax) minmax[row] = make_float2(mn, mx);
    const float range = mx - mn;
    int head = 0;
    const int kk = (int)((int64_t)k < M ? k : M);
    for (int round = 0; round < k; ++round) {
        uint64_t cand = 0ull;
#pragma unroll
        for (int j = 0; j < K; ++j) if (j == head) cand = best[j];
        uint64_t m = cand;
        for (int off = 16; off > 0; off >>= 1) { const uint64_t o = shfl_xor_u64(m, off); m = o > m ? o : m; }
        if (lane == 0) s_key[warp] = m;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint64_t b = s_key[0];
#pragma unroll
            for (int wi = 1; wi < kSelThreads / 32; ++wi) b = s_key[wi] > b ? s_key[wi] : b;
            s_pick = b;
            if (raw_keys) {
                raw_keys[(size_t)row * k + round] = b;          // 0 when fewer than k candidates exist
            } else if (round < kk) {
                top_idx[(size_t)row * k + round] = (int)key_index(b);
                top_score[(size_t)row * k + round] = range == 0.f ? 1.f : __fdiv_rn(key_score(b) - mn, range);
            } else {
                top_idx[(size_t)row * k + round] = -1;
                top_score[(size_t)row * k + round] = 0.f;
            }
        }
        __syncthreads();
        if (cand != 0ull && cand == s_pick) ++head;
        __syncthreads();
    }
    if (threadIdx.x == 0 && n_valid) n_valid[row] = kk;
}


// Finishes the fused similarity epilogue: per query, min/max over the per-tile (min, max) pairs
// and the k best of the per-tile 8-best rank keys (every global top-8 member is in its tile's top-8).
// Strided form: tile t of row r lives at part_mm[r * row_stride + t * tile_stride] (keys: 8 per entry), so the
// same kernel merges the per-rank candidates of a fact-sharded stage A ([rank, query] layout after the all-gather).
// idx_offset is added to every key's index (local fact row -> global row); with raw_keys != null the 8 best
// keys are written raw (no normalisation) for a later cross-rank merge.  With gate != null the kernel runs only when
// *gate != 0 (the exact fallback of the stage-A screen), and then the first CTA counts it in *fallbacks.
__global__ void __launch_bounds__(kSelThreads)
k_merge_minmax_topk(const float2* __restrict__ part_mm, const uint64_t* __restrict__ part_keys, int n_tiles,
                    int64_t row_stride, int64_t tile_stride, uint32_t idx_offset, int64_t M, int k,
                    float2* __restrict__ minmax, int* __restrict__ top_idx, float* __restrict__ top_score,
                    int* __restrict__ n_valid, uint64_t* __restrict__ raw_keys, const int* __restrict__ gate,
                    unsigned long long* __restrict__ fallbacks) {
    constexpr int K = kMaxSmallK;
    const int row = blockIdx.x;
    if (gate) {
        if (*reinterpret_cast<const volatile int*>(gate) == 0) return;
        if (row == 0 && threadIdx.x == 0) atomicAdd(fallbacks, 1ull);
    }
    float mn = INFINITY, mx = -INFINITY;
    uint64_t best[K];
#pragma unroll
    for (int j = 0; j < K; ++j) best[j] = 0ull;
    for (int t = threadIdx.x; t < n_tiles; t += kSelThreads) {
        const size_t e = (size_t)row * row_stride + (size_t)t * tile_stride;
        const float2 mm = __ldg(part_mm + e);
        mn = fminf(mn, mm.x);
        mx = fmaxf(mx, mm.y);
        const uint64_t* kp = part_keys + e * K;
#pragma unroll
        for (int i = 0; i < K; ++i) {
            uint64_t key = __ldg(kp + i);
            if (key != 0ull) key -= (uint64_t)idx_offset;        // the index is stored as 0xffffffff - idx
            if (key > best[K - 1]) {
#pragma unroll
                for (int j = 0; j < K; ++j) if (key > best[j]) { const uint64_t tmp = best[j]; best[j] = key; key = tmp; }
            }
        }
    }
    finish_minmax_topk(row, mn, mx, best, M, k, minmax, top_idx, top_score, n_valid, raw_keys);
}

// ---- exact top-k (k <= 2048) of a row by rank key: MSB radix select + bitonic sort ----
// A key policy fixes the score type and how (score desc, index asc) is encoded as one unsigned key that is unique per
// element, larger = better, and never 0 (0 pads the sort).  The select walks the key 8 bits at a time from the top.
constexpr int kTopkThreads = 512;
constexpr int kTopkMax = 2048;

// fp32 scores: rank_key, the score and the index in 64 bits
struct RankKeyF32 {
    using Score = float;
    using Key = uint64_t;
    static constexpr int kBits = 64;
    static constexpr int kUnroll = 4;   // of the histogram loop (what the compiler picks unasked)
    __device__ static Key make(float s, uint32_t i) { return rank_key(s, i); }
    __device__ static uint32_t digit(Key k, int shift) { return (uint32_t)(k >> shift) & 0xffu; }
    __device__ static bool above_equal(Key k, Key prefix, int shift) {   // bits above shift + 8 agree
        const uint64_t himask = shift == 56 ? 0ull : (~0ull << (shift + 8));
        return (k & himask) == prefix;
    }
    __device__ static Key with_digit(Key prefix, uint32_t d, int shift) { return prefix | ((uint64_t)d << shift); }
    __device__ static uint32_t index(Key k) { return key_index(k); }
    __device__ static float score(Key k) { return key_score(k); }
};

// fp64 scores: an order-preserving 64-bit image of the double does not leave room for the index, so the key is 96 bits
// wide, {ordered score, 0xffffffff - index}.  The select runs 4 more passes over the index bits: ties straddling the
// cut resolve to the lower indices like any other key.
struct Key96 {
    uint64_t s;
    uint64_t i;      // 0xffffffff - index (32 bits used)
    __device__ bool operator<(const Key96& o) const { return s < o.s || (s == o.s && i < o.i); }
    __device__ bool operator>=(const Key96& o) const { return !(*this < o); }
};
struct RankKeyF64 {
    using Score = double;
    using Key = Key96;
    static constexpr int kBits = 96;
    static constexpr int kUnroll = 1;   // unrolled, the loop spills its invariants to the stack
    __device__ static Key make(double s, uint32_t i) {
        const uint64_t u = (uint64_t)__double_as_longlong(s);
        return Key96{(u >> 63) ? ~u : (u | (1ull << 63)), (uint64_t)(0xffffffffu - i)};
    }
    __device__ static uint32_t digit(Key k, int shift) {
        return shift >= 32 ? (uint32_t)(k.s >> (shift - 32)) & 0xffu : (uint32_t)(k.i >> shift) & 0xffu;
    }
    __device__ static bool above_equal(Key k, Key prefix, int shift) {
        const int top = shift + 8;
        if (top >= 96) return true;
        if (top >= 32) return (k.s >> (top - 32)) == (prefix.s >> (top - 32));
        return k.s == prefix.s && (k.i >> top) == (prefix.i >> top);
    }
    __device__ static Key with_digit(Key p, uint32_t d, int shift) {
        if (shift >= 32) p.s |= (uint64_t)d << (shift - 32);
        else p.i |= (uint64_t)d << shift;
        return p;
    }
    __device__ static uint32_t index(Key k) { return 0xffffffffu - (uint32_t)k.i; }
    __device__ static double score(Key k) {
        const uint64_t u = (k.s >> 63) ? (k.s & ~(1ull << 63)) : ~k.s;
        return __longlong_as_double((long long)u);
    }
};

template <class Pol>
__global__ void __launch_bounds__(kTopkThreads)
k_row_topk(const typename Pol::Score* __restrict__ S, int64_t M, int64_t ld, int k, int* __restrict__ out_ids,
           typename Pol::Score* __restrict__ out_scores) {
    using Key = typename Pol::Key;
    __shared__ unsigned int hist[256];
    __shared__ Key s_prefix;
    __shared__ int s_need;
    __shared__ int s_count;
    __shared__ Key keys[kTopkMax];
    const int row = blockIdx.x;
    const typename Pol::Score* s = S + (size_t)row * ld;
    const int kk = (int)((int64_t)k < M ? k : M);   // number of real results
    int k2 = 1;
    while (k2 < k) k2 <<= 1;
    for (int i = threadIdx.x; i < k2; i += kTopkThreads) keys[i] = Key{};
    if (threadIdx.x == 0) { s_prefix = Key{}; s_need = kk; s_count = 0; }
    __syncthreads();
    if (kk > 0) {
        // find the kk-th largest key, 8 bits at a time from the top
        for (int shift = Pol::kBits - 8; shift >= 0; shift -= 8) {
            for (int i = threadIdx.x; i < 256; i += kTopkThreads) hist[i] = 0u;
            __syncthreads();
            const Key prefix = s_prefix;
#pragma unroll Pol::kUnroll
            for (int64_t i = threadIdx.x; i < M; i += kTopkThreads) {
                const Key key = Pol::make(__ldg(s + i), (uint32_t)i);
                if (Pol::above_equal(key, prefix, shift)) atomicAdd(&hist[Pol::digit(key, shift)], 1u);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                int need = s_need;
                int d = 255;
                for (; d > 0; --d) {
                    if ((int)hist[d] >= need) break;
                    need -= (int)hist[d];
                }
                s_prefix = Pol::with_digit(prefix, (uint32_t)d, shift);
                s_need = need;
            }
            __syncthreads();
        }
        const Key kth = s_prefix;   // keys are unique, so exactly kk keys are >= kth
        for (int64_t i = threadIdx.x; i < M; i += kTopkThreads) {
            const Key key = Pol::make(__ldg(s + i), (uint32_t)i);
            if (key >= kth) {
                const int pos = atomicAdd(&s_count, 1);
                if (pos < kTopkMax) keys[pos] = key;
            }
        }
        __syncthreads();
        // bitonic sort, descending
        for (int size = 2; size <= k2; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int i = threadIdx.x; i < k2 / 2; i += kTopkThreads) {
                    const int lo = 2 * i - (i & (stride - 1));
                    const int hi = lo + stride;
                    const bool desc = (lo & size) == 0;
                    const Key a = keys[lo], b = keys[hi];
                    if ((a < b) == desc) { keys[lo] = b; keys[hi] = a; }
                }
                __syncthreads();
            }
        }
    }
    for (int i = threadIdx.x; i < k; i += kTopkThreads) {
        if (i < kk) {
            out_ids[(size_t)row * k + i] = (int)Pol::index(keys[i]);
            out_scores[(size_t)row * k + i] = Pol::score(keys[i]);
        } else {
            out_ids[(size_t)row * k + i] = -1;
            out_scores[(size_t)row * k + i] = 0;
        }
    }
}

// S[row, i] <- (S[row, i] - min) / (max - min)   (all-equal -> 1), misc_utils.py:130-139
__global__ void __launch_bounds__(256)
k_minmax_apply(float* __restrict__ S, int64_t M, int64_t ld, const float2* __restrict__ minmax) {
    const int row = blockIdx.y;
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= M) return;
    const float2 mm = __ldg(minmax + row);
    const float range = mm.y - mm.x;
    float* p = S + (size_t)row * ld + i;
    *p = range == 0.f ? 1.f : __fdiv_rn(*p - mm.x, range);
}

// Finishes the threshold epilogue of the similarity GEMM: sorts each query's candidate keys (score desc, row asc)
// and writes the first kmax as (id, score); n_found[row] = candidates that cleared the threshold (may exceed cap:
// the caller then re-runs that query through the exact path).
constexpr int kCandCap = 512;
__global__ void __launch_bounds__(256)
k_sort_candidates(const uint64_t* __restrict__ cand_keys, const int* __restrict__ cand_count, int cap, int kmax,
                  int* __restrict__ out_ids, float* __restrict__ out_scores, int* __restrict__ n_found) {
    __shared__ uint64_t keys[kCandCap];
    const int row = blockIdx.x;
    const int cnt = cand_count[row];
    const int n = cnt < cap ? cnt : cap;
    for (int i = threadIdx.x; i < kCandCap; i += 256) keys[i] = i < n ? cand_keys[(size_t)row * cap + i] : 0ull;
    __syncthreads();
    for (int size = 2; size <= kCandCap; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = threadIdx.x; i < kCandCap / 2; i += 256) {
                const int lo = 2 * i - (i & (stride - 1));
                const int hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const uint64_t a = keys[lo], b = keys[hi];
                if ((a < b) == desc) { keys[lo] = b; keys[hi] = a; }
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < kmax; i += 256) {
        const bool ok = i < n;
        out_ids[(size_t)row * kmax + i] = ok ? (int)key_index(keys[i]) : -1;
        out_scores[(size_t)row * kmax + i] = ok ? key_score(keys[i]) : 0.f;
    }
    if (threadIdx.x == 0) n_found[row] = cnt;
}

// after row_topk on raw scores: min-max-normalise the k winners of each row (all-equal -> 1) and report how many
// are real (rerank_facts with linking_top_k > 8, HippoRAG.py:1683-1688)
__global__ void __launch_bounds__(256)
k_topk_normalize(int rows, int k, int64_t M, const float2* __restrict__ minmax, const int* __restrict__ ids,
                 float* __restrict__ scores, int* __restrict__ n_valid) {
    const int t = blockIdx.x * 256 + threadIdx.x;
    const int row = t / k, j = t % k;
    if (row >= rows) return;
    const float2 mm = __ldg(minmax + row);
    const float range = mm.y - mm.x;
    if (ids[t] >= 0) scores[t] = range == 0.f ? 1.f : __fdiv_rn(scores[t] - mm.x, range);
    if (j == 0) n_valid[row] = (int)((int64_t)k < M ? k : M);
}

// One thread per row: merges the running k best with a later slice's k best by rank key.  Both lists are sorted by
// rank key, so one pass of two cursors picks the k best; an equal score resolves to the lower global row, which is
// the running list's since every slice row follows the rows folded before it.
constexpr int kFoldMaxK = 32;
__global__ void __launch_bounds__(128)
k_fold_topk(int rows, int k, uint32_t idx_offset, const int* __restrict__ slice_ids,
            const float* __restrict__ slice_scores, const float2* __restrict__ slice_mm, int* run_ids,
            float* run_scores, float2* run_mm, int first) {
    const int row = blockIdx.x * 128 + threadIdx.x;
    if (row >= rows) return;
    const size_t base = (size_t)row * k;
    uint64_t a[kFoldMaxK], b[kFoldMaxK];   // running, slice (0 = none)
    for (int j = 0; j < k; ++j) {
        const int ia = first ? -1 : run_ids[base + j];
        const int ib = slice_ids[base + j];
        a[j] = ia >= 0 ? rank_key(run_scores[base + j], (uint32_t)ia) : 0ull;
        b[j] = ib >= 0 ? rank_key(slice_scores[base + j], (uint32_t)ib + idx_offset) : 0ull;
    }
    int i = 0, j = 0;
    for (int o = 0; o < k; ++o) {
        const uint64_t ka = i < k ? a[i] : 0ull, kb = j < k ? b[j] : 0ull;
        const uint64_t pick = ka >= kb ? ka : kb;
        if (ka >= kb) ++i; else ++j;
        run_ids[base + o] = pick ? (int)key_index(pick) : -1;
        run_scores[base + o] = pick ? key_score(pick) : 0.f;
    }
    const float2 s = slice_mm[row];
    if (first) {
        run_mm[row] = s;
    } else {
        const float2 r = run_mm[row];
        run_mm[row] = make_float2(fminf(r.x, s.x), fmaxf(r.y, s.y));
    }
}


// ---- stage-A screen (DESIGN.md section 4, the K2 screen): candidates from the s1 = hi.hi tile lists, staged per
// 128-query m-tile, rescored by the split K2 and selected exactly.  Any case the screen cannot prove sets *flag; the
// chunk then reruns the exact path (gated kernels).
__device__ __forceinline__ void raise_flag(int* flag) { atomicExch(flag, 1); }

// One CTA per query: L = the 8th best s1 key over the tile lists, U = the smallest s1; every listed key with
// s1 >= L - 2 E_q and every kept low entry with s1 <= U + 2 E_q is a candidate.  A tile whose list is full with its 8th
// key in the band, or whose second smallest is in the band, may have dropped band members: it is saturated (all its
// rows become candidates).
__global__ void __launch_bounds__(kSelThreads)
k_screen_select(const uint64_t* __restrict__ part_keys, const uint4* __restrict__ part_low, int n_tiles,
                const float* __restrict__ err, int* __restrict__ cand_ids, float* __restrict__ cand_s1,
                int* __restrict__ cand_n, int* __restrict__ sat, int* __restrict__ sat_n, int* flag) {
    constexpr int K = kMaxSmallK;
    const int row = blockIdx.x;
    const float E = err[row];
    if (!(E <= 3.0e38f)) {   // a non-finite bound: NaN / inf in the query or the fact planes
        if (threadIdx.x == 0) { cand_n[row] = 0; sat_n[row] = 0; raise_flag(flag); }
        return;
    }
    const uint64_t* kp_row = part_keys + (size_t)row * n_tiles * K;
    const uint4* lo_row = part_low + (size_t)row * n_tiles;
    uint64_t best[K];
#pragma unroll
    for (int j = 0; j < K; ++j) best[j] = 0ull;
    float U = INFINITY;
    for (int t = threadIdx.x; t < n_tiles; t += kSelThreads) {
        U = fminf(U, __uint_as_float(__ldg(&lo_row[t].x)));
#pragma unroll
        for (int i = 0; i < K; ++i) {
            uint64_t key = __ldg(kp_row + (size_t)t * K + i);
            if (key > best[K - 1]) {
#pragma unroll
                for (int j = 0; j < K; ++j) if (key > best[j]) { const uint64_t tmp = best[j]; best[j] = key; key = tmp; }
            }
        }
    }
    __shared__ float s_u[kSelThreads / 32];
    __shared__ uint64_t s_key[kSelThreads / 32];
    __shared__ uint64_t s_pick;
    __shared__ int s_n, s_nsat;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int off = 16; off > 0; off >>= 1) U = fminf(U, __shfl_xor_sync(0xffffffffu, U, off));
    if (lane == 0) s_u[warp] = U;
    if (threadIdx.x == 0) { s_n = 0; s_nsat = 0; }
    __syncthreads();
    U = s_u[0];
#pragma unroll
    for (int wi = 1; wi < kSelThreads / 32; ++wi) U = fminf(U, s_u[wi]);
    int head = 0;
    uint64_t L = 0ull;
    for (int round = 0; round < K; ++round) {
        uint64_t cand = 0ull;
#pragma unroll
        for (int j = 0; j < K; ++j) if (j == head) cand = best[j];
        uint64_t m = cand;
        for (int off = 16; off > 0; off >>= 1) { const uint64_t o = shfl_xor_u64(m, off); m = o > m ? o : m; }
        if (lane == 0) s_key[warp] = m;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint64_t b = s_key[0];
#pragma unroll
            for (int wi = 1; wi < kSelThreads / 32; ++wi) b = s_key[wi] > b ? s_key[wi] : b;
            s_pick = b;
        }
        __syncthreads();
        L = s_pick;
        if (cand != 0ull && cand == s_pick) ++head;
        __syncthreads();
    }
    // fewer than 8 keys in all (F < 8): no threshold, and no list is full
    const float band_lo = L ? __fsub_rd(key_score(L), 2.f * E) : -INFINITY;
    const float band_hi = __fadd_ru(U, 2.f * E);
    auto push = [&](uint32_t id, float s1) {
        const int pos = atomicAdd(&s_n, 1);
        if (pos < kScreenCand) {
            cand_ids[(size_t)row * kScreenCand + pos] = (int)id;
            cand_s1[(size_t)row * kScreenCand + pos] = s1;
        }
    };
    for (int t = threadIdx.x; t < n_tiles; t += kSelThreads) {
        const uint64_t* kp = kp_row + (size_t)t * K;
        bool saturated = false;
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const uint64_t key = __ldg(kp + i);
            if (key != 0ull && key_score(key) >= band_lo) {
                push(key_index(key), key_score(key));
                if (i == K - 1) saturated = true;   // a full list whose last key is in the band
            }
        }
        const uint4 lo = __ldg(lo_row + t);
        if (lo.y != 0xffffffffu && __uint_as_float(lo.x) <= band_hi) push(lo.y, __uint_as_float(lo.x));
        if (lo.w != 0xffffffffu && __uint_as_float(lo.z) <= band_hi) {
            push(lo.w, __uint_as_float(lo.z));
            saturated = true;
        }
        if (saturated) {
            const int pos = atomicAdd(&s_nsat, 1);
            if (pos < kScreenSat) sat[(size_t)row * kScreenSat + pos] = t;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        cand_n[row] = min(s_n, kScreenCand);
        sat_n[row] = min(s_nsat, kScreenSat);
        if (s_n > kScreenCand || s_nsat > kScreenSat) raise_flag(flag);
    }
}

// One CTA per query: every candidate row (listed, or in a saturated tile) of the query's m-tile mt = row / 128 gets
// one slot, claimed through pos_of[mt, f] (-1 = none, set by the caller): f goes to column f mod 256 of the m-tile's
// first staged tile whose column is free.  pos_of then holds f's staged column, j * 256 + f mod 256.
__global__ void __launch_bounds__(kSelThreads)
k_screen_stage(const int* __restrict__ cand_ids, const int* __restrict__ cand_n, const int* __restrict__ sat,
               const int* __restrict__ sat_n, int64_t F, int stage_tiles, int* __restrict__ pos_of,
               int* __restrict__ slot_ids, int* __restrict__ res_count, int* __restrict__ stage_count, int* flag) {
    const int row = blockIdx.x, mt = row / 128;
    int* pos = pos_of + (size_t)mt * F;
    auto claim = [&](int64_t f) {
        if (atomicCAS(pos + f, -1, -2) != -1) return;
        const int c = (int)(f & 255);
        const int j = atomicAdd(res_count + mt * 256 + c, 1);
        if (j >= stage_tiles) { raise_flag(flag); return; }
        slot_ids[((size_t)mt * stage_tiles + j) * 256 + c] = (int)f;
        pos[f] = j * 256 + c;
        atomicMax(stage_count + mt, j + 1);
    };
    const int n = cand_n[row];
    for (int i = threadIdx.x; i < n; i += kSelThreads) claim(cand_ids[(size_t)row * kScreenCand + i]);
    const int ns = sat_n[row];
    for (int s = 0; s < ns; ++s)
        for (int c = threadIdx.x; c < 256; c += kSelThreads) {   // the tile's 256 rows
            const int64_t f = (int64_t)sat[(size_t)row * kScreenSat + s] * 256 + c;
            if (f < F) claim(f);
        }
}

// One warp per staged slot of a live staged tile: its fact's hi / lo rows (zeros for an empty slot) into the staging
// planes, row (mt * stage_tiles + j) * 256 + c
__global__ void __launch_bounds__(256)
k_screen_gather(const int* __restrict__ slot_ids, const int* __restrict__ stage_count, int stage_tiles,
                const uint4* __restrict__ e_hi, const uint4* __restrict__ e_lo, int dim, uint4* __restrict__ st_hi,
                uint4* __restrict__ st_lo) {
    const int slot = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, mt = blockIdx.y;
    if (slot / 256 >= __ldg(stage_count + mt)) return;
    const size_t r = (size_t)mt * stage_tiles * 256 + slot;
    const int id = __ldg(slot_ids + r);
    const int n16 = dim / 8;
    for (int i = lane; i < n16; i += 32) {
        st_hi[r * n16 + i] = id >= 0 ? __ldg(e_hi + (size_t)id * n16 + i) : make_uint4(0u, 0u, 0u, 0u);
        st_lo[r * n16 + i] = id >= 0 ? __ldg(e_lo + (size_t)id * n16 + i) : make_uint4(0u, 0u, 0u, 0u);
    }
}

// 16 bytes of host memory through a plain global load: the mapped lo plane is read over PCIe, where a non-coherent
// (texture-path) load has nothing to gain
__device__ __forceinline__ uint4 ld_global_u4(const uint4* p) {
    uint4 v;
    asm("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

// k_screen_gather with the lo rows read from the mapped pinned lo plane (HRAG_FACT_LO_ON_HOST): one warp per staged
// slot, zeros for an empty slot, the hi row from the resident plane.  A lane issues all of its 16-byte loads of a lo
// row (up to 8 at a time: dim <= 2048 in one round) before it stores them, so every warp keeps a whole row in flight over PCIe
// (64 warps per SM: about 100 KB per SM at dim 768).  *lo_bytes counts the lo bytes read, once per CTA.
constexpr int kGatherInFlight = 8;
__global__ void __launch_bounds__(256)
k_screen_gather_mapped(const int* __restrict__ slot_ids, const int* __restrict__ stage_count, int stage_tiles,
                       const uint4* __restrict__ e_hi, const uint4* e_lo, int dim, uint4* __restrict__ st_hi,
                       uint4* __restrict__ st_lo, unsigned long long* __restrict__ lo_bytes) {
    __shared__ int s_rows;
    const int slot = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, mt = blockIdx.y;
    if (threadIdx.x == 0) s_rows = 0;
    __syncthreads();
    if (slot / 256 < __ldg(stage_count + mt)) {
        const size_t r = (size_t)mt * stage_tiles * 256 + slot;
        const int id = __ldg(slot_ids + r);
        const int n16 = dim / 8;
        if (id < 0) {
            for (int i = lane; i < n16; i += 32) st_hi[r * n16 + i] = st_lo[r * n16 + i] = make_uint4(0u, 0u, 0u, 0u);
        } else {
            const uint4* src = e_lo + (size_t)id * n16;
            for (int i0 = lane; i0 < n16; i0 += 32 * kGatherInFlight) {
                uint4 v[kGatherInFlight];
#pragma unroll
                for (int j = 0; j < kGatherInFlight; ++j)
                    if (i0 + 32 * j < n16) v[j] = ld_global_u4(src + i0 + 32 * j);
#pragma unroll
                for (int j = 0; j < kGatherInFlight; ++j)
                    if (i0 + 32 * j < n16) st_lo[r * n16 + i0 + 32 * j] = v[j];
            }
            for (int i = lane; i < n16; i += 32) st_hi[r * n16 + i] = __ldg(e_hi + (size_t)id * n16 + i);
            if (lane == 0) atomicAdd(&s_rows, 1);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_rows) atomicAdd(lo_bytes, (unsigned long long)s_rows * dim * 2);
}

// One CTA per query: the exact min / max and k best over the rescored staged columns of its m-tile (every candidate
// is there, with the bits K2 gives it), after checking |s4 - s1| <= E_q on each listed candidate.
__global__ void __launch_bounds__(kSelThreads)
k_screen_finish(const float* __restrict__ S, int stage_tiles, const int* __restrict__ slot_ids,
                const int* __restrict__ stage_count, const int* __restrict__ pos_of, int64_t F,
                const int* __restrict__ cand_ids, const float* __restrict__ cand_s1, const int* __restrict__ cand_n,
                const float* __restrict__ err, int k, float2* __restrict__ minmax, int* __restrict__ top_idx,
                float* __restrict__ top_score, int* __restrict__ n_valid, int* flag) {
    constexpr int K = kMaxSmallK;
    const int row = blockIdx.x, mt = row / 128;
    const int64_t ld = (int64_t)stage_tiles * 256;
    const float* s = S + (size_t)row * ld;
    const int* ids = slot_ids + (size_t)mt * ld;
    const int cols = __ldg(stage_count + mt) * 256;
    float mn = INFINITY, mx = -INFINITY;
    uint64_t best[K];
#pragma unroll
    for (int j = 0; j < K; ++j) best[j] = 0ull;
    for (int c = threadIdx.x; c < cols; c += kSelThreads) {
        const int id = __ldg(ids + c);
        if (id < 0) continue;
        const float f = __ldg(s + c);
        mn = fminf(mn, f);
        mx = fmaxf(mx, f);
        uint64_t key = rank_key(f, (uint32_t)id);
        if (key > best[K - 1]) {
#pragma unroll
            for (int j = 0; j < K; ++j) if (key > best[j]) { const uint64_t tmp = best[j]; best[j] = key; key = tmp; }
        }
    }
    const float E = err[row];
    const int* pos = pos_of + (size_t)mt * F;
    const int n = cand_n[row];
    for (int i = threadIdx.x; i < n; i += kSelThreads) {
        const int p = pos[cand_ids[(size_t)row * kScreenCand + i]];
        if (p < 0 || !(fabsf(s[p] - cand_s1[(size_t)row * kScreenCand + i]) <= E)) raise_flag(flag);
    }
    finish_minmax_topk(row, mn, mx, best, F, k, minmax, top_idx, top_score, n_valid, nullptr);
}

}  // namespace

int screen_select(const uint64_t* part_keys, const uint4* part_low, int rows, int n_tiles, const float* err,
                  int* cand_ids, float* cand_s1, int* cand_n, int* sat, int* sat_n, int* flag, cudaStream_t stream) {
    if (rows == 0) return 0;
    k_screen_select<<<rows, kSelThreads, 0, stream>>>(part_keys, part_low, n_tiles, err, cand_ids, cand_s1, cand_n,
                                                      sat, sat_n, flag);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int screen_stage(const int* cand_ids, const int* cand_n, const int* sat, const int* sat_n, int rows, int64_t F,
                 int stage_tiles, int* pos_of, int* slot_ids, int* res_count, int* stage_count, int* flag,
                 cudaStream_t stream) {
    if (rows == 0) return 0;
    k_screen_stage<<<rows, kSelThreads, 0, stream>>>(cand_ids, cand_n, sat, sat_n, F, stage_tiles, pos_of, slot_ids,
                                                     res_count, stage_count, flag);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int screen_gather(const int* slot_ids, const int* stage_count, int m_tiles, int stage_tiles, const void* e_hi,
                  const void* e_lo, int dim, void* st_hi, void* st_lo, cudaStream_t stream) {
    HRAG_CHECK(dim % 8 == 0, "screen_gather: dim must be a multiple of 8");
    if (m_tiles == 0) return 0;
    k_screen_gather<<<dim3((unsigned)(stage_tiles * 256 / 8), (unsigned)m_tiles), 256, 0, stream>>>(
        slot_ids, stage_count, stage_tiles, static_cast<const uint4*>(e_hi), static_cast<const uint4*>(e_lo), dim,
        static_cast<uint4*>(st_hi), static_cast<uint4*>(st_lo));
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int screen_gather_mapped(const int* slot_ids, const int* stage_count, int m_tiles, int stage_tiles, const void* e_hi,
                         const void* lo_mapped, int dim, void* st_hi, void* st_lo, unsigned long long* lo_bytes,
                         cudaStream_t stream) {
    HRAG_CHECK(dim % 8 == 0, "screen_gather_mapped: dim must be a multiple of 8");
    if (m_tiles == 0) return 0;
    k_screen_gather_mapped<<<dim3((unsigned)(stage_tiles * 256 / 8), (unsigned)m_tiles), 256, 0, stream>>>(
        slot_ids, stage_count, stage_tiles, static_cast<const uint4*>(e_hi), static_cast<const uint4*>(lo_mapped),
        dim, static_cast<uint4*>(st_hi), static_cast<uint4*>(st_lo), lo_bytes);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int screen_finish(const float* S, int rows, int stage_tiles, const int* slot_ids, const int* stage_count,
                  const int* pos_of, int64_t F, const int* cand_ids, const float* cand_s1, const int* cand_n,
                  const float* err, int k, float2* minmax, int* top_idx, float* top_score, int* n_valid, int* flag,
                  cudaStream_t stream) {
    HRAG_CHECK(k >= 1 && k <= kMaxSmallK, "screen_finish: k must be in [1, 8]");
    if (rows == 0) return 0;
    k_screen_finish<<<rows, kSelThreads, 0, stream>>>(S, stage_tiles, slot_ids, stage_count, pos_of, F, cand_ids,
                                                      cand_s1, cand_n, err, k, minmax, top_idx, top_score, n_valid,
                                                      flag);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int fold_topk(int rows, int k, int64_t idx_offset, const int* slice_ids, const float* slice_scores,
              const float2* slice_mm, int* run_ids, float* run_scores, float2* run_mm, int first, cudaStream_t stream) {
    HRAG_CHECK(k >= 1 && k <= kFoldMaxK, "fold_topk: k must be in [1, 32]");
    HRAG_CHECK(idx_offset >= 0 && idx_offset < (int64_t)0xffffffff, "fold_topk: bad index offset");
    if (rows == 0) return 0;
    k_fold_topk<<<(unsigned)ceil_div((int64_t)rows, 128), 128, 0, stream>>>(rows, k, (uint32_t)idx_offset, slice_ids,
                                                                            slice_scores, slice_mm, run_ids,
                                                                            run_scores, run_mm, first);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int sort_candidates(const uint64_t* cand_keys, const int* cand_count, int rows, int cap, int kmax, int* out_ids,
                    float* out_scores, int* n_found, cudaStream_t stream) {
    HRAG_CHECK(cap == kCandCap && kmax >= 1 && kmax <= kCandCap, "sort_candidates: cap must be 512 and kmax in [1, 512]");
    if (rows == 0) return 0;
    k_sort_candidates<<<rows, 256, 0, stream>>>(cand_keys, cand_count, cap, kmax, out_ids, out_scores, n_found);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int topk_normalize(int rows, int k, int64_t M, const float2* minmax, const int* ids, float* scores, int* n_valid,
                   cudaStream_t stream) {
    if (rows == 0) return 0;
    k_topk_normalize<<<(unsigned)ceil_div((int64_t)rows * k, 256), 256, 0, stream>>>(rows, k, M, minmax, ids, scores,
                                                                                      n_valid);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int minmax_apply(float* S, int rows, int64_t M, int64_t ld, const float2* minmax, cudaStream_t stream) {
    if (rows == 0 || M == 0) return 0;
    dim3 grid((unsigned)ceil_div(M, 256), (unsigned)rows);
    k_minmax_apply<<<grid, 256, 0, stream>>>(S, M, ld, minmax);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int row_minmax_topk(const float* S, int rows, int64_t M, int64_t ld, int k, float2* minmax, int* top_idx,
                    float* top_score, int* n_valid, cudaStream_t stream) {
    HRAG_CHECK(k >= 0 && k <= kMaxSmallK, "row_minmax_topk: k must be in [0, 8]");
    HRAG_CHECK(M > 0 && M < (int64_t)0xffffffff, "row_minmax_topk: bad column count");
    if (rows == 0) return 0;
    if (k == 0)
        k_row_minmax_topk<0><<<rows, kSelThreads, 0, stream>>>(S, M, ld, 0, minmax, nullptr, nullptr, nullptr);
    else
        k_row_minmax_topk<kMaxSmallK><<<rows, kSelThreads, 0, stream>>>(S, M, ld, k, minmax, top_idx, top_score,
                                                                        n_valid);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int merge_minmax_topk(const float2* part_mm, const uint64_t* part_keys, int rows, int n_tiles, int64_t M, int k,
                      float2* minmax, int* top_idx, float* top_score, int* n_valid, cudaStream_t stream) {
    return merge_minmax_topk_ex(part_mm, part_keys, rows, n_tiles, n_tiles, 1, 0, M, k, minmax, top_idx, top_score,
                                n_valid, nullptr, stream);
}

int merge_minmax_topk_gated(const float2* part_mm, const uint64_t* part_keys, int rows, int n_tiles, int64_t M, int k,
                            float2* minmax, int* top_idx, float* top_score, int* n_valid, const int* gate,
                            unsigned long long* fallbacks, cudaStream_t stream) {
    HRAG_CHECK(k >= 1 && k <= kMaxSmallK, "merge_minmax_topk: k must be in [1, 8]");
    if (rows == 0) return 0;
    k_merge_minmax_topk<<<rows, kSelThreads, 0, stream>>>(part_mm, part_keys, n_tiles, n_tiles, 1, 0u, M, k, minmax,
                                                          top_idx, top_score, n_valid, nullptr, gate, fallbacks);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int merge_minmax_topk_ex(const float2* part_mm, const uint64_t* part_keys, int rows, int n_tiles, int64_t row_stride,
                         int64_t tile_stride, int64_t idx_offset, int64_t M, int k, float2* minmax, int* top_idx,
                         float* top_score, int* n_valid, uint64_t* raw_keys, cudaStream_t stream) {
    HRAG_CHECK(k >= 1 && k <= kMaxSmallK, "merge_minmax_topk: k must be in [1, 8]");
    HRAG_CHECK(idx_offset >= 0 && idx_offset < (int64_t)0xffffffff, "merge_minmax_topk: bad index offset");
    if (rows == 0) return 0;
    k_merge_minmax_topk<<<rows, kSelThreads, 0, stream>>>(part_mm, part_keys, n_tiles, row_stride, tile_stride,
                                                          (uint32_t)idx_offset, M, k, minmax, top_idx, top_score,
                                                          n_valid, raw_keys, nullptr, nullptr);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

template <class Pol>
static int launch_row_topk(const typename Pol::Score* S, int rows, int64_t M, int64_t ld, int k, int* out_ids,
                           typename Pol::Score* out_scores, cudaStream_t stream) {
    HRAG_CHECK(k >= 1 && k <= kTopkMax, "row_topk: k must be in [1, 2048]");
    HRAG_CHECK(M > 0 && M < (int64_t)0xffffffff, "row_topk: bad column count");
    if (rows == 0) return 0;
    k_row_topk<Pol><<<rows, kTopkThreads, 0, stream>>>(S, M, ld, k, out_ids, out_scores);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int row_topk(const float* S, int rows, int64_t M, int64_t ld, int k, int* out_ids, float* out_scores,
             cudaStream_t stream) {
    return launch_row_topk<RankKeyF32>(S, rows, M, ld, k, out_ids, out_scores, stream);
}

int row_topk(const double* S, int rows, int64_t M, int64_t ld, int k, int* out_ids, double* out_scores,
             cudaStream_t stream) {
    return launch_row_topk<RankKeyF64>(S, rows, M, ld, k, out_ids, out_scores, stream);
}

}  // namespace hrag
