// Shared helpers for libhrag_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

namespace hrag {

void set_error(const std::string& msg);

#define HRAG_CUDA(expr)                                                                   \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            ::hrag::set_error(std::string(#expr) + " -> " + cudaGetErrorString(_e) +      \
                              " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")");    \
            return 1;                                                                     \
        }                                                                                 \
    } while (0)

#define HRAG_CHECK(cond, msg)                                                             \
    do {                                                                                  \
        if (!(cond)) {                                                                    \
            ::hrag::set_error(std::string(msg) + " (" + __FILE__ + ":" +                  \
                              std::to_string(__LINE__) + ")");                            \
            return 2;                                                                     \
        }                                                                                 \
    } while (0)

#define HRAG_TRY(expr)                                                                    \
    do {                                                                                  \
        int _rc = (expr);                                                                 \
        if (_rc != 0) return _rc;                                                         \
    } while (0)

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- device helpers ---------------------------------------------------------------------
#ifdef __CUDACC__

// Monotone map float -> uint32 (larger float = larger key); -0.0 < +0.0 is harmless here.
__device__ __forceinline__ uint32_t float_to_ordered(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_float(uint32_t k) {
    uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(u);
}
// Ranking key: score descending, then index ascending  <=>  key descending.
__device__ __forceinline__ uint64_t rank_key(float score, uint32_t idx) {
    return ((uint64_t)float_to_ordered(score) << 32) | (uint64_t)(0xffffffffu - idx);
}
__device__ __forceinline__ uint32_t key_index(uint64_t key) { return 0xffffffffu - (uint32_t)key; }
__device__ __forceinline__ float key_score(uint64_t key) { return ordered_to_float((uint32_t)(key >> 32)); }

__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void f4_fma(float4& acc, float a, const float4& x) {
    acc.x = fmaf(a, x.x, acc.x);
    acc.y = fmaf(a, x.y, acc.y);
    acc.z = fmaf(a, x.z, acc.z);
    acc.w = fmaf(a, x.w, acc.w);
}
__device__ __forceinline__ void f4_add(float4& a, const float4& b) {
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
}

// Streaming (read-once) 16-byte load: ld.global.cs = evict-first, keeps L2 for the gather target.
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) { return __ldcs(p); }
#endif  // __CUDACC__

}  // namespace hrag
