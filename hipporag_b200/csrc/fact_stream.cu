// Fact matrices larger than the device budget of hrag_set_fact_memory: the bf16 hi / lo fact planes live in pinned
// host memory and stream through a device ring of two slices while stage A runs.  A copy stream fills one half of the
// ring with slice s + 1 while the similarity GEMM (K2, unchanged) reads slice s from the other half; events order the
// two.  One call streams the planes once for all of its queries: slices are the outer loop, query chunks the inner.
//
// Results are bit for bit those of the resident planes: K2's accumulator for a (query, fact) pair does not depend on
// the tile the fact falls in, and a slice starts on a 256-row tile boundary.  The fused top-8 path merges each slice's
// per-tile lists with the slice's first row as index offset and folds the per-slice lists into a running one with the
// same kernel the fact-sharded stage A uses across ranks (merge_minmax_topk_ex); the materialised path (k > 8, or
// hrag_debug_keep_scores) takes each slice's exact top-k and (min, max) and folds them with fold_topk (select.cu).
//
// The ring walker (stream_slices, handle.h) and the fill (planes_fill) take any plane set (HostPlanes): the synonymy
// KNN index streams its planes through them too when they exceed the hrag_knn_set_memory budget (knn_index.cu).
//
// HRAG_FACT_LO_ON_HOST keeps the hi plane resident and only the lo plane here, mapped (DESIGN.md section 7h).  Stage A
// then runs the stage-A screen per query chunk (api.cu screened_stage_a): the hi.hi screen over the resident hi plane,
// the staged candidates' lo rows read from the mapped plane by the gather.  One flag per chunk; after the call's
// chunks the flags are read at once and a flagged chunk reruns the split K2 with hi in place and lo streamed through
// the lo-only ring.  The routes that need every lo row stream the lo plane only (stream_slices' lo-only form).
#include <algorithm>
#include <cstring>
#include <vector>

#include "handle.h"

namespace hrag {

int split_queries(hrag_t* h, const float* dQ, int Bq, cudaStream_t s);   // api.cu
int64_t pad4(int64_t x);                                                  // api.cu

namespace {

constexpr int64_t kSliceAlign = 256;                // K2's tile width: every slice boundary is a tile boundary
constexpr int kPassChunk = 1024;                     // queries per K2 launch, as in the resident fused stage A
constexpr size_t kPassSplitBytes = size_t(256) << 20;   // bound on one pass's query splits (bf16 hi + lo)
constexpr int kFusedK = 8;                           // the fused epilogue's list length

const char* kNoFp32 = "similarity: the fact planes are held in host memory (hrag_set_fact_memory) and no fp32 copy "
                      "of the fact rows is kept; only the tensor-core modes are available";

}  // namespace

int HostPlanes::alloc(size_t bytes, int64_t slice, int dim, bool lo_only) {
    release();
    if (lo_only) {
        HRAG_CUDA(cudaHostAlloc(&lo, bytes, cudaHostAllocMapped));
        HRAG_CUDA(cudaHostGetDevicePointer(&lo_dev, lo, 0));
    } else {
        HRAG_CUDA(cudaHostAlloc(&hi, bytes, cudaHostAllocDefault));
        HRAG_CUDA(cudaHostAlloc(&lo, bytes, cudaHostAllocDefault));
    }
    plane_bytes = bytes;
    slice_rows = slice;
    HRAG_TRY(ring.ensure((size_t)2 * slice * dim * (lo_only ? 2 : 4)));
    HRAG_CUDA(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
        HRAG_CUDA(cudaEventCreateWithFlags(&loaded[i], cudaEventDisableTiming));
        HRAG_CUDA(cudaEventCreateWithFlags(&freed[i], cudaEventDisableTiming));
    }
    return 0;
}

void HostPlanes::release() {
    if (copy) cudaStreamSynchronize(copy);
    if (hi) cudaFreeHost(hi);
    if (lo) cudaFreeHost(lo);
    hi = lo = lo_dev = nullptr;
    plane_bytes = 0;
    slice_rows = 0;
    ring.reset();
    for (int i = 0; i < 2; ++i) {
        if (loaded[i]) cudaEventDestroy(loaded[i]);
        if (freed[i]) cudaEventDestroy(freed[i]);
        loaded[i] = freed[i] = nullptr;
    }
    if (copy) cudaStreamDestroy(copy);
    copy = nullptr;
}

void FactPlanes::release() {
    HostPlanes::release();
    run_mm.reset();
    run_keys.reset();
    sl_ids.reset();
    sl_scores.reset();
    sl_mm.reset();
    tail.reset();
}

int host_planes_plan(int64_t budget, const std::string& who, const char* setter, int64_t rows, int dim,
                     int64_t* slice_rows) {
    *slice_rows = 0;
    const int64_t plane_bytes = rows * (int64_t)dim * 4;   // hi + lo
    if (budget <= 0 || plane_bytes <= budget) return 0;
    const int64_t slice = budget / (2 * (int64_t)dim * 4) / kSliceAlign * kSliceAlign;
    HRAG_CHECK(slice >= kSliceAlign,
               who + ": " + setter + " budget of " + std::to_string(budget) + " bytes is below the " +
                   std::to_string(2 * kSliceAlign * dim * 4) + " bytes of a ring of two 256-row slices at dim " +
                   std::to_string(dim));
    *slice_rows = slice;
    return 0;
}

int fact_planes_plan(const hrag_t* h, const std::string& who, int64_t rows, int dim, int64_t* slice_rows,
                     bool* lo_only) {
    *slice_rows = 0;
    *lo_only = false;
    const int64_t plane_bytes = rows * (int64_t)dim * 4;   // hi + lo
    if (h->fact_budget <= 0 || plane_bytes <= h->fact_budget) return 0;
    HRAG_CHECK(h->world == 1, who + ": fact planes in host memory (hrag_set_fact_memory) serve one GPU only; a "
                                    "node-range-sharded handle (world > 1) keeps its fact slice resident");
    HRAG_CHECK(dim % 8 == 0, who + ": fact planes in host memory need dim % 8 == 0 (the tensor-core layout)");
    if (h->fact_placement != HRAG_FACT_LO_ON_HOST)
        return host_planes_plan(h->fact_budget, who, "hrag_set_fact_memory", rows, dim, slice_rows);
    // the hi plane resident, the rest of the budget a ring of two lo slices
    const int64_t hi_bytes = rows * (int64_t)dim * 2, lo_row = (int64_t)dim * 2;
    const int64_t slice = (h->fact_budget - hi_bytes) / (2 * lo_row) / kSliceAlign * kSliceAlign;
    HRAG_CHECK(h->fact_budget >= hi_bytes && slice >= kSliceAlign,
               who + ": HRAG_FACT_LO_ON_HOST keeps the hi fact plane of " + std::to_string(hi_bytes) +
                   " bytes resident, and it with a lo ring of two 256-row slices (" +
                   std::to_string(2 * kSliceAlign * lo_row) + " bytes) exceeds the hrag_set_fact_memory budget of " +
                   std::to_string(h->fact_budget) + " bytes");
    *slice_rows = slice;
    *lo_only = true;
    return 0;
}

int fact_planes_alloc(hrag_t* h, int64_t slice_rows, bool lo_only) {
    h->fplanes.release();
    EmbMem& e = h->emb[0];
    if (lo_only) {   // the resident hi plane and the norm maxima its fill raises from zero
        HRAG_TRY(e.hi.ensure((size_t)e.rows * h->dim * 2));
        HRAG_TRY(e.nmax.zeros(2 * sizeof(float)));
    }
    return h->fplanes.alloc((size_t)e.rows * h->dim * 2, slice_rows, h->dim, lo_only);
}

int planes_fill(hrag_t* h, HostPlanes& ps, int dim, int64_t row0, int64_t n, const float* src, bool src_on_device,
                const BeforeWrite& before_write, char* hi_dev) {
    const int64_t d = dim, S = hi_dev ? ps.slice_rows / 2 : ps.slice_rows;   // rows per step
    char* stage = ps.ring.as<char>();
    char* split = stage + (size_t)S * d * 4;
    for (int64_t r = 0; r < n; r += S) {
        const int64_t m = std::min(S, n - r);
        const size_t ne = (size_t)m * d;
        const float* x = src + (size_t)r * d;
        if (!src_on_device) {
            HRAG_CUDA(cudaMemcpyAsync(stage, x, ne * 4, cudaMemcpyHostToDevice, h->stream));
            x = reinterpret_cast<const float*>(stage);
        }
        const size_t at = (size_t)(row0 + r) * d * 2;
        char* hi = hi_dev ? hi_dev + at : split;   // lo_only: the hi rows go straight to the resident plane
        char* lo = hi_dev ? split : split + (size_t)S * d * 2;
        HRAG_TRY(split_bf16(x, (int64_t)ne, hi, lo, h->stream));
        if (before_write) HRAG_TRY(before_write(r, m, hi, lo));
        if (!hi_dev)
            HRAG_CUDA(cudaMemcpyAsync(static_cast<char*>(ps.hi) + at, hi, ne * 2, cudaMemcpyDeviceToHost, h->stream));
        HRAG_CUDA(cudaMemcpyAsync(static_cast<char*>(ps.lo) + at, lo, ne * 2, cudaMemcpyDeviceToHost, h->stream));
    }
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    return 0;
}

// Ring half 0 stages up to slice_rows fp32 rows (slice_rows x dim x 4 bytes: exactly one half), half 1 takes their
// split (hi rows, then lo rows), which goes back to the pinned planes.  split_bf16 is element-wise, so the planes are
// byte for byte those of a resident load.  lo_only: the hi rows go to the resident plane, and the split rows raise the
// norm maxima, as fact_norms_update raises them over resident planes (a maximum: any order of rows gives its bits).
int fact_planes_fill(hrag_t* h, int64_t row0, int64_t n, const float* src, bool src_on_device) {
    FactPlanes& fp = h->fplanes;
    if (!fp.lo_only()) return planes_fill(h, fp, h->dim, row0, n, src, src_on_device);
    EmbMem& e = h->emb[0];
    auto norms = [&](int64_t, int64_t m, const char* hi, const char* lo) {
        return plane_norm_max(hi, lo, m, h->dim, e.nmax.as<unsigned int>(), h->stream);
    };
    return planes_fill(h, fp, h->dim, row0, n, src, src_on_device, norms, e.hi.as<char>());
}

// Queries per pass: their bf16 hi / lo splits (dim x 4 bytes each) stay on the device for the whole pass and are
// bounded by kPassSplitBytes (256 MB): 65,536 queries at dim 1024, 16,384 at dim 4096.  A call with more queries
// streams the planes once per pass.
int64_t fact_stream_pass_cap(const hrag_t* h) {
    const int64_t per_query = 4 * (int64_t)std::max(h->dim, 1);
    return std::max<int64_t>(kPassChunk, (int64_t)kPassSplitBytes / per_query / kPassChunk * kPassChunk);
}

// The split K2 over every fact, the planes streamed once per pass (lo only when lo_only: hi is read in place).
static int streamed_stage_a(hrag_t* h, int B, const float* q, bool q_on_device, int k, int* d_top_idx,
                            float* d_top_score, int* d_nvalid) {
    FactPlanes& fp = h->fplanes;
    const int64_t F = h->emb[0].rows, d = h->dim, S = fp.slice_rows;
    const int64_t n_slices = ceil_div(F, S);
    const bool fused = !h->keep_fact_scores && k <= kFusedK;
    const int n_seg = h->sim_mode == HRAG_SIM_BF16X3 ? 4 : 1;
    const int n_ctas = h->debug_sim_ctas > 0 ? h->debug_sim_ctas : h->num_sms;
    const int64_t cap = fact_stream_pass_cap(h);
    const int64_t Bmax = std::min<int64_t>(cap, B);
    // query chunk of one K2 launch: the fused partials are 72 B per (query, tile of the slice); a materialised slice
    // row is pad4(slice_rows) floats (the resident rule of chunk_a, per slice instead of per matrix)
    const int64_t ldS = pad4(S);
    const int64_t chunk = fused ? kPassChunk
                                : std::max<int64_t>(1, std::min<int64_t>((int64_t)(4e9 / (4.0 * (double)ldS)),
                                                                         kPassChunk));
    const int64_t cb = std::min<int64_t>(chunk, Bmax);
    HRAG_TRY(h->q_hi.ensure((size_t)Bmax * d * 2));
    HRAG_TRY(h->q_lo.ensure((size_t)Bmax * d * 2));
    if (!q_on_device) HRAG_TRY(h->d_q.ensure((size_t)std::min<int64_t>(kPassChunk, Bmax) * d * 4));
    if (fused) {
        const int nt = sim_tc_n_tiles(S);
        HRAG_TRY(h->part_mm.ensure((size_t)cb * nt * sizeof(float2)));
        HRAG_TRY(h->part_keys.ensure((size_t)cb * nt * 8 * sizeof(uint64_t)));
        HRAG_TRY(h->part_bound.ensure((size_t)cb * sizeof(uint64_t)));
        HRAG_TRY(h->mm_fact.ensure((size_t)Bmax * sizeof(float2)));
        HRAG_TRY(fp.run_mm.ensure((size_t)3 * Bmax * sizeof(float2)));     // slots: running x 2, this slice
        HRAG_TRY(fp.run_keys.ensure((size_t)3 * Bmax * 8 * sizeof(uint64_t)));
    } else {
        HRAG_TRY(h->S_fact.ensure((size_t)cb * ldS * sizeof(float)));
        HRAG_TRY(fp.sl_ids.ensure((size_t)cb * k * sizeof(int)));
        HRAG_TRY(fp.sl_scores.ensure((size_t)cb * k * sizeof(float)));
        HRAG_TRY(fp.sl_mm.ensure((size_t)cb * sizeof(float2)));
        HRAG_TRY(fp.run_mm.ensure((size_t)Bmax * sizeof(float2)));
    }
    const char* q_hi = h->q_hi.as<char>();
    const char* q_lo = h->q_lo.as<char>();
    for (int64_t p0 = 0; p0 < B; p0 += cap) {
        const int64_t Bp = std::min<int64_t>(cap, B - p0);
        {   // the pass's query splits, once
            StageTimer tm(h, ST_SIM_FACT);
            for (int64_t q0 = 0; q0 < Bp; q0 += kPassChunk) {
                const int64_t nb = std::min<int64_t>(kPassChunk, Bp - q0);
                const float* x = q + (size_t)(p0 + q0) * d;
                if (!q_on_device) {
                    HRAG_TRY(h2d(h, h->d_q.p, x, (size_t)nb * d * 4));
                    x = h->d_q.as<float>();
                }
                HRAG_TRY(split_bf16(x, nb * d, h->q_hi.as<char>() + (size_t)q0 * d * 2,
                                    h->q_lo.as<char>() + (size_t)q0 * d * 2, h->stream));
            }
        }
        float2* run_mm = fp.run_mm.as<float2>();
        uint64_t* run_keys = fp.run_keys.as<uint64_t>();
        int cur = 0;   // fused: the running slot (0 or 1); slot 2 takes the slice being folded in
        auto body = [&](int64_t s, int64_t r0, int64_t ns, const void* e_hi, const void* e_lo) -> int {
            const bool last = s == n_slices - 1;
            for (int64_t q0 = 0; q0 < Bp; q0 += chunk) {
                const int nb = (int)std::min<int64_t>(chunk, Bp - q0);
                const int64_t o = p0 + q0;   // output row
                const void* qh = q_hi + (size_t)q0 * d * 2;
                const void* ql = q_lo + (size_t)q0 * d * 2;
                if (fused) {
                    const int nt = sim_tc_n_tiles(ns);
                    {
                        StageTimer tm(h, ST_SIM_FACT);
                        HRAG_TRY(sim_tc(qh, ql, nb, e_hi, e_lo, ns, (int)d, n_seg, nullptr, 0, h->part_mm.as<float2>(),
                                        h->part_keys.as<uint64_t>(), h->part_bound.as<uint64_t>(), n_ctas, h->stream));
                    }
                    StageTimer tm(h, ST_SEL_FACT);
                    const float2* pmm = h->part_mm.as<float2>();
                    const uint64_t* pkeys = h->part_keys.as<uint64_t>();
                    if (n_slices == 1) {
                        HRAG_TRY(merge_minmax_topk_ex(pmm, pkeys, nb, nt, nt, 1, 0, F, k, h->mm_fact.as<float2>() + q0,
                                                      d_top_idx + o * k, d_top_score + o * k, d_nvalid + o, nullptr,
                                                      h->stream));
                        continue;
                    }
                    // this slice's 8 best (global rows) and (min, max): into the running slot for the first slice,
                    // else into slot 2, then folded with the running slot into the other one -- or, after the
                    // last slice, into the normalised outputs, exactly as the sharded path merges its ranks' lists
                    const int tgt = s == 0 ? cur : 2;
                    HRAG_TRY(merge_minmax_topk_ex(pmm, pkeys, nb, nt, nt, 1, r0, ns, kFusedK,
                                                  run_mm + tgt * Bp + q0, nullptr, nullptr, nullptr,
                                                  run_keys + (size_t)(tgt * Bp + q0) * 8, h->stream));
                    if (s == 0) continue;
                    const int nxt = 1 - cur;
                    const float2* amm = run_mm + cur * Bp + q0;
                    const uint64_t* akeys = run_keys + (size_t)(cur * Bp + q0) * 8;
                    if (last)
                        HRAG_TRY(merge_minmax_topk_ex(amm, akeys, nb, 2, 1, (2 - cur) * Bp, 0, F, k,
                                                      h->mm_fact.as<float2>() + q0, d_top_idx + o * k,
                                                      d_top_score + o * k, d_nvalid + o, nullptr, h->stream));
                    else
                        HRAG_TRY(merge_minmax_topk_ex(amm, akeys, nb, 2, 1, (2 - cur) * Bp, 0, F, kFusedK,
                                                      run_mm + nxt * Bp + q0, nullptr, nullptr, nullptr,
                                                      run_keys + (size_t)(nxt * Bp + q0) * 8, h->stream));
                } else {
                    float* Sf = h->S_fact.as<float>();
                    {
                        StageTimer tm(h, ST_SIM_FACT);
                        HRAG_TRY(sim_tc(qh, ql, nb, e_hi, e_lo, ns, (int)d, n_seg, Sf, ldS, nullptr, nullptr, nullptr,
                                        n_ctas, h->stream));
                    }
                    StageTimer tm(h, ST_SEL_FACT);
                    HRAG_TRY(row_minmax_topk(Sf, nb, ns, ldS, 0, fp.sl_mm.as<float2>(), nullptr, nullptr, nullptr,
                                             h->stream));
                    HRAG_TRY(row_topk(Sf, nb, ns, ldS, k, fp.sl_ids.as<int>(), fp.sl_scores.as<float>(), h->stream));
                    HRAG_TRY(fold_topk(nb, k, r0, fp.sl_ids.as<int>(), fp.sl_scores.as<float>(),
                                       fp.sl_mm.as<float2>(), d_top_idx + o * k, d_top_score + o * k,
                                       run_mm + q0, s == 0, h->stream));
                }
            }
            if (fused && s > 0) cur = 1 - cur;
            return 0;
        };
        HRAG_TRY(stream_slices(h, fp, d, 0, F, n_seg == 4, body, fp.lo_only() ? h->emb[0].hi.as<char>() : nullptr));
        if (!fused) {
            StageTimer tm(h, ST_SEL_FACT);
            HRAG_TRY(topk_normalize((int)Bp, k, F, run_mm, d_top_idx + p0 * k, d_top_score + p0 * k, d_nvalid + p0,
                                    h->stream));
        }
    }
    return 0;
}

// Queries per screened chunk with the lo plane in host memory: the screen's partials (part_keys, part_low, part_mm)
// take 88 bytes per query and 256-fact tile; the chunk keeps them within kLoHostPartialBytes in multiples of 128
// queries (one m-tile), at most kPassChunk (the resident chunk): 1,024 at 2.75 M facts, 128 at 17 M.  A smaller chunk
// reads the hi plane once more per chunk.
constexpr int64_t kLoHostPartialBytes = int64_t(1) << 30;
static int64_t lo_host_chunk(const hrag_t* h) {
    const int64_t per_query = 88 * (int64_t)sim_tc_n_tiles(std::max<int64_t>(h->emb[0].rows, 1));
    return std::min<int64_t>(kPassChunk, std::max<int64_t>(128, kLoHostPartialBytes / per_query / 128 * 128));
}

// The screen over chunks of lo_host_chunk queries, each raising its own flag; then the flags and the lo bytes the
// gathers read are copied back at once (the one synchronise of the call), and each flagged chunk reruns exactly
// (streamed_stage_a: the split K2, lo streamed) over its outputs and counts as a fallback.
static int lo_host_screened_stage_a(hrag_t* h, int B, const float* q, bool q_on_device, int k, int* d_top_idx,
                                    float* d_top_score, int* d_nvalid) {
    const int64_t d = h->dim, chunk = lo_host_chunk(h), n_chunks = ceil_div(B, chunk);
    const int n_ctas = h->debug_sim_ctas > 0 ? h->debug_sim_ctas : h->num_sms;
    const size_t flag_bytes = sizeof(unsigned long long) + (size_t)n_chunks * sizeof(int);
    HRAG_TRY(h->scr.call_flags.ensure(flag_bytes));
    HRAG_TRY(h->mm_fact.ensure((size_t)std::min<int64_t>(chunk, B) * sizeof(float2)));
    if (!q_on_device) HRAG_TRY(h->d_q.ensure((size_t)std::min<int64_t>(chunk, B) * d * 4));
    unsigned long long* lo_bytes = h->scr.call_flags.as<unsigned long long>();
    int* flags = reinterpret_cast<int*>(lo_bytes + 1);
    HRAG_CUDA(cudaMemsetAsync(lo_bytes, 0, flag_bytes, h->stream));
    auto chunk_queries = [&](int64_t q0, int nb, const float** x) -> int {   // device fp32 queries of the chunk
        *x = q + (size_t)q0 * d;
        if (!q_on_device) {
            HRAG_TRY(h2d(h, h->d_q.p, *x, (size_t)nb * d * 4));
            *x = h->d_q.as<float>();
        }
        return 0;
    };
    for (int64_t c = 0; c < n_chunks; ++c) {
        const int64_t q0 = c * chunk;
        const int nb = (int)std::min<int64_t>(chunk, B - q0);
        const float* x = nullptr;
        HRAG_TRY(chunk_queries(q0, nb, &x));
        HRAG_TRY(screened_stage_a(h, nb, x, k, d_top_idx + q0 * k, d_top_score + q0 * k, d_nvalid + q0, h->stream,
                                  n_ctas, flags + c, lo_bytes));
    }
    std::vector<char> host(flag_bytes);
    HRAG_CUDA(cudaMemcpyAsync(host.data(), lo_bytes, flag_bytes, cudaMemcpyDeviceToHost, h->stream));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    unsigned long long gathered = 0;
    std::memcpy(&gathered, host.data(), sizeof(gathered));
    h->stats.h2d_bytes += (int64_t)gathered;
    for (int64_t c = 0; c < n_chunks; ++c) {
        int flagged = 0;
        std::memcpy(&flagged, host.data() + sizeof(gathered) + (size_t)c * sizeof(int), sizeof(int));
        if (!flagged) continue;
        const int64_t q0 = c * chunk;
        const int nb = (int)std::min<int64_t>(chunk, B - q0);
        const float* x = nullptr;
        HRAG_TRY(chunk_queries(q0, nb, &x));
        HRAG_TRY(streamed_stage_a(h, nb, x, true, k, d_top_idx + q0 * k, d_top_score + q0 * k, d_nvalid + q0));
        h->stats.stage_a_fallbacks += 1;
    }
    h->last_mm_rows = n_chunks == 1 ? B : 0;   // mm_fact holds the one chunk's (min, max)
    return 0;
}

int fact_stream_stage_a(hrag_t* h, int B, const float* q, bool q_on_device, int k, int* d_top_idx,
                        float* d_top_score, int* d_nvalid) {
    HRAG_CHECK(h->sim_mode != HRAG_SIM_FP32, std::string("stage A ") + kNoFp32);
    h->last_fact_rows = 0;
    h->last_mm_rows = 0;
    if (B == 0) return 0;
    if (h->fplanes.lo_only() && !h->keep_fact_scores && k <= kFusedK && screened(h))
        return lo_host_screened_stage_a(h, B, q, q_on_device, k, d_top_idx, d_top_score, d_nvalid);
    return streamed_stage_a(h, B, q, q_on_device, k, d_top_idx, d_top_score, d_nvalid);
}

// K2 writes a score tile up to its 256-column end, clipped at ldS columns from the pointer it is given.  A slice that
// ends on a tile boundary therefore writes in place (S + its first row); a ragged last slice would spill into the
// next row, so it goes through `tail` [nb, pad4(rows)] and a 2-D copy.
int fact_stream_scores(hrag_t* h, int nb, const float* d_q, float* S, int64_t ldS) {
    HRAG_CHECK(h->sim_mode != HRAG_SIM_FP32, kNoFp32);
    FactPlanes& fp = h->fplanes;
    const int n_seg = h->sim_mode == HRAG_SIM_BF16X3 ? 4 : 1;
    const int64_t F = h->emb[0].rows, last_rows = F - (ceil_div(F, fp.slice_rows) - 1) * fp.slice_rows;
    HRAG_TRY(split_queries(h, d_q, nb, h->stream));
    if (last_rows % kSliceAlign) HRAG_TRY(fp.tail.ensure((size_t)nb * pad4(last_rows) * sizeof(float)));
    auto body = [&](int64_t, int64_t r0, int64_t ns, const void* e_hi, const void* e_lo) -> int {
        const bool ragged = ns % kSliceAlign != 0;
        float* out = ragged ? fp.tail.as<float>() : S + r0;
        const int64_t ld = ragged ? pad4(ns) : ldS;
        HRAG_TRY(sim_tc(h->q_hi.p, h->q_lo.p, nb, e_hi, e_lo, ns, h->dim, n_seg, out, ld, nullptr, nullptr, nullptr,
                        h->num_sms, h->stream));
        if (ragged)
            HRAG_CUDA(cudaMemcpy2DAsync(S + r0, (size_t)ldS * sizeof(float), out, (size_t)ld * sizeof(float),
                                        (size_t)ns * sizeof(float), (size_t)nb, cudaMemcpyDeviceToDevice, h->stream));
        return 0;
    };
    return stream_slices(h, fp, h->dim, 0, F, n_seg == 4, body, fp.lo_only() ? h->emb[0].hi.as<char>() : nullptr);
}

}  // namespace hrag

using namespace hrag;

extern "C" {

int hrag_set_fact_memory(hrag_t* h, int64_t max_device_bytes) {
    HRAG_CHECK(h, "hrag_set_fact_memory: null handle");
    HRAG_CHECK(max_device_bytes >= 0, "hrag_set_fact_memory: the budget must be >= 0 bytes (0 = no limit)");
    HRAG_CHECK(h->world == 1 || max_device_bytes == 0,
               "hrag_set_fact_memory: fact planes in host memory serve one GPU only; a node-range-sharded handle "
               "(world > 1) keeps its fact slice resident");
    h->fact_budget = max_device_bytes;
    return 0;
}

int hrag_set_fact_placement(hrag_t* h, int placement) {
    HRAG_CHECK(h, "hrag_set_fact_placement: null handle");
    HRAG_CHECK(placement == HRAG_FACT_PLANES_BY_BUDGET || placement == HRAG_FACT_LO_ON_HOST,
               "hrag_set_fact_placement: placement must be HRAG_FACT_PLANES_BY_BUDGET (0) or HRAG_FACT_LO_ON_HOST (1)");
    HRAG_CHECK(h->world == 1 || placement == HRAG_FACT_PLANES_BY_BUDGET,
               "hrag_set_fact_placement: fact planes in host memory serve one GPU only; a node-range-sharded handle "
               "(world > 1) keeps its fact slice resident");
    h->fact_placement = placement;
    return 0;
}

int hrag_fact_planes_info(hrag_t* h, int* on_host, int64_t* slice_rows, int64_t* device_bytes, int64_t* host_bytes) {
    HRAG_CHECK(h && on_host && slice_rows && device_bytes && host_bytes, "hrag_fact_planes_info: null argument");
    const FactPlanes& fp = h->fplanes;
    *on_host = fp.lo_only() ? 2 : fp.held() ? 1 : 0;
    *slice_rows = fp.slice_rows;
    *device_bytes = fp.lo_only() ? (int64_t)(h->emb[0].hi.cap + fp.ring.cap)
                    : fp.held()  ? (int64_t)fp.ring.cap
                                 : (int64_t)(h->emb[0].hi.cap + h->emb[0].lo.cap);
    *host_bytes = fp.lo_only() ? (int64_t)fp.plane_bytes : fp.held() ? 2 * (int64_t)fp.plane_bytes : 0;
    return 0;
}

}  // extern "C"
