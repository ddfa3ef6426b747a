// The fact planes: where they live, how they are filled, and stage A and the raw fact scores walked over them.
//
// Planes over the device budget of hrag_set_fact_memory live in pinned host memory (both, or under
// HRAG_FACT_LO_ON_HOST the lo plane only, mapped; DESIGN.md sections 7e and 7h) and stream through a device ring of
// two slices: a copy stream fills one half with slice s + 1 while the similarity GEMM (K2, unchanged) reads slice s
// from the other; events order the two.  The walker (stream_slices, handle.h) reads a resident plane in place; over
// resident planes it is one slice, one body call on the caller's stream.  Stage A walks the planes once per pass of
// queries (one query chunk on resident planes, fact_stream_pass_cap queries when a plane streams): slices are the
// outer loop, query chunks the inner.
//
// Results do not depend on the placement, bit for bit: K2's accumulator for a (query, fact) pair does not depend on
// the tile the fact falls in, and a slice starts on a 256-row tile boundary.  Over several slices the fused top-8 path
// merges each slice's per-tile lists with the slice's first row as index offset and folds the per-slice lists into a
// running one with the same kernel the fact-sharded stage A uses across ranks (merge_minmax_topk_ex); the materialised
// path (k > 8, or hrag_debug_keep_scores) takes each slice's exact top-k and (min, max) and folds them with fold_topk
// (select.cu).  One slice selects directly.
//
// The walker and the fill (planes_fill) take any plane set: the synonymy KNN index walks its planes through them too
// (knn_index.cu).
//
// With the lo plane on the host, the stage-A screen (api.cu screened_stage_a) runs per query chunk: the hi.hi screen
// over the resident hi plane, the staged candidates' lo rows read from the mapped plane by the gather.  One flag per
// chunk; after the call's chunks the flags are read at once and a flagged chunk reruns the split K2, lo streamed.
#include <algorithm>
#include <cstring>
#include <vector>

#include "handle.h"

namespace hrag {

int split_queries(hrag_t* h, const float* dQ, int Bq, cudaStream_t s);   // api.cu
int64_t pad4(int64_t x);                                                  // api.cu

namespace {

constexpr int64_t kSliceAlign = 256;                // K2's tile width: every slice boundary is a tile boundary
constexpr size_t kPassSplitBytes = size_t(256) << 20;   // bound on one pass's query splits (bf16 hi + lo)
constexpr int kFusedTopK = 8;                        // candidates the GEMM epilogue / row_minmax_topk keep in registers

const char* kNoFp32 = "similarity: the fact planes are held in host memory (hrag_set_fact_memory) and no fp32 copy "
                      "of the fact rows is kept; only the tensor-core modes are available";

// Queries per K2 launch over `rows` facts: the fused partials are 72 B per (query, 256 facts), 0.8 GB at F = 2.75 M;
// a materialised score row is pad4(rows) floats.
int64_t chunk_for(bool fused, int64_t rows) {
    if (fused) return kQueryChunk;
    const int64_t c = (int64_t)(4e9 / (4.0 * (double)pad4(std::max<int64_t>(rows, 1))));
    return std::max<int64_t>(1, std::min<int64_t>(c, kQueryChunk));
}

// Queries per pass when a plane streams: their bf16 hi / lo splits (dim x 4 bytes each) stay on the device for the
// whole pass and are bounded by kPassSplitBytes (256 MB): 65,536 queries at dim 1024, 16,384 at dim 4096.  A call with
// more queries streams the planes once per pass.
int64_t fact_stream_pass_cap(const hrag_t* h) {
    const int64_t per_query = 4 * (int64_t)std::max(h->dim, 1);
    return std::max<int64_t>(kQueryChunk, (int64_t)kPassSplitBytes / per_query / kQueryChunk * kQueryChunk);
}

// sim_fp32 over the resident fp32 rows of matrix `which`
int fp32_scores(hrag_t* h, int which, const float* dQ, int nb, float* S, int64_t ldS, cudaStream_t s) {
    HRAG_CHECK(!emb_planes(h, which).streams(), kNoFp32);
    const EmbMem& e = h->emb[which];
    HRAG_CHECK(e.f32 != nullptr, "similarity: the fp32 embedding matrix was not kept (streamed upload); only the "
                                 "tensor-core modes are available");
    return sim_fp32(dQ, nb, e.f32, e.rows, h->dim, S, ldS, s);
}

// Fact-sharded stage A (world > 1; SURVEY.md 8(e)): the local top-8 and (min, max) per query from the K2 partials of
// the rank's fact rows, all-gathered, and the same merge kernel over the `world` candidate lists.
int sharded_select(hrag_t* h, int Bq, int nt, int k, float2* mm, int* idx, float* score, int* nv, cudaStream_t s) {
    const int64_t F = h->emb[0].rows;
    HRAG_TRY(h->xr_mm.ensure((size_t)h->world * Bq * sizeof(float2)));
    HRAG_TRY(h->xr_keys.ensure((size_t)h->world * Bq * 8 * sizeof(uint64_t)));
    float2* mm_all = h->xr_mm.as<float2>();
    uint64_t* keys_all = h->xr_keys.as<uint64_t>();
    {
        StageTimer tm(h, ST_SEL_FACT, s);
        HRAG_TRY(merge_minmax_topk_ex(h->part_mm.as<float2>(), h->part_keys.as<uint64_t>(), Bq, nt, nt, 1,
                                      h->fact_row_lo, F, 8, mm_all + (size_t)h->rank * Bq, nullptr, nullptr, nullptr,
                                      keys_all + (size_t)h->rank * Bq * 8, s));
    }
    {
        StageTimer tc(h, ST_COMM, s);
        HRAG_NCCL(g_nccl.AllGather(mm_all + (size_t)h->rank * Bq, mm_all, (size_t)Bq * sizeof(float2), ncclInt8,
                                   h->comm, s));
        HRAG_NCCL(g_nccl.AllGather(keys_all + (size_t)h->rank * Bq * 8, keys_all, (size_t)Bq * 8 * sizeof(uint64_t),
                                   ncclInt8, h->comm, s));
    }
    StageTimer tm(h, ST_SEL_FACT, s);
    return merge_minmax_topk_ex(mm_all, keys_all, Bq, h->world, 1, Bq, 0, h->n_facts_global, k, mm, idx, score, nv,
                                nullptr, s);
}

}  // namespace

int HostPlanes::alloc(size_t bytes, int64_t slice, int dim, bool with_hi) {
    release();
    if (with_hi) {
        HRAG_CUDA(cudaHostAlloc(&hi, bytes, cudaHostAllocDefault));
        HRAG_CUDA(cudaHostAlloc(&lo, bytes, cudaHostAllocDefault));
    } else {   // the stage-A screen's gather reads lo rows in place
        HRAG_CUDA(cudaHostAlloc(&lo, bytes, cudaHostAllocMapped));
    }
    plane_bytes = bytes;
    slice_rows = slice;
    HRAG_TRY(ring.ensure((size_t)2 * slice * dim * (with_hi ? 4 : 2)));
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
    hi = lo = nullptr;
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
                     bool* hi_resident) {
    *slice_rows = 0;
    *hi_resident = false;
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
    *hi_resident = true;
    return 0;
}

int fact_planes_alloc(hrag_t* h, int64_t slice_rows, bool hi_resident) {
    h->fplanes.release();
    EmbMem& e = h->emb[0];
    if (hi_resident) {   // the resident hi plane and the norm maxima its fill raises from zero
        HRAG_TRY(e.hi.ensure((size_t)e.rows * h->dim * 2));
        HRAG_TRY(e.nmax.zeros(2 * sizeof(float)));
    }
    return h->fplanes.alloc((size_t)e.rows * h->dim * 2, slice_rows, h->dim, !hi_resident);
}

int planes_fill(hrag_t* h, const PlaneSet& P, int dim, int64_t row0, int64_t n, const float* src, bool src_on_device,
                const BeforeWrite& before_write) {
    const size_t rb = (size_t)dim * 2;
    const size_t half_bytes = (size_t)P.host->slice_rows * rb * ((P.on_host[0] ? 1 : 0) + (P.on_host[1] ? 1 : 0));
    const int64_t d = dim, S = (int64_t)(half_bytes / (rb * 2));   // fp32 rows per step: one ring half
    char* stage = P.host->ring.as<char>();
    char* split = stage + half_bytes;
    for (int64_t r = 0; r < n; r += S) {
        const int64_t m = std::min(S, n - r);
        const size_t ne = (size_t)m * d;
        const float* x = src + (size_t)r * d;
        if (!src_on_device) {
            HRAG_CUDA(cudaMemcpyAsync(stage, x, ne * 4, cudaMemcpyHostToDevice, h->stream));
            x = reinterpret_cast<const float*>(stage);
        }
        const size_t at = (size_t)(row0 + r) * rb;
        char* hi = P.on_host[0] ? split : P.plane[0] + at;   // a resident plane takes its rows directly
        char* lo = P.on_host[1] ? split + (P.on_host[0] ? (size_t)S * rb : 0) : P.plane[1] + at;
        HRAG_TRY(split_bf16(x, (int64_t)ne, hi, lo, h->stream));
        if (before_write) HRAG_TRY(before_write(r, m, hi, lo));
        if (P.on_host[0]) HRAG_CUDA(cudaMemcpyAsync(P.plane[0] + at, hi, ne * 2, cudaMemcpyDeviceToHost, h->stream));
        if (P.on_host[1]) HRAG_CUDA(cudaMemcpyAsync(P.plane[1] + at, lo, ne * 2, cudaMemcpyDeviceToHost, h->stream));
    }
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    return 0;
}

// split_bf16 is element-wise, so the planes are byte for byte those of a resident load.  A resident hi plane's rows
// raise the norm maxima, as fact_norms_update raises them over resident planes (a maximum: any order of rows gives its
// bits).
int fact_planes_fill(hrag_t* h, int64_t row0, int64_t n, const float* src, bool src_on_device) {
    const PlaneSet P = emb_planes(h, 0);
    if (P.on_host[0]) return planes_fill(h, P, h->dim, row0, n, src, src_on_device);
    EmbMem& e = h->emb[0];
    auto norms = [&](int64_t, int64_t m, const char* hi, const char* lo) {
        return plane_norm_max(hi, lo, m, h->dim, e.nmax.as<unsigned int>(), h->stream);
    };
    return planes_fill(h, P, h->dim, row0, n, src, src_on_device, norms);
}

bool fused_stage_a(const hrag_t* h, int k) {   // tensor-core modes select facts in the GEMM epilogue (no score matrix)
    return h->sim_mode != HRAG_SIM_FP32 && emb_planes(h, 0).plane[0] != nullptr && !h->keep_fact_scores &&
           k <= kFusedTopK;
}

int64_t chunk_a(const hrag_t* h, int k) { return chunk_for(fused_stage_a(h, k), h->emb[0].rows); }

// The split K2 over every fact, walked over the planes in passes of chunk_a queries (resident) or
// fact_stream_pass_cap queries (a plane streams); `screen` (resident planes): each pass runs the stage-A screen with
// its gated exact rerun instead.
static int walk_stage_a(hrag_t* h, const PlaneSet& P, int B, const float* q, bool q_on_device, int k, int* d_top_idx,
                        float* d_top_score, int* d_nvalid, cudaStream_t s, int n_ctas, bool screen) {
    FactPlanes& fp = h->fplanes;
    const int64_t F = h->emb[0].rows, d = h->dim;
    const int64_t S = P.streams() ? fp.slice_rows : F, n_slices = P.streams() ? ceil_div(F, S) : 1;
    const bool fused = fused_stage_a(h, k), one = n_slices == 1;
    const bool tc = h->sim_mode != HRAG_SIM_FP32 && P.plane[0] != nullptr;   // else sim_fp32 (resident planes)
    const int n_seg = h->sim_mode == HRAG_SIM_BF16X3 ? 4 : 1;
    HRAG_CHECK(h->world == 1 || fused, "node-range sharding: stage A needs the tensor-core similarity with "
                                       "linking_top_k <= 8 (the fact rows are sharded; the fp32 / materialised paths "
                                       "are single-GPU)");
    const int64_t cap = P.streams() ? fact_stream_pass_cap(h) : chunk_for(fused, F);
    const int64_t Bmax = std::min<int64_t>(cap, B);
    const int64_t ldS = pad4(S), chunk = chunk_for(fused, S), cb = std::min<int64_t>(chunk, Bmax);
    if (tc) {
        HRAG_TRY(h->q_hi.ensure((size_t)Bmax * d * 2));
        HRAG_TRY(h->q_lo.ensure((size_t)Bmax * d * 2));
    }
    if (!q_on_device) HRAG_TRY(h->d_q.ensure((size_t)std::min<int64_t>(kQueryChunk, Bmax) * d * 4));
    if (fused || one) HRAG_TRY(h->mm_fact.ensure((size_t)Bmax * sizeof(float2)));
    if (fused && !screen) {
        const int nt = sim_tc_n_tiles(S);
        HRAG_TRY(h->part_mm.ensure((size_t)cb * nt * sizeof(float2)));
        HRAG_TRY(h->part_keys.ensure((size_t)cb * nt * 8 * sizeof(uint64_t)));
        HRAG_TRY(h->part_bound.ensure((size_t)cb * sizeof(uint64_t)));
        if (!one) {
            HRAG_TRY(fp.run_mm.ensure((size_t)3 * Bmax * sizeof(float2)));     // slots: running x 2, this slice
            HRAG_TRY(fp.run_keys.ensure((size_t)3 * Bmax * 8 * sizeof(uint64_t)));
        }
    } else if (!fused) {
        HRAG_TRY(h->S_fact.ensure((size_t)cb * ldS * sizeof(float)));
        if (!one) {
            HRAG_TRY(fp.sl_ids.ensure((size_t)cb * k * sizeof(int)));
            HRAG_TRY(fp.sl_scores.ensure((size_t)cb * k * sizeof(float)));
            HRAG_TRY(fp.sl_mm.ensure((size_t)cb * sizeof(float2)));
            HRAG_TRY(fp.run_mm.ensure((size_t)Bmax * sizeof(float2)));
        }
    }
    const char* q_hi = h->q_hi.as<char>();
    const char* q_lo = h->q_lo.as<char>();
    float2* mm = h->mm_fact.as<float2>();
    for (int64_t p0 = 0; p0 < B; p0 += cap) {
        const int64_t Bp = std::min<int64_t>(cap, B - p0);
        auto queries = [&](int64_t q0, int64_t nb, const float** x) -> int {   // fp32 rows p0 + q0 .. on the device
            *x = q + (size_t)(p0 + q0) * d;
            if (!q_on_device) {
                HRAG_TRY(h2d(h, h->d_q.p, *x, (size_t)nb * d * 4));
                *x = h->d_q.as<float>();
            }
            return 0;
        };
        h->last_mm_rows = P.streams() ? 0 : Bp;
        if (screen) {   // a resident pass is one query chunk
            const float* x = nullptr;
            HRAG_TRY(queries(0, Bp, &x));
            HRAG_TRY(screened_stage_a(h, (int)Bp, x, k, d_top_idx + p0 * k, d_top_score + p0 * k, d_nvalid + p0, s,
                                      n_ctas));
            continue;
        }
        const float* x32 = nullptr;   // !tc: the pass's fp32 queries (resident planes: one upload chunk)
        if (tc) {   // the pass's query splits, once
            StageTimer tm(h, ST_SIM_FACT, s);
            for (int64_t q0 = 0; q0 < Bp; q0 += kQueryChunk) {
                const int64_t nb = std::min<int64_t>(kQueryChunk, Bp - q0);
                const float* x = nullptr;
                HRAG_TRY(queries(q0, nb, &x));
                HRAG_TRY(split_bf16(x, nb * d, h->q_hi.as<char>() + (size_t)q0 * d * 2,
                                    h->q_lo.as<char>() + (size_t)q0 * d * 2, s));
            }
        } else {
            HRAG_TRY(queries(0, Bp, &x32));
        }
        float2* run_mm = fp.run_mm.as<float2>();
        uint64_t* run_keys = fp.run_keys.as<uint64_t>();
        int cur = 0;   // fused: the running slot (0 or 1); slot 2 takes the slice being folded in
        auto body = [&](int64_t sl, int64_t r0, int64_t ns, const void* e_hi, const void* e_lo) -> int {
            const bool last = sl == n_slices - 1;
            for (int64_t q0 = 0; q0 < Bp; q0 += chunk) {
                const int nb = (int)std::min<int64_t>(chunk, Bp - q0);
                const int64_t o = p0 + q0;   // output row
                int* idx = d_top_idx + o * k;
                float* score = d_top_score + o * k;
                const void* qh = q_hi + (size_t)q0 * d * 2;
                const void* ql = q_lo + (size_t)q0 * d * 2;
                if (fused) {
                    const int nt = sim_tc_n_tiles(ns);
                    {
                        StageTimer tm(h, ST_SIM_FACT, s);
                        HRAG_TRY(sim_tc(qh, ql, nb, e_hi, e_lo, ns, (int)d, n_seg, nullptr, 0, h->part_mm.as<float2>(),
                                        h->part_keys.as<uint64_t>(), h->part_bound.as<uint64_t>(), n_ctas, s));
                    }
                    if (h->world > 1) {
                        HRAG_TRY(sharded_select(h, nb, nt, k, mm + q0, idx, score, d_nvalid + o, s));
                        continue;
                    }
                    StageTimer tm(h, ST_SEL_FACT, s);
                    const float2* pmm = h->part_mm.as<float2>();
                    const uint64_t* pkeys = h->part_keys.as<uint64_t>();
                    if (one) {
                        HRAG_TRY(merge_minmax_topk(pmm, pkeys, nb, nt, F, k, mm + q0, idx, score, d_nvalid + o, s));
                        continue;
                    }
                    // this slice's 8 best (global rows) and (min, max): into the running slot for the first slice,
                    // else into slot 2, then folded with the running slot into the other one -- or, after the
                    // last slice, into the normalised outputs, exactly as the sharded path merges its ranks' lists
                    const int tgt = sl == 0 ? cur : 2;
                    HRAG_TRY(merge_minmax_topk_ex(pmm, pkeys, nb, nt, nt, 1, r0, ns, kFusedTopK,
                                                  run_mm + tgt * Bp + q0, nullptr, nullptr, nullptr,
                                                  run_keys + (size_t)(tgt * Bp + q0) * 8, s));
                    if (sl == 0) continue;
                    const int nxt = 1 - cur;
                    const float2* amm = run_mm + cur * Bp + q0;
                    const uint64_t* akeys = run_keys + (size_t)(cur * Bp + q0) * 8;
                    if (last)
                        HRAG_TRY(merge_minmax_topk_ex(amm, akeys, nb, 2, 1, (2 - cur) * Bp, 0, F, k, mm + q0, idx,
                                                      score, d_nvalid + o, nullptr, s));
                    else
                        HRAG_TRY(merge_minmax_topk_ex(amm, akeys, nb, 2, 1, (2 - cur) * Bp, 0, F, kFusedTopK,
                                                      run_mm + nxt * Bp + q0, nullptr, nullptr, nullptr,
                                                      run_keys + (size_t)(nxt * Bp + q0) * 8, s));
                } else {
                    float* Sf = h->S_fact.as<float>();
                    {
                        StageTimer tm(h, ST_SIM_FACT, s);
                        if (tc)
                            HRAG_TRY(sim_tc(qh, ql, nb, e_hi, e_lo, ns, (int)d, n_seg, Sf, ldS, nullptr, nullptr,
                                            nullptr, n_ctas, s));
                        else
                            HRAG_TRY(fp32_scores(h, 0, x32 + (size_t)q0 * d, nb, Sf, ldS, s));
                    }
                    StageTimer tm(h, ST_SEL_FACT, s);
                    h->last_fact_rows = one ? nb : 0;   // S_fact holds the chunk's scores over all facts
                    if (one && k <= kFusedTopK) {
                        HRAG_TRY(row_minmax_topk(Sf, nb, ns, ldS, k, mm + q0, idx, score, d_nvalid + o, s));
                    } else if (one) {   // linking_top_k > 8 (config_utils.py:184): exact radix select
                        HRAG_TRY(row_minmax_topk(Sf, nb, ns, ldS, 0, mm + q0, nullptr, nullptr, nullptr, s));
                        HRAG_TRY(row_topk(Sf, nb, ns, ldS, k, idx, score, s));
                        HRAG_TRY(topk_normalize(nb, k, F, mm + q0, idx, score, d_nvalid + o, s));
                    } else {
                        HRAG_TRY(row_minmax_topk(Sf, nb, ns, ldS, 0, fp.sl_mm.as<float2>(), nullptr, nullptr, nullptr,
                                                 s));
                        HRAG_TRY(row_topk(Sf, nb, ns, ldS, k, fp.sl_ids.as<int>(), fp.sl_scores.as<float>(), s));
                        HRAG_TRY(fold_topk(nb, k, r0, fp.sl_ids.as<int>(), fp.sl_scores.as<float>(),
                                           fp.sl_mm.as<float2>(), idx, score, run_mm + q0, sl == 0, s));
                    }
                }
            }
            if (fused && sl > 0) cur = 1 - cur;
            return 0;
        };
        HRAG_TRY(stream_slices(h, P, d, 0, F, n_seg == 4, body));
        if (!fused && !one) {
            StageTimer tm(h, ST_SEL_FACT, s);
            HRAG_TRY(topk_normalize((int)Bp, k, F, run_mm, d_top_idx + p0 * k, d_top_score + p0 * k, d_nvalid + p0,
                                    s));
        }
    }
    return 0;
}

// Queries per screened chunk with the lo plane in host memory: the screen's partials (part_keys, part_low, part_mm)
// take 88 bytes per query and 256-fact tile; the chunk keeps them within kLoHostPartialBytes in multiples of 128
// queries (one m-tile), at most kQueryChunk (the resident chunk): 1,024 at 2.75 M facts, 128 at 17 M.  A smaller chunk
// reads the hi plane once more per chunk.
constexpr int64_t kLoHostPartialBytes = int64_t(1) << 30;
static int64_t lo_host_chunk(const hrag_t* h) {
    const int64_t per_query = 88 * (int64_t)sim_tc_n_tiles(std::max<int64_t>(h->emb[0].rows, 1));
    return std::min<int64_t>(kQueryChunk, std::max<int64_t>(128, kLoHostPartialBytes / per_query / 128 * 128));
}

// The screen over chunks of lo_host_chunk queries, each raising its own flag; then the flags and the lo bytes the
// gathers read are copied back at once (the one synchronise of the call), and each flagged chunk reruns exactly
// (walk_stage_a: the split K2, lo streamed) over its outputs and counts as a fallback.
static int lo_host_screened_stage_a(hrag_t* h, const PlaneSet& P, int B, const float* q, bool q_on_device, int k,
                                    int* d_top_idx, float* d_top_score, int* d_nvalid, int n_ctas) {
    const int64_t d = h->dim, chunk = lo_host_chunk(h), n_chunks = ceil_div(B, chunk);
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
        HRAG_TRY(walk_stage_a(h, P, nb, x, true, k, d_top_idx + q0 * k, d_top_score + q0 * k, d_nvalid + q0,
                              h->stream, n_ctas, false));
        h->stats.stage_a_fallbacks += 1;
    }
    h->last_mm_rows = n_chunks == 1 ? B : 0;   // mm_fact holds the one chunk's (min, max)
    return 0;
}

int fact_stage_a(hrag_t* h, int B, const float* q, bool q_on_device, int k, int* top_idx, float* top_score,
                 int* nvalid, cudaStream_t s, int n_ctas) {
    if (B == 0) return 0;
    if ((h->world > 1 ? h->n_facts_global : h->emb[0].rows) == 0) {   // no facts: get_fact_scores returns an empty array (HippoRAG.py:1454-1456)
        HRAG_CUDA(cudaMemsetAsync(top_idx, 0xff, (size_t)B * k * sizeof(int), s));
        HRAG_CUDA(cudaMemsetAsync(top_score, 0, (size_t)B * k * sizeof(float), s));
        HRAG_CUDA(cudaMemsetAsync(nvalid, 0, (size_t)B * sizeof(int), s));
        return 0;
    }
    const PlaneSet P = emb_planes(h, 0);
    HRAG_CHECK(!P.streams() || h->sim_mode != HRAG_SIM_FP32, std::string("stage A ") + kNoFp32);
    HRAG_CHECK(!P.streams() || s == h->stream, "internal: fact_stage_a: planes in host memory stream on `stream`");
    h->last_fact_rows = 0;
    h->last_mm_rows = 0;
    const bool screen = fused_stage_a(h, k) && screened(h);
    if (screen && P.on_host[1])
        return lo_host_screened_stage_a(h, P, B, q, q_on_device, k, top_idx, top_score, nvalid, n_ctas);
    return walk_stage_a(h, P, B, q, q_on_device, k, top_idx, top_score, nvalid, s, n_ctas, screen);
}

// K2 writes a score tile up to its 256-column end, clipped at ldS columns from the pointer it is given.  The first
// slice, and a slice that ends on a tile boundary, therefore write in place (S + its first row); a ragged slice after
// the first would spill into the next row, so it goes through `tail` [nb, pad4(rows)] and a 2-D copy.
int sim_scores(hrag_t* h, int which, const float* dQ, int nb, float* S, int64_t ldS, cudaStream_t s, int n_ctas) {
    const PlaneSet P = emb_planes(h, which);
    if (h->sim_mode == HRAG_SIM_FP32 || P.plane[0] == nullptr)   // dim % 8 != 0 has no TMA layout
        return fp32_scores(h, which, dQ, nb, S, ldS, s);
    const int64_t M = h->emb[which].rows;
    const int n_seg = h->sim_mode == HRAG_SIM_BF16X3 ? 4 : 1;
    Buf& tail = h->fplanes.tail;
    HRAG_TRY(split_queries(h, dQ, nb, s));
    if (P.streams()) {
        const int64_t last_rows = M - (ceil_div(M, P.host->slice_rows) - 1) * P.host->slice_rows;
        if (last_rows % kSliceAlign) HRAG_TRY(tail.ensure((size_t)nb * pad4(last_rows) * sizeof(float)));
    }
    auto body = [&](int64_t, int64_t r0, int64_t ns, const void* e_hi, const void* e_lo) -> int {
        const bool ragged = r0 > 0 && ns % kSliceAlign != 0;
        float* out = ragged ? tail.as<float>() : S + r0;
        const int64_t ld = ragged ? pad4(ns) : ldS;
        HRAG_TRY(sim_tc(h->q_hi.p, h->q_lo.p, nb, e_hi, e_lo, ns, h->dim, n_seg, out, ld, nullptr, nullptr, nullptr,
                        n_ctas, s));
        if (ragged)
            HRAG_CUDA(cudaMemcpy2DAsync(S + r0, (size_t)ldS * sizeof(float), out, (size_t)ld * sizeof(float),
                                        (size_t)ns * sizeof(float), (size_t)nb, cudaMemcpyDeviceToDevice, s));
        return 0;
    };
    return stream_slices(h, P, h->dim, 0, M, n_seg == 4, body);
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
    const PlaneSet P = emb_planes(h, 0);
    *on_host = P.on_host[1] ? (P.on_host[0] ? 1 : 2) : 0;
    *slice_rows = h->fplanes.slice_rows;
    *device_bytes = (int64_t)(h->emb[0].hi.cap + h->emb[0].lo.cap + h->fplanes.ring.cap);
    *host_bytes = P.host_bytes();
    return 0;
}

}  // extern "C"
