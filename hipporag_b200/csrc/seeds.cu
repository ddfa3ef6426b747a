// K3 / K4 glue kernels (sm_90a): the reset vector of graph_search_with_fact_entities
// (reference HippoRAG.py:1577-1638 + get_top_k_weights :1505-1542), the passage-score gather
// of run_ppr (:1745) and the layout changes around hrag_ppr.  The reference does this with
// O(N) + O(P) Python loops and md5/dict lookups per query; here the dicts are the integer
// tables uploaded once (SeedTables) and one thread handles one (passage, query) pair.
#include "common.cuh"
#include "kernels.h"

namespace hrag {

namespace {

// V[passage_vid[p], b] = fp32(minmax(S[q0+b, p])) * fp32(pnw)      (HippoRAG.py:1626-1633;
// the product is formed in the score dtype, fp32, as numpy does for float32 * python float)
__global__ void __launch_bounds__(256)
k_seed_passages(int P, int B, int nb, const int* __restrict__ passage_vid, const float* __restrict__ S,
                int64_t ldS, int q0, const float2* __restrict__ minmax, float pnw, float* __restrict__ V) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int p = (int)(t / nb), b = (int)(t % nb);
    if (p >= P) return;
    const float2 mm = __ldg(minmax + q0 + b);
    const float range = mm.y - mm.x;
    const float s = __ldg(S + (size_t)(q0 + b) * ldS + p);
    const float nrm = range == 0.f ? 1.f : __fdiv_rn(s - mm.x, range);   // misc_utils.py:130-139
    V[(size_t)__ldg(passage_vid + p) * B + b] = nrm * pnw;
}

constexpr int kMaxFacts = kMaxKeptFacts;         // 32 (kernels.h): linking_top_k of the reference is configurable
constexpr int kSeedSlots = kSeedSlotsPerQuery;   // a query keeps at most 2 phrases per kept fact (link_top_k = 0 keeps all)

// One thread per query of the chunk: phrase weights of the kept facts -> compact seed list
// seed_vid / seed_w [q, kSeedSlots] (unused slots: vid = -1) and mode[q] (1 = PPR, 0 = DPR fallback).  seed_w is the
// float64 mean the reference stores in node_weights; the fp32 solvers round it where they read it.
__global__ void __launch_bounds__(64)
k_seed_entities(int nq, const int* __restrict__ fact_subj, const int* __restrict__ fact_obj,
                const int* __restrict__ chunk_count, int64_t n_facts, const int* __restrict__ kept_idx,
                const float* __restrict__ kept_score, int k_facts, const uint8_t* __restrict__ dpr_only,
                int link_top_k, int* __restrict__ seed_vid, double* __restrict__ seed_w, int* __restrict__ mode) {
    const int q = blockIdx.x * 64 + threadIdx.x;
    if (q >= nq) return;
    int vid[2 * kMaxFacts];
    double wsum[2 * kMaxFacts];
    int occ[2 * kMaxFacts];
    int n = 0, n_kept = 0;
    for (int i = 0; i < k_facts; ++i) {                       // :1583
        const int f = kept_idx[(size_t)q * k_facts + i];
        if (f < 0 || f >= n_facts) continue;
        ++n_kept;
        const float fs = kept_score[(size_t)q * k_facts + i]; // :1587-1588
        for (int side = 0; side < 2; ++side) {                // :1590 subject, then object
            const int v = side == 0 ? __ldg(fact_subj + f) : __ldg(fact_obj + f);
            if (v < 0) continue;                              // :1597 phrase not in the graph
            float w = fs;
            const int c = __ldg(chunk_count + v);
            if (c > 0) w = __fdiv_rn(fs, (float)c);           // :1600-1601 (fp32, as numpy)
            int j = 0;
            for (; j < n; ++j) if (vid[j] == v) break;
            if (j == n) { vid[n] = v; wsum[n] = 0.0; occ[n] = 0; ++n; }
            wsum[j] += (double)w;                             // :1603 (float64 accumulator)
            occ[j] += 1;                                      // :1604
        }
    }
    const bool flagged = dpr_only != nullptr && dpr_only[q] != 0;
    for (int r = 0; r < kSeedSlots; ++r) { seed_vid[(size_t)q * kSeedSlots + r] = -1; seed_w[(size_t)q * kSeedSlots + r] = 0.0; }
    if (!flagged && n_kept > 0) {
        for (int j = 0; j < n; ++j) wsum[j] /= (double)occ[j];  // :1608 mean over occurrences
        int keep = (link_top_k > 0 && link_top_k < n) ? link_top_k : n;   // :1620, :1528
        for (int r = 0; r < keep; ++r) {                      // selection: weight desc, vertex id asc
            int best = -1;
            for (int j = 0; j < n; ++j) {
                if (occ[j] == 0) continue;
                if (best < 0 || wsum[j] > wsum[best] || (wsum[j] == wsum[best] && vid[j] < vid[best])) best = j;
            }
            if (best < 0) break;
            seed_vid[(size_t)q * kSeedSlots + r] = vid[best];
            seed_w[(size_t)q * kSeedSlots + r] = wsum[best];
            occ[best] = 0;
        }
    }
    // :467-469 no fact survived -> DPR; a zero-mass phrase set still runs PPR on the passage
    // weights alone (the reference asserts sum(node_weights) > 0, which those satisfy).
    mode[q] = (!flagged && n_kept > 0) ? 1 : 0;
}

// V[seed_vid, b] += seed_w for the nb queries of one PPR sub-batch (:1638 phrase + passage weights)
__global__ void __launch_bounds__(256)
k_seed_scatter(int B, int nb, int q0, const int* __restrict__ seed_vid, const double* __restrict__ seed_w,
               float* __restrict__ V) {
    const int t = blockIdx.x * 256 + threadIdx.x;
    const int b = t / kSeedSlots, r = t % kSeedSlots;
    if (b >= nb) return;
    const int v = seed_vid[(size_t)(q0 + b) * kSeedSlots + r];
    if (v >= 0) V[(size_t)v * B + b] += (float)seed_w[(size_t)(q0 + b) * kSeedSlots + r];   // distinct (v, b) per thread
}

// ---- the float64 reset of stage B (hrag_stage_b_f64), in the reference's dtypes -------------------------------
// R [nb, N] is the host-layout staging reset_to_state_f64 reads (zeroed by the caller).
// R[b, passage_vid[p]] = double(fp32(minmax(S[q0+b, p])) * fp32(pnw)): k_seed_passages' fp32 product, stored into the
// float64 passage_weights array (HippoRAG.py:1626-1633)
__global__ void __launch_bounds__(256)
k_seed_passages_f64(int P, int nb, int N, const int* __restrict__ passage_vid, const float* __restrict__ S,
                    int64_t ldS, int q0, const float2* __restrict__ minmax, float pnw, double* __restrict__ R) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int p = (int)(t / nb), b = (int)(t % nb);
    if (p >= P) return;
    const float2 mm = __ldg(minmax + q0 + b);
    const float range = mm.y - mm.x;
    const float s = __ldg(S + (size_t)(q0 + b) * ldS + p);
    const float nrm = range == 0.f ? 1.f : __fdiv_rn(s - mm.x, range);
    R[(size_t)b * N + __ldg(passage_vid + p)] = (double)(nrm * pnw);
}

// R[b, seed_vid] += seed_w: phrase_weights + passage_weights in float64 (:1638)
__global__ void __launch_bounds__(256)
k_seed_scatter_f64(int nb, int N, int q0, const int* __restrict__ seed_vid, const double* __restrict__ seed_w,
                   double* __restrict__ R) {
    const int t = blockIdx.x * 256 + threadIdx.x;
    const int b = t / kSeedSlots, r = t % kSeedSlots;
    if (b >= nb) return;
    const int v = seed_vid[(size_t)(q0 + b) * kSeedSlots + r];
    if (v >= 0) R[(size_t)b * N + v] += seed_w[(size_t)(q0 + b) * kSeedSlots + r];   // distinct (v, b) per thread
}

// out[b, p] (row stride ld) for the nb queries [q0, q0 + nb) of a sub-batch: PPR rows pi = X[passage_vid[p], b] /
// xsum[b] in float64 (:1745); DPR-fallback rows the fp32 min-maxed score of k_gather_passage_scores, widened.
__global__ void __launch_bounds__(256)
k_gather_passage_scores_f64(int P, int B, int nb, int q0, const int* __restrict__ passage_vid,
                            const double* __restrict__ X, const double* __restrict__ xsum, const int* __restrict__ mode,
                            const float2* __restrict__ minmax, const float* __restrict__ S, int64_t ldS,
                            double* __restrict__ out, int64_t ld) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int p = (int)(t / nb), b = (int)(t % nb);
    if (p >= P) return;
    double v;
    if (mode[q0 + b]) {
        v = X[(size_t)__ldg(passage_vid + p) * B + b] / xsum[b];
    } else {
        const float2 mm = __ldg(minmax + q0 + b);
        const float range = mm.y - mm.x;
        v = range == 0.f ? 1.f : __fdiv_rn(__ldg(S + (size_t)(q0 + b) * ldS + p) - mm.x, range);
    }
    out[(size_t)b * ld + p] = v;
}

__global__ void __launch_bounds__(256)
k_gather_passage_scores(int P, int B, int nb, int q0, const int* __restrict__ passage_vid,
                        const float* __restrict__ Z, const double* __restrict__ sums,
                        const int* __restrict__ mode, const float2* __restrict__ minmax, float* S, int64_t ldS) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int p = (int)(t / nb), b = (int)(t % nb);
    if (p >= P) return;
    float* dst = S + (size_t)(q0 + b) * ldS + p;
    if (mode[q0 + b]) {
        const float z = __ldg(Z + (size_t)__ldg(passage_vid + p) * B + b);   // HippoRAG.py:1745
        *dst = __fdiv_rn(z, (float)sums[b]);                                 // pi = z / ||z||_1
    } else {
        const float2 mm = __ldg(minmax + q0 + b);                            // DPR fallback :1498
        const float range = mm.y - mm.x;
        *dst = range == 0.f ? 1.f : __fdiv_rn(*dst - mm.x, range);
    }
}

// V[n, b] = sanitised R[b, n]  (run_ppr, HippoRAG.py:1735)
__global__ void __launch_bounds__(256)
k_reset_to_state(const float* __restrict__ R, int nb, int N, int B, float* __restrict__ V) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int n = (int)(t / B), b = (int)(t % B);
    if (n >= N) return;
    float r = 0.f;
    if (b < nb) {
        r = R[(size_t)b * N + n];
        if (!(r >= 0.f)) r = 0.f;    // NaN and negatives -> 0
    }
    V[(size_t)n * B + b] = r;
}

__global__ void __launch_bounds__(256)
k_state_to_scores(const float* __restrict__ Z, int nb, int N, int B, const double* __restrict__ sums,
                  float* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int n = (int)(t / nb), b = (int)(t % nb);
    if (n >= N) return;
    out[(size_t)b * N + n] = __fdiv_rn(Z[(size_t)n * B + b], (float)sums[b]);
}

}  // namespace

int seed_passages(const SeedTables& t, int B, int nb, const float* S, int64_t ldS, int q0, const float2* minmax,
                  float pnw, float* V, cudaStream_t stream) {
    if (t.n_passages == 0 || nb == 0) return 0;
    const int64_t total = (int64_t)t.n_passages * nb;
    k_seed_passages<<<(unsigned)ceil_div(total, 256), 256, 0, stream>>>(t.n_passages, B, nb, t.passage_vid, S, ldS,
                                                                         q0, minmax, pnw, V);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int seed_entities(const SeedTables& t, int nq, const int* kept_idx, const float* kept_score, int k_facts,
                  const uint8_t* dpr_only, int link_top_k, int* seed_vid, double* seed_w, int* mode,
                  cudaStream_t stream) {
    HRAG_CHECK(k_facts >= 0 && k_facts <= kMaxFacts, "seed_entities: at most 32 kept facts per query");
    if (nq == 0) return 0;
    k_seed_entities<<<(unsigned)ceil_div(nq, 64), 64, 0, stream>>>(nq, t.fact_subj_vid, t.fact_obj_vid,
                                                                    t.ent_chunk_count, t.n_facts, kept_idx,
                                                                    kept_score, k_facts, dpr_only, link_top_k,
                                                                    seed_vid, seed_w, mode);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int seed_scatter(int B, int nb, int q0, const int* seed_vid, const double* seed_w, float* V, cudaStream_t stream) {
    if (nb == 0) return 0;
    k_seed_scatter<<<(unsigned)ceil_div(nb * kSeedSlots, 256), 256, 0, stream>>>(B, nb, q0, seed_vid, seed_w, V);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int seed_reset_f64(const SeedTables& t, int nb, int N, int q0, const float* S, int64_t ldS, const float2* minmax,
                   float pnw, const int* seed_vid, const double* seed_w, double* R, cudaStream_t stream) {
    if (nb == 0) return 0;
    HRAG_CUDA(cudaMemsetAsync(R, 0, (size_t)nb * N * sizeof(double), stream));
    if (t.n_passages > 0) {
        const int64_t total = (int64_t)t.n_passages * nb;
        k_seed_passages_f64<<<(unsigned)ceil_div(total, 256), 256, 0, stream>>>(t.n_passages, nb, N, t.passage_vid, S,
                                                                                 ldS, q0, minmax, pnw, R);
        count_launch(1);
    }
    k_seed_scatter_f64<<<(unsigned)ceil_div(nb * kSeedSlots, 256), 256, 0, stream>>>(nb, N, q0, seed_vid, seed_w, R);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int gather_passage_scores_f64(const SeedTables& t, int B, int nb, int q0, const double* X, const double* xsum,
                              const int* mode, const float2* minmax, const float* S, int64_t ldS, double* out,
                              int64_t ld, cudaStream_t stream) {
    if (t.n_passages == 0 || nb == 0) return 0;
    const int64_t total = (int64_t)t.n_passages * nb;
    k_gather_passage_scores_f64<<<(unsigned)ceil_div(total, 256), 256, 0, stream>>>(t.n_passages, B, nb, q0,
                                                                                     t.passage_vid, X, xsum, mode,
                                                                                     minmax, S, ldS, out, ld);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int gather_passage_scores(const SeedTables& t, int B, int nb, int q0, const float* Z, const double* sums,
                          const int* mode, const float2* minmax, float* S, int64_t ldS, cudaStream_t stream) {
    if (t.n_passages == 0 || nb == 0) return 0;
    const int64_t total = (int64_t)t.n_passages * nb;
    k_gather_passage_scores<<<(unsigned)ceil_div(total, 256), 256, 0, stream>>>(t.n_passages, B, nb, q0,
                                                                                 t.passage_vid, Z, sums, mode,
                                                                                 minmax, S, ldS);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int reset_to_state(const float* R, int nb, int N, int B, float* V, cudaStream_t stream) {
    const int64_t total = (int64_t)N * B;
    k_reset_to_state<<<(unsigned)ceil_div(total, 256), 256, 0, stream>>>(R, nb, N, B, V);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

int state_to_scores(const float* Z, int nb, int N, int B, const double* sums, float* out, cudaStream_t stream) {
    const int64_t total = (int64_t)N * nb;
    k_state_to_scores<<<(unsigned)ceil_div(total, 256), 256, 0, stream>>>(Z, nb, N, B, sums, out);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace hrag
