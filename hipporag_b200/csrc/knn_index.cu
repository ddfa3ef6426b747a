// The synonymy KNN of add_synonymy_edges (reference HippoRAG.py:959-1020) kept on the device between calls.
//
// HippoRAG.index() runs add_synonymy_edges after every insert, and it asks retrieve_knn for the neighbours of every
// entity among every entity (:986-992).  The entity store only appends on insert and compacts in order on delete
// (embedding_store.py:176-191), so from one call to the next the keys are the old keys minus some, in their old order,
// followed by new keys.  hrag_knn_index_update applies such a change to the lists it keeps instead of recomputing all
// pairs, and ends with what hrag_knn_threshold (+ the overflow redo of knn.py) gives over the new rows, bit for bit:
//   1. upload + split the new rows chunk by chunk; before a chunk overwrites its rows in place, every kept row's new
//      bf16 hi / lo is compared with the planes held at its old row (kept_from[i] >= i: no chunk overwrites a row a
//      later chunk still reads).  The planes are all a score depends on, so equal planes mean equal scores; a
//      mismatch (a kept key's vector changed) rebuilds from the new planes;
//   2. every kept list is relabelled old -> new and loses its deleted keys (order kept), then the lists are compacted
//      in place; a list that loses a listed key and does not hold every key >= thr is refilled in step 4;
//   3. the kept rows (read from the planes) against the new keys [n_kept, rows): threshold GEMM + sort_candidates on
//      that key slice, then k_knn_merge keeps the first kmax of (list u candidates) by (score desc, id asc);
//   4. refilled rows and the new rows against all keys: their lists are replaced;
//   5. a row whose candidates overflow the 512-entry buffer is redone by the score GEMM + row_topk over the same key
//      range and merged the same way.
// Scores come from the same K2 accumulators whatever the tile a pair falls in, so the lists equal a fresh all-pairs
// run.  Every argument is checked before the index is touched; a failure after that clears it (the next call builds).
//
// Planes over the hrag_knn_set_memory budget live in pinned host memory (KnnIndex::host); the lists stay on the
// device.  Steps 3 - 5 walk the keys with the walker of the fact planes (stream_slices, handle.h), one slice on device
// planes: the query rows are read in place or gathered (device planes, passes of kChunk) or staged (host planes,
// passes of up to kHostPass), each query's 512 candidates persist across the key slices (moved to rows of the key
// range after every slice but the first), and in step 5 the overflowing rows are scored one key slice at a time and
// each slice's exact top-k is folded into the row's list by k_knn_merge.  A (score desc, id asc) fold of per-slice
// top-kmax lists is the top-kmax of their union, so the lists do not depend on the placement, bit for bit.  In step 1
// host rows are split through the ring by planes_fill, and before a chunk is written back the held rows its kept rows
// come from are copied into ring half 0 and compared there.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "handle.h"

namespace hrag {
namespace {

constexpr int kThreads = 256;
constexpr int kMergeWarps = 4;                      // rows per k_knn_merge block (one warp each)
constexpr int64_t kChunk = 1024;                    // queries per threshold GEMM, as in hrag_knn_threshold
constexpr size_t kUploadBytes = (size_t)64 << 20;   // fp32 rows per upload chunk
constexpr double kRedoBytes = 2e9;                  // score matrix of one overflow-redo chunk
constexpr int64_t kHostPass = 65536;                // host planes: queries staged per pass over the keys (their planes
                                                    // and 512 candidates each, 4 KB + 4 dim bytes a query)

int blocks_for(int64_t n) { return (int)ceil_div(std::max<int64_t>(n, 1), kThreads); }

__device__ __forceinline__ int64_t thread_index() { return blockIdx.x * (int64_t)blockDim.x + threadIdx.x; }

// *mismatch = 1 when a kept row's new planes (rows r0 .. r0 + n_rows of the chunk) differ from the planes held at its
// old row kept_from[r]; rows are w16 16-byte words long
__global__ void k_knn_compare(int64_t n_rows, int64_t w16, int64_t r0, const int* __restrict__ kept_from,
                              const int4* __restrict__ nhi, const int4* __restrict__ nlo, const int4* __restrict__ ohi,
                              const int4* __restrict__ olo, int* __restrict__ mismatch) {
    const int64_t i = thread_index();
    if (i >= n_rows * w16) return;
    const int64_t r = i / w16, c = i - r * w16;
    const int64_t o = (int64_t)kept_from[r0 + r] * w16 + c;
    const int4 a = nhi[i], b = ohi[o], x = nlo[i], y = olo[o];
    if (a.x != b.x || a.y != b.y || a.z != b.z || a.w != b.w || x.x != y.x || x.y != y.y || x.z != y.z || x.w != y.w)
        *mismatch = 1;
}

// map[kept_from[i]] = i (map pre-filled with -1: deleted rows)
__global__ void k_knn_map(int64_t n_kept, const int* __restrict__ kept_from, int* __restrict__ map) {
    const int64_t i = thread_index();
    if (i < n_kept) map[kept_from[i]] = (int)i;
}

// Host planes: query b's candidates appended by the threshold GEMM over one key slice (slots prev[b] .. count[b],
// below the cap) carry their row in the slice; + off moves them to rows of the key range the query set is scored on.
__global__ void k_knn_shift(uint64_t* __restrict__ cand, const int* __restrict__ count, const int* __restrict__ prev,
                            uint32_t off) {
    const int b = blockIdx.x;
    const int end = min(count[b], kCandidateCap);
    uint64_t* c = cand + (size_t)b * kCandidateCap;
    for (int j = prev[b] + threadIdx.x; j < end; j += blockDim.x)
        c[j] = rank_key(key_score(c[j]), key_index(c[j]) + off);
}

// One warp per kept row i: the list at its old row kept_from[i] is relabelled through map in place, deleted keys
// dropped and the order kept.  A list that lost a listed key and is not complete is flagged for a refill (and i
// appended to `refill`): the keys after its last entry are unknown.  One that lost only unlisted keys is still the
// first kmax of what is left.
__global__ void k_knn_relabel(int64_t n_kept, const int* __restrict__ kept_from, const int* __restrict__ map,
                              int* __restrict__ ids, float* __restrict__ scores, int width, int kmax,
                              int* __restrict__ refill, int* __restrict__ n_refill) {
    const int64_t i = thread_index() >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n_kept) return;
    int* lid = ids + (int64_t)kept_from[i] * width;
    float* lsc = scores + (int64_t)kept_from[i] * width;
    int out = 0;
    bool lost = false;
    for (int j0 = 0; j0 < kmax; j0 += 32) {
        const int j = j0 + lane;
        const int id = j < kmax ? lid[j] : -1;
        const float s = j < kmax ? lsc[j] : 0.f;
        const int nid = id >= 0 ? map[id] : -1;
        const unsigned keep = __ballot_sync(0xffffffffu, nid >= 0);
        lost |= __any_sync(0xffffffffu, id >= 0 && nid < 0) != 0;
        __syncwarp();   // the whole 32-entry window is read before any of it is written
        if (nid >= 0) {
            const int p = out + __popc(keep & ((1u << lane) - 1u));
            lid[p] = nid;
            lsc[p] = s;
        }
        out += __popc(keep);
        __syncwarp();
    }
    for (int p = out + lane; p < kmax; p += 32) { lid[p] = -1; lsc[p] = 0.f; }
    if (lane == 0 && lost && !(lid[kmax] & kKnnComplete)) {
        lid[kmax] |= kKnnRefill;
        refill[atomicAdd(n_refill, 1)] = (int)i;
    }
}

// entries of x[0 .. n) (descending, distinct) greater than key
__device__ __forceinline__ int count_greater(const uint64_t* x, int n, uint64_t key) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (x[mid] > key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// One warp per query b < n: the list of row t = rows ? rows[b] : r0 + b becomes the first kmax of (its list, when
// `merge`) u (b's candidates, ids + id_offset) by (score desc, id asc), each element placed by its rank in the other
// list.  found != null: the candidates are sort_candidates' (found[b] keys cleared thr; > the 512-entry cap: the row
// is left to the overflow redo); found == null: they are row_topk's over the key range, of which the entries >= thr
// count, and the list is not complete.  With `merge`, rows flagged for a refill are left alone (they are replaced).
__global__ void __launch_bounds__(32 * kMergeWarps)
k_knn_merge(int n, const int* __restrict__ rows, int64_t r0, const int* __restrict__ cand_ids,
            const float* __restrict__ cand_scores, int cstride, const int* __restrict__ found, int64_t id_offset,
            float thr, int merge, int* __restrict__ ids, float* __restrict__ scores, int width, int kmax) {
    extern __shared__ uint64_t knn_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * kMergeWarps + warp;
    if (b >= n) return;
    uint64_t* A = knn_smem + (size_t)warp * 2 * kmax;
    uint64_t* Bk = A + kmax;
    const int64_t t = rows ? rows[b] : r0 + b;
    int* lid = ids + t * width;
    float* lsc = scores + t * width;
    const int flags = lid[kmax];
    const int cnt = found ? found[b] : 0;
    if ((found && cnt > kCandidateCap) || (merge && (flags & kKnnRefill))) return;
    int nb = 0, na = 0;
    for (int j0 = 0; j0 < cstride; j0 += 32) {   // valid candidates are a prefix (sorted, -1 padded)
        const int j = j0 + lane;
        const int id = j < cstride ? cand_ids[(size_t)b * cstride + j] : -1;
        const float s = j < cstride ? cand_scores[(size_t)b * cstride + j] : 0.f;
        const bool ok = id >= 0 && (found != nullptr || s >= thr);
        if (ok) Bk[j] = rank_key(s, (uint32_t)(id + id_offset));
        nb += __popc(__ballot_sync(0xffffffffu, ok));
    }
    if (merge)
        for (int j0 = 0; j0 < kmax; j0 += 32) {
            const int j = j0 + lane;
            const int id = j < kmax ? lid[j] : -1;
            if (id >= 0) A[j] = rank_key(lsc[j], (uint32_t)id);
            na += __popc(__ballot_sync(0xffffffffu, id >= 0));
        }
    __syncwarp();   // both inputs are in shared memory: the list can be overwritten
    for (int i = lane; i < na; i += 32) {
        const int p = i + count_greater(Bk, nb, A[i]);
        if (p < kmax) { lid[p] = (int)key_index(A[i]); lsc[p] = key_score(A[i]); }
    }
    for (int j = lane; j < nb; j += 32) {
        const int p = j + count_greater(A, na, Bk[j]);
        if (p < kmax) { lid[p] = (int)key_index(Bk[j]); lsc[p] = key_score(Bk[j]); }
    }
    for (int p = (na + nb < kmax ? na + nb : kmax) + lane; p < kmax; p += 32) { lid[p] = -1; lsc[p] = 0.f; }
    if (lane == 0) {
        const bool complete = found != nullptr && (!merge || (flags & kKnnComplete)) && na + cnt <= kmax;
        lid[kmax] = complete ? kKnnComplete : 0;
    }
}

int launch_merge(hrag_t* h, int n, const int* rows, int64_t r0, const int* cand_ids, const float* cand_scores,
                 int cstride, const int* found, int64_t id_offset, bool merge) {
    if (n == 0) return 0;
    KnnIndex& K = h->knn;
    const size_t smem = (size_t)kMergeWarps * 2 * K.kmax * sizeof(uint64_t);   // <= 32 KB at kmax = 512
    k_knn_merge<<<(unsigned)ceil_div(n, kMergeWarps), 32 * kMergeWarps, smem, h->stream>>>(
        n, rows, r0, cand_ids, cand_scores, cstride, found, id_offset, K.thr, merge ? 1 : 0, K.ids.as<int>(),
        K.scores.as<float>(), K.width, K.kmax);
    count_launch(1);
    HRAG_CUDA(cudaGetLastError());
    return 0;
}

// Scratch of one update call (freed on return).
struct Scratch { Buf q_hi, q_lo, cand, count, prev, out_ids, out_scores, found, rows, redo_rows, S; };

// Host planes: rows of the pinned planes into dense device rows dst_hi / dst_lo (row i = list[i], or r0 + i without a
// list), one copy per run of consecutive rows.
int stage_rows(hrag_t* h, const PlaneSet& P, size_t rb, const int* list, int64_t r0, int64_t n, char* dst_hi,
               char* dst_lo) {
    for (int64_t i = 0; i < n;) {
        const int64_t first = list ? list[i] : r0 + i;
        int64_t j = list ? i + 1 : n;
        while (j < n && list[j] == list[j - 1] + 1) ++j;
        const size_t at = (size_t)first * rb, bytes = (size_t)(j - i) * rb;
        HRAG_TRY(h2d(h, dst_hi + (size_t)i * rb, P.plane[0] + at, bytes));
        HRAG_TRY(h2d(h, dst_lo + (size_t)i * rb, P.plane[1] + at, bytes));
        i = j;
    }
    return 0;
}

// Query rows i < n (row list[i] (host; d_list: the same on the device), or r0 + i) of the planes, for the GEMMs:
// resident rows without a list are read in place, with one gathered into s.q_hi / s.q_lo; host rows are staged there.
int query_rows(hrag_t* h, Scratch& s, const PlaneSet& P, const int* list, const int* d_list, int64_t r0, int64_t n,
               const void** qh, const void** ql) {
    const size_t rb = (size_t)h->knn.dim * 2;
    *qh = s.q_hi.p;
    *ql = s.q_lo.p;
    if (P.streams()) return stage_rows(h, P, rb, list, r0, n, s.q_hi.as<char>(), s.q_lo.as<char>());
    if (list) {
        HRAG_TRY(gather_rows(h, P.plane[0], rb, d_list, n, s.q_hi.p));
        return gather_rows(h, P.plane[1], rb, d_list, n, s.q_lo.p);
    }
    *qh = P.plane[0] + (size_t)r0 * rb;
    *ql = P.plane[1] + (size_t)r0 * rb;
    return 0;
}

// The query rows (`list` (host) of n_q rows, or the range [r0, r0 + n_q)) against keys [key0, key0 + M): each
// query's list becomes the first kmax of its keys >= thr there, merged with the list it has when `merge`.  Passes of
// kChunk query rows on resident planes, of up to kHostPass staged rows on host planes, each walking the key slices
// once; a query's candidate buffer and count persist across the slices (moved to rows of the key range after each
// slice but the first), so the overflow test sees every key >= thr in the range, as one GEMM over it does.
int run_queries(hrag_t* h, Scratch& s, const std::vector<int>* list, int64_t r0, int64_t n_q, int64_t key0, int64_t M,
                bool merge) {
    if (n_q == 0 || M == 0) return 0;
    KnnIndex& K = h->knn;
    const PlaneSet P = plane_set(K.hi, K.lo, &K.host);
    cudaStream_t st = h->stream;
    const size_t rb = (size_t)K.dim * 2;
    const int64_t Qp = P.streams() ? std::min(n_q, kHostPass) : kChunk;
    HRAG_TRY(s.q_hi.ensure((size_t)Qp * rb));
    HRAG_TRY(s.q_lo.ensure((size_t)Qp * rb));
    HRAG_TRY(s.cand.ensure((size_t)Qp * kCandidateCap * sizeof(uint64_t)));
    HRAG_TRY(s.count.ensure((size_t)Qp * 4));
    if (P.streams()) HRAG_TRY(s.prev.ensure((size_t)Qp * 4));
    HRAG_TRY(s.found.ensure((size_t)Qp * 4));
    HRAG_TRY(s.out_ids.ensure((size_t)kChunk * K.kmax * 4));
    HRAG_TRY(s.out_scores.ensure((size_t)kChunk * K.kmax * 4));
    if (list) HRAG_TRY(s.rows.ensure((size_t)std::min(n_q, Qp) * 4));
    uint64_t* cand = s.cand.as<uint64_t>();
    int* count = s.count.as<int>();
    std::vector<int> found((size_t)Qp), over;   // over: positions in the query set whose candidates overflowed
    for (int64_t p0 = 0; p0 < n_q; p0 += Qp) {
        const int64_t np = std::min(Qp, n_q - p0);
        const int* plist = list ? list->data() + p0 : nullptr;
        if (list) HRAG_TRY(h2d(h, s.rows.p, plist, (size_t)np * 4));
        const void *q_hi = nullptr, *q_lo = nullptr;
        HRAG_TRY(query_rows(h, s, P, plist, s.rows.as<int>(), r0 + p0, np, &q_hi, &q_lo));
        HRAG_CUDA(cudaMemsetAsync(count, 0, (size_t)np * 4, st));
        auto slice = [&](int64_t, int64_t a, int64_t ns, const void* e_hi, const void* e_lo) -> int {
            for (int64_t q0 = 0; q0 < np; q0 += kChunk) {
                const int nb = (int)std::min<int64_t>(kChunk, np - q0);
                if (a > key0)
                    HRAG_CUDA(cudaMemcpyAsync(s.prev.as<int>() + q0, count + q0, (size_t)nb * 4,
                                              cudaMemcpyDeviceToDevice, st));
                HRAG_TRY(sim_tc_threshold(static_cast<const char*>(q_hi) + (size_t)q0 * rb,
                                          static_cast<const char*>(q_lo) + (size_t)q0 * rb, nb, e_hi, e_lo, ns, K.dim,
                                          4, K.thr, cand + (size_t)q0 * kCandidateCap, count + q0, kCandidateCap,
                                          h->num_sms, st));
                if (a > key0) {
                    k_knn_shift<<<nb, 64, 0, st>>>(cand + (size_t)q0 * kCandidateCap, count + q0,
                                                   s.prev.as<int>() + q0, (uint32_t)(a - key0));
                    count_launch(1);
                    HRAG_CUDA(cudaGetLastError());
                }
            }
            return 0;
        };
        {
            StageTimer tm(h, ST_SIM_FACT);
            HRAG_TRY(stream_slices(h, P, K.dim, key0, key0 + M, true, slice));
        }
        {
            StageTimer tm(h, ST_TOPK);
            for (int64_t q0 = 0; q0 < np; q0 += kChunk) {
                const int nb = (int)std::min<int64_t>(kChunk, np - q0);
                HRAG_TRY(sort_candidates(cand + (size_t)q0 * kCandidateCap, count + q0, nb, kCandidateCap, K.kmax,
                                         s.out_ids.as<int>(), s.out_scores.as<float>(), s.found.as<int>() + q0, st));
                HRAG_TRY(launch_merge(h, nb, list ? s.rows.as<int>() + q0 : nullptr, r0 + p0 + q0, s.out_ids.as<int>(),
                                      s.out_scores.as<float>(), K.kmax, s.found.as<int>() + q0, key0, merge));
            }
        }
        HRAG_TRY(d2h(h, found.data(), s.found.p, (size_t)np * 4));
        HRAG_CUDA(cudaStreamSynchronize(st));
        for (int64_t b = 0; b < np; ++b)
            if (found[b] > kCandidateCap) over.push_back((int)(p0 + b));
    }
    if (over.empty()) return 0;

    // the overflow redo, one key slice at a time: the slice's scores and exact top-k, folded into the list (the first
    // slice replaces it unless `merge`), cut at thr
    std::vector<int> tgt(over.size());
    for (size_t i = 0; i < over.size(); ++i) tgt[i] = list ? (*list)[over[i]] : (int)(r0 + over[i]);
    const int64_t n_over = (int64_t)tgt.size(), ld = (P.streams() ? P.host->slice_rows + 3 : M + 3) & ~(int64_t)3;
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(kChunk, (int64_t)(kRedoBytes / (4.0 * (double)ld))));
    HRAG_TRY(s.redo_rows.ensure((size_t)n_over * 4));
    HRAG_TRY(h2d(h, s.redo_rows.p, tgt.data(), (size_t)n_over * 4));
    HRAG_TRY(s.S.ensure((size_t)std::min(chunk, n_over) * ld * 4));
    for (int64_t o0 = 0; o0 < n_over; o0 += chunk) {
        const int nb = (int)std::min<int64_t>(chunk, n_over - o0);
        const int* r = s.redo_rows.as<int>() + o0;
        const void *q_hi = nullptr, *q_lo = nullptr;
        HRAG_TRY(query_rows(h, s, P, tgt.data() + o0, r, 0, nb, &q_hi, &q_lo));
        auto slice = [&](int64_t sl, int64_t a, int64_t ns, const void* e_hi, const void* e_lo) -> int {
            const int64_t lds = (ns + 3) & ~(int64_t)3;
            const int k = (int)std::min<int64_t>(K.kmax, ns);
            {
                StageTimer tm(h, ST_SIM_FACT);
                HRAG_TRY(sim_tc(q_hi, q_lo, nb, e_hi, e_lo, ns, K.dim, 4, s.S.as<float>(), lds, nullptr, nullptr,
                                nullptr, h->num_sms, st));
            }
            StageTimer tm(h, ST_TOPK);
            HRAG_TRY(row_topk(s.S.as<float>(), nb, ns, lds, k, s.out_ids.as<int>(), s.out_scores.as<float>(), st));
            return launch_merge(h, nb, r, 0, s.out_ids.as<int>(), s.out_scores.as<float>(), k, nullptr, a,
                                merge || sl > 0);
        };
        HRAG_TRY(stream_slices(h, P, K.dim, key0, key0 + M, true, slice));
    }
    HRAG_CUDA(cudaStreamSynchronize(st));   // the scratch is freed on return
    return 0;
}

// Step 1 on host planes: the new rows are split through the ring into the pinned planes (planes_fill).  A chunk's kept
// rows come from held rows kept_from[r .. r + nc) (ascending, >= r, so no later chunk reads a row this one writes):
// before the chunk overwrites rows [r, r + m) they are copied into ring half 0, at most slice_rows at a time, and
// compared by k_knn_compare; *mismatch (device) is set when a kept row's planes changed.
int fill_host(hrag_t* h, int64_t rows, int dim, const float* emb, bool on_device, int64_t n_kept,
              const int64_t* kept_from, const int* d_kept, int* mismatch) {
    HostPlanes& P = h->knn.host;
    const size_t rb = (size_t)dim * 2;
    const int64_t w16 = (int64_t)(rb / 16), S = P.slice_rows;
    int4* ring_hi = P.ring.as<int4>();
    int4* ring_lo = ring_hi + S * w16;
    auto verify = [&](int64_t r, int64_t m, const char* nhi, const char* nlo) -> int {
        const int64_t nc = std::max<int64_t>(0, std::min(m, n_kept - r));
        for (int64_t i = 0; i < nc;) {
            const int64_t a = kept_from[r + i];
            int64_t j = i + 1;
            while (j < nc && kept_from[r + j] < a + S) ++j;
            const size_t bytes = (size_t)(kept_from[r + j - 1] + 1 - a) * rb;
            HRAG_TRY(h2d(h, ring_hi, static_cast<const char*>(P.hi) + (size_t)a * rb, bytes));
            HRAG_TRY(h2d(h, ring_lo, static_cast<const char*>(P.lo) + (size_t)a * rb, bytes));
            // held row a is the first of the copy: the base moved back by a rows lets kept_from[] index it
            k_knn_compare<<<blocks_for((j - i) * w16), kThreads, 0, h->stream>>>(
                j - i, w16, r + i, d_kept, reinterpret_cast<const int4*>(nhi) + i * w16,
                reinterpret_cast<const int4*>(nlo) + i * w16, ring_hi - a * w16, ring_lo - a * w16, mismatch);
            count_launch(1);
            HRAG_CUDA(cudaGetLastError());
            i = j;
        }
        return 0;
    };
    return planes_fill(h, plane_set(h->knn.hi, h->knn.lo, &P), dim, 0, rows, emb, on_device, verify);
}

// The planes of an index of `rows` rows, the first `keep` of them kept, placed in pinned host memory with a ring of
// slice_rows-row halves: capacity grows by half at a time; resident planes move to the host with one copy.
int place_host(hrag_t* h, int64_t keep, int64_t rows, int dim, int64_t slice_rows) {
    KnnIndex& K = h->knn;
    HostPlanes& P = K.host;
    const size_t rb = (size_t)dim * 2, need = (size_t)std::max<int64_t>({rows, keep, 1}) * rb;   // old rows too
    if (!P.held() || need > P.plane_bytes) {
        HostPlanes np;
        HRAG_TRY(np.alloc(P.held() ? std::max(need, P.plane_bytes + P.plane_bytes / 2) : need, slice_rows, dim));
        if (keep && P.held()) {
            std::memcpy(np.hi, P.hi, (size_t)keep * rb);
            std::memcpy(np.lo, P.lo, (size_t)keep * rb);
        }
        P = std::move(np);
    } else if (P.slice_rows != slice_rows) {   // the budget changed: a new ring
        P.ring.reset();
        HRAG_TRY(P.ring.ensure((size_t)2 * slice_rows * dim * 4));
        P.slice_rows = slice_rows;
    }
    if (K.hi.p) {
        if (keep) {
            HRAG_TRY(d2h(h, P.hi, K.hi.p, (size_t)keep * rb));
            HRAG_TRY(d2h(h, P.lo, K.lo.p, (size_t)keep * rb));
            HRAG_CUDA(cudaStreamSynchronize(h->stream));
        }
        K.hi.reset();
        K.lo.reset();
    }
    return 0;
}

// The planes of an index of `rows` rows, the first `keep` of them kept, placed on the device: host planes move back
// with one copy, resident ones grow by half at a time.
int place_device(hrag_t* h, int64_t keep, int64_t rows, int dim) {
    KnnIndex& K = h->knn;
    const size_t rb = (size_t)dim * 2;
    if (!K.host.held()) {
        HRAG_TRY(grow_keep(h, K.hi, (size_t)keep * rb, (size_t)rows * rb));
        return grow_keep(h, K.lo, (size_t)keep * rb, (size_t)rows * rb);
    }
    Buf hi, lo;   // the kept old rows are read until step 1 has compacted them: room for both counts
    HRAG_TRY(hi.ensure((size_t)std::max<int64_t>({rows, keep, 1}) * rb));
    HRAG_TRY(lo.ensure((size_t)std::max<int64_t>({rows, keep, 1}) * rb));
    if (keep) {
        HRAG_TRY(h2d(h, hi.p, K.host.hi, (size_t)keep * rb));
        HRAG_TRY(h2d(h, lo.p, K.host.lo, (size_t)keep * rb));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
    }
    K.hi = std::move(hi);
    K.lo = std::move(lo);
    K.host.release();
    return 0;
}

}  // namespace
}  // namespace hrag

using namespace hrag;

extern "C" {

int hrag_knn_index_update(hrag_t* h, int64_t rows, int32_t dim, const float* emb, int on_device, int64_t n_kept,
                          const int64_t* kept_from, float min_score, int32_t kmax, int32_t* mode) {
    const std::string who = "hrag_knn_index_update";
    HRAG_CHECK(h && mode, who + ": null argument");
    HRAG_CHECK(h->world == 1, who + ": a node-range-sharded handle (world > 1) keeps no KNN index");
    HRAG_CHECK(rows >= 0 && rows < ((int64_t)1 << 31) - 1, who + ": rows out of range");
    HRAG_CHECK(dim > 0 && dim % 8 == 0, who + ": dim must be a positive multiple of 8 (the tensor-core layout)");
    HRAG_CHECK(rows == 0 || emb, who + ": null embeddings");
    HRAG_CHECK(kmax >= 1 && kmax <= kCandidateCap, who + ": kmax must be in [1, 512]");
    HRAG_CHECK(std::isfinite(min_score), who + ": min_score must be finite");
    KnnIndex& K = h->knn;
    if (kept_from) {
        HRAG_CHECK(n_kept >= 0 && n_kept <= rows, who + ": n_kept must be in [0, rows]");
        const int64_t lim = K.held ? K.rows : rows;   // kept_from[i] >= i: at most rows - 1 without an index
        for (int64_t i = 0; i < n_kept; ++i)
            HRAG_CHECK(kept_from[i] >= 0 && kept_from[i] < lim && (i == 0 || kept_from[i] > kept_from[i - 1]),
                       who + ": kept_from must be strictly increasing and index the rows held");
    }
    int64_t slice_rows = 0;   // > 0: the planes of these rows go to pinned host memory
    HRAG_TRY(host_planes_plan(h->knn_budget, who, "hrag_knn_set_memory", rows, dim, &slice_rows));
    const bool on_host = slice_rows > 0;
    HRAG_CUDA(cudaSetDevice(h->device));
    bool build = !K.held || !kept_from || dim != K.dim || kmax != K.kmax || min_score != K.thr;
    if (build) n_kept = 0;

    auto apply = [&]() -> int {
        cudaStream_t st = h->stream;
        const int64_t old_rows = build ? 0 : K.rows;
        const size_t rb = (size_t)dim * 2;
        const int width = (kmax + 1 + 3) & ~3;
        const size_t lb = (size_t)width * 4;
        if (on_host) HRAG_TRY(place_host(h, old_rows, rows, dim, slice_rows));
        else HRAG_TRY(place_device(h, old_rows, rows, dim));
        HRAG_TRY(grow_keep(h, K.ids, (size_t)old_rows * lb, (size_t)rows * lb));
        HRAG_TRY(grow_keep(h, K.scores, (size_t)old_rows * lb, (size_t)rows * lb));

        // 1. upload + split; kept rows compared with their old planes before their rows are overwritten
        Buf d_kept, d_flag, f32, shi, slo;
        std::vector<int> kept32((size_t)n_kept);
        int64_t first = n_kept;   // the first kept row that moves
        for (int64_t i = 0; i < n_kept; ++i) {
            kept32[i] = (int)kept_from[i];
            if (first == n_kept && kept_from[i] != i) first = i;
        }
        HRAG_TRY(d_kept.ensure((size_t)std::max<int64_t>(n_kept, 1) * 4));
        if (n_kept) HRAG_TRY(h2d(h, d_kept.p, kept32.data(), (size_t)n_kept * 4));
        HRAG_TRY(d_flag.zeros(sizeof(int)));
        const int64_t w16 = (int64_t)(rb / 16);
        if (on_host) {
            HRAG_TRY(fill_host(h, rows, dim, emb, on_device != 0, n_kept, kept_from, d_kept.as<int>(),
                               d_flag.as<int>()));
        } else {
            const int64_t chunk = std::max<int64_t>(1, (int64_t)(kUploadBytes / ((size_t)dim * 4)));
            const int64_t cr = std::max<int64_t>(1, std::min(chunk, rows));
            HRAG_TRY(shi.ensure((size_t)cr * rb));
            HRAG_TRY(slo.ensure((size_t)cr * rb));
            if (!on_device) HRAG_TRY(f32.ensure((size_t)cr * dim * 4));
            for (int64_t r0 = 0; r0 < rows; r0 += chunk) {
                const int64_t n = std::min(chunk, rows - r0);
                const float* src = emb + (size_t)r0 * dim;
                if (!on_device) {
                    HRAG_TRY(h2d(h, f32.p, src, (size_t)n * dim * 4));
                    src = f32.as<float>();
                }
                HRAG_TRY(split_bf16(src, n * dim, shi.p, slo.p, st));
                const int64_t nc = std::max<int64_t>(0, std::min(n, n_kept - r0));
                if (nc) {
                    k_knn_compare<<<blocks_for(nc * w16), kThreads, 0, st>>>(
                        nc, w16, r0, d_kept.as<int>(), shi.as<int4>(), slo.as<int4>(), K.hi.as<int4>(),
                        K.lo.as<int4>(), d_flag.as<int>());
                    count_launch(1);
                    HRAG_CUDA(cudaGetLastError());
                }
                HRAG_CUDA(cudaMemcpyAsync(static_cast<char*>(K.hi.p) + (size_t)r0 * rb, shi.p, (size_t)n * rb,
                                          cudaMemcpyDeviceToDevice, st));
                HRAG_CUDA(cudaMemcpyAsync(static_cast<char*>(K.lo.p) + (size_t)r0 * rb, slo.p, (size_t)n * rb,
                                          cudaMemcpyDeviceToDevice, st));
            }
        }
        int mismatch = 0;
        HRAG_CUDA(cudaMemcpyAsync(&mismatch, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
        HRAG_CUDA(cudaStreamSynchronize(st));
        if (mismatch) build = true;

        const bool unchanged = !build && n_kept == rows && rows == old_rows;
        K.dim = dim;
        K.kmax = kmax;
        K.width = width;
        K.thr = min_score;
        K.held = true;
        if (build) {
            K.rows = rows;
            Scratch s;
            HRAG_TRY(run_queries(h, s, nullptr, 0, rows, 0, rows, false));
            *mode = 0;
            return 0;
        }
        if (unchanged) { *mode = 2; return 0; }

        // 2. relabel + drop deleted keys, then move the kept lists to their new rows
        std::vector<int> refill;
        if (n_kept) {
            Buf map, d_refill, n_refill, staging;
            HRAG_TRY(map.ensure((size_t)std::max<int64_t>(old_rows, 1) * 4));
            HRAG_CUDA(cudaMemsetAsync(map.p, 0xff, (size_t)std::max<int64_t>(old_rows, 1) * 4, st));
            k_knn_map<<<blocks_for(n_kept), kThreads, 0, st>>>(n_kept, d_kept.as<int>(), map.as<int>());
            count_launch(1);
            HRAG_CUDA(cudaGetLastError());
            HRAG_TRY(d_refill.ensure((size_t)n_kept * 4));
            HRAG_TRY(n_refill.zeros(sizeof(int)));
            {
                StageTimer tm(h, ST_TOPK);
                k_knn_relabel<<<blocks_for(n_kept * 32), kThreads, 0, st>>>(n_kept, d_kept.as<int>(), map.as<int>(),
                                                                             K.ids.as<int>(), K.scores.as<float>(),
                                                                             width, kmax, d_refill.as<int>(),
                                                                             n_refill.as<int>());
                count_launch(1);
                HRAG_CUDA(cudaGetLastError());
                HRAG_TRY(compact_rows(h, K.ids.p, lb, n_kept, first, d_kept.as<int>(), staging));
                HRAG_TRY(compact_rows(h, K.scores.p, lb, n_kept, first, d_kept.as<int>(), staging));
            }
            int nr = 0;
            HRAG_CUDA(cudaMemcpyAsync(&nr, n_refill.p, sizeof(int), cudaMemcpyDeviceToHost, st));
            HRAG_CUDA(cudaStreamSynchronize(st));
            refill.resize((size_t)nr);
            if (nr) HRAG_TRY(d2h(h, refill.data(), d_refill.p, (size_t)nr * 4));
            HRAG_CUDA(cudaStreamSynchronize(st));
            std::sort(refill.begin(), refill.end());
        }
        K.rows = rows;
        Scratch s;
        // 3. kept rows x new keys, merged; 4. refilled rows and new rows x all keys, replaced
        HRAG_TRY(run_queries(h, s, nullptr, 0, n_kept, n_kept, rows - n_kept, true));
        HRAG_TRY(run_queries(h, s, &refill, 0, (int64_t)refill.size(), 0, rows, false));
        HRAG_TRY(run_queries(h, s, nullptr, n_kept, rows - n_kept, 0, rows, false));
        *mode = 1;
        return 0;
    };
    if (const int rc = apply()) {
        cudaStreamSynchronize(h->stream);
        K = KnnIndex{};
        return rc;
    }
    return resolve_spans(h);
}

int hrag_knn_index_read(hrag_t* h, int64_t row0, int64_t n, int32_t* ids, float* scores, int32_t* n_valid) {
    HRAG_CHECK(h, "hrag_knn_index_read: null handle");
    const KnnIndex& K = h->knn;
    HRAG_CHECK(row0 >= 0 && n >= 0 && row0 + n <= K.rows, "hrag_knn_index_read: rows out of range of the index");
    HRAG_CHECK(n == 0 || (ids && scores), "hrag_knn_index_read: null argument");
    if (n == 0) return 0;
    HRAG_CUDA(cudaSetDevice(h->device));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    const size_t lb = (size_t)K.width * 4, out = (size_t)K.kmax * 4;
    HRAG_CUDA(cudaMemcpy2D(ids, out, K.ids.as<char>() + (size_t)row0 * lb, lb, out, (size_t)n, cudaMemcpyDeviceToHost));
    HRAG_CUDA(cudaMemcpy2D(scores, out, K.scores.as<char>() + (size_t)row0 * lb, lb, out, (size_t)n,
                           cudaMemcpyDeviceToHost));
    h->stats.d2h_bytes += (int64_t)(2 * out * n);
    if (n_valid)
        for (int64_t r = 0; r < n; ++r) {
            int c = 0;
            while (c < K.kmax && ids[r * K.kmax + c] >= 0) ++c;
            n_valid[r] = c;
        }
    return 0;
}

int hrag_knn_index_info(hrag_t* h, int64_t* rows, int32_t* dim, int32_t* kmax) {
    HRAG_CHECK(h && rows && dim && kmax, "hrag_knn_index_info: null argument");
    *rows = h->knn.rows;
    *dim = h->knn.held ? h->knn.dim : 0;
    *kmax = h->knn.held ? h->knn.kmax : 0;
    return 0;
}

int hrag_knn_set_memory(hrag_t* h, int64_t max_device_bytes) {
    HRAG_CHECK(h, "hrag_knn_set_memory: null handle");
    HRAG_CHECK(max_device_bytes >= 0, "hrag_knn_set_memory: the budget must be >= 0 bytes (0 = no limit)");
    HRAG_CHECK(h->world == 1 || max_device_bytes == 0,
               "hrag_knn_set_memory: a node-range-sharded handle (world > 1) keeps no KNN index");
    h->knn_budget = max_device_bytes;
    return 0;
}

int hrag_knn_planes_info(hrag_t* h, int* on_host, int64_t* slice_rows, int64_t* device_bytes, int64_t* host_bytes) {
    HRAG_CHECK(h && on_host && slice_rows && device_bytes && host_bytes, "hrag_knn_planes_info: null argument");
    const KnnIndex& K = h->knn;
    *on_host = K.host.held() ? 1 : 0;
    *slice_rows = K.host.slice_rows;
    *device_bytes = K.host.held() ? (int64_t)K.host.ring.cap : (int64_t)(K.hi.cap + K.lo.cap);
    *host_bytes = K.host.held() ? 2 * (int64_t)K.host.plane_bytes : 0;
    return 0;
}

int hrag_knn_index_clear(hrag_t* h) {
    HRAG_CHECK(h, "hrag_knn_index_clear: null handle");
    HRAG_CUDA(cudaSetDevice(h->device));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    h->knn = KnnIndex{};
    return 0;
}

}  // extern "C"
