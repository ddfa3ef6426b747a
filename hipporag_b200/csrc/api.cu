// C ABI of libhrag_b200.so (declared in include/hrag_b200.h): handle lifecycle, options, and the stage orchestration
// that stands in for the body of HippoRAG.retrieve()'s per-query loop (reference HippoRAG.py:459-480) -- batched, on
// one H100, all intermediate state in HBM.  The handle and its HBM layout: handle.h.
#include <algorithm>
#include <cmath>
#include <memory>

#include "handle.h"

namespace hrag {

static thread_local std::string g_error;
void set_error(const std::string& msg) { g_error = msg; }

int64_t pad4(int64_t x) { return (x + 3) & ~(int64_t)3; }

// bf16 hi / lo split of Bq queries into q_hi / q_lo, the query operand of the tensor-core kernels
int split_queries(hrag_t* h, const float* dQ, int Bq, cudaStream_t s) {
    const size_t n = (size_t)Bq * h->dim;
    HRAG_TRY(h->q_hi.ensure(n * 2));
    HRAG_TRY(h->q_lo.ensure(n * 2));
    return split_bf16(dQ, (int64_t)n, h->q_hi.p, h->q_lo.p, s);
}

int64_t chunk_b(hrag_t* h) {
    const int64_t P = std::max<int64_t>(h->t.n_passages, 1);
    int64_t c = (int64_t)(4e9 / (4.0 * (double)pad4(P)));
    return std::max<int64_t>(1, std::min<int64_t>(c, kQueryChunk));
}

int fact_norms_update(hrag_t* h, int64_t row0, int64_t n, bool reset) {
    EmbMem& e = h->emb[0];
    if (e.hi.p == nullptr) return 0;
    const bool fresh = e.nmax.p == nullptr;
    HRAG_TRY(e.nmax.ensure(2 * sizeof(float)));
    if (reset || fresh) HRAG_CUDA(cudaMemsetAsync(e.nmax.p, 0, 2 * sizeof(float), h->stream));
    return plane_norm_max(static_cast<const char*>(e.hi.p) + (size_t)row0 * h->dim * 2,
                          static_cast<const char*>(e.lo.p) + (size_t)row0 * h->dim * 2, n, h->dim,
                          e.nmax.as<unsigned int>(), h->stream);
}

// The stage-A screen replaces the split K2 over all facts on one GPU with resident planes (DESIGN.md section 4, K2).
// Below 65,536 facts the split K2 takes a fraction of a millisecond per chunk and the screen's dozen extra launches
// cost more than they save (MuSiQue-1k, 10,734 facts: 0.9 against 0.7 ms per 64-query step).
constexpr int64_t kScreenMinFacts = 65536;
bool screened(const hrag_t* h) {
    return h->world == 1 && h->sim_mode == HRAG_SIM_BF16X3 && !h->debug_exact_stage_a && h->emb[0].hi.p != nullptr &&
           h->emb[0].nmax.p != nullptr && h->emb[0].rows >= kScreenMinFacts;
}

// Stage A of Bq <= 1024 queries (split into q_hi / q_lo) by the screen: hi.hi over all facts with the screen epilogue,
// the candidates of each query (screen_select), their rows staged per 128-query m-tile at column f mod 256, the split
// K2 over the staged tiles and the exact selection over them.  Every score the selection reads is the one the split K2
// gives over all facts, bit for bit (same query row, same column, same k sequence), and the candidates hold the k best
// and the minimum, so the outputs are those of the exact path.  When the screen cannot prove that (a non-finite bound,
// a cap overflowed, or a rescored score outside the bound) it raises scr.flag, and the gated exact path below reruns
// the chunk and counts it.  With the lo plane in host memory the staged lo rows come from the mapped plane, and the
// flag is the caller's (chunk_flag): fact_stream.cu reruns the flagged chunks with the lo plane streamed.
int screened_stage_a(hrag_t* h, int Bq, const float* d_qf, int k, int* d_top_idx, float* d_top_score, int* d_nvalid,
                     cudaStream_t s, int n_ctas, int* chunk_flag, unsigned long long* lo_bytes) {
    const int64_t F = h->emb[0].rows;
    const int nt = sim_tc_n_tiles(F), mtiles = (int)ceil_div(Bq, 128), ST = kScreenStageTiles;
    auto& c = h->scr;
    HRAG_TRY(h->part_mm.ensure((size_t)Bq * nt * sizeof(float2)));
    HRAG_TRY(h->part_keys.ensure((size_t)Bq * nt * 8 * sizeof(uint64_t)));
    HRAG_TRY(h->part_bound.ensure((size_t)Bq * sizeof(uint64_t)));
    HRAG_TRY(c.err.ensure((size_t)Bq * sizeof(float)));
    HRAG_TRY(c.part_low.ensure((size_t)Bq * nt * sizeof(uint4)));
    HRAG_TRY(c.cand_ids.ensure((size_t)Bq * kScreenCandidates * sizeof(int)));
    HRAG_TRY(c.cand_s1.ensure((size_t)Bq * kScreenCandidates * sizeof(float)));
    HRAG_TRY(c.cand_n.ensure((size_t)Bq * sizeof(int)));
    HRAG_TRY(c.sat.ensure((size_t)Bq * kScreenSatTiles * sizeof(int)));
    HRAG_TRY(c.sat_n.ensure((size_t)Bq * sizeof(int)));
    HRAG_TRY(c.pos_of.ensure((size_t)mtiles * F * sizeof(int)));
    HRAG_TRY(c.slot_ids.ensure((size_t)mtiles * ST * 256 * sizeof(int)));
    HRAG_TRY(c.res_count.ensure((size_t)mtiles * 256 * sizeof(int)));
    HRAG_TRY(c.stage_count.ensure((size_t)mtiles * sizeof(int)));
    HRAG_TRY(c.st_hi.ensure((size_t)mtiles * ST * 256 * h->dim * 2));
    HRAG_TRY(c.st_lo.ensure((size_t)mtiles * ST * 256 * h->dim * 2));
    HRAG_TRY(c.st_S.ensure((size_t)Bq * ST * 256 * sizeof(float)));
    HRAG_TRY(c.flag.ensure(sizeof(int)));
    if (c.fallbacks.p == nullptr) HRAG_TRY(c.fallbacks.zeros(sizeof(unsigned long long)));
    void* lo_mapped = nullptr;   // lo on the host: its device address, which the gather reads over PCIe
    const PlaneSet P = emb_planes(h, 0);
    const bool lo_host = P.on_host[1];
    HRAG_CHECK(lo_host == (chunk_flag != nullptr) && lo_host == (lo_bytes != nullptr),
               "internal: screened_stage_a: a chunk flag and a byte count go with the lo plane in host memory");
    if (lo_host) HRAG_CUDA(cudaHostGetDevicePointer(&lo_mapped, P.plane[1], 0));
    int* flag = lo_host ? chunk_flag : c.flag.as<int>();
    const EmbMem& e = h->emb[0];
    const int dim = h->dim;
    {
        StageTimer tm(h, ST_SIM_FACT, s);
        HRAG_TRY(split_queries(h, d_qf, Bq, s));
        HRAG_TRY(query_err(h->q_hi.p, h->q_lo.p, Bq, dim, e.nmax.as<unsigned int>(), c.err.as<float>(), s));
        HRAG_TRY(sim_tc_screen(h->q_hi.p, Bq, e.hi.p, F, dim, c.err.as<float>(), h->part_keys.as<uint64_t>(),
                               c.part_low.as<uint4>(), h->part_bound.as<uint64_t>(), n_ctas, s));
    }
    {
        StageTimer tm(h, ST_SEL_FACT, s);
        HRAG_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), s));
        HRAG_CUDA(cudaMemsetAsync(c.pos_of.p, 0xff, (size_t)mtiles * F * sizeof(int), s));
        HRAG_CUDA(cudaMemsetAsync(c.slot_ids.p, 0xff, (size_t)mtiles * ST * 256 * sizeof(int), s));
        HRAG_CUDA(cudaMemsetAsync(c.res_count.p, 0, (size_t)mtiles * 256 * sizeof(int), s));
        HRAG_CUDA(cudaMemsetAsync(c.stage_count.p, 0, (size_t)mtiles * sizeof(int), s));
        HRAG_TRY(screen_select(h->part_keys.as<uint64_t>(), c.part_low.as<uint4>(), Bq, nt, c.err.as<float>(),
                               c.cand_ids.as<int>(), c.cand_s1.as<float>(), c.cand_n.as<int>(), c.sat.as<int>(),
                               c.sat_n.as<int>(), flag, s));
        HRAG_TRY(screen_stage(c.cand_ids.as<int>(), c.cand_n.as<int>(), c.sat.as<int>(), c.sat_n.as<int>(), Bq, F, ST,
                              c.pos_of.as<int>(), c.slot_ids.as<int>(), c.res_count.as<int>(), c.stage_count.as<int>(),
                              flag, s));
        if (lo_host)
            HRAG_TRY(screen_gather_mapped(c.slot_ids.as<int>(), c.stage_count.as<int>(), mtiles, ST, e.hi.p,
                                          lo_mapped, dim, c.st_hi.p, c.st_lo.p, lo_bytes, s));
        else
            HRAG_TRY(screen_gather(c.slot_ids.as<int>(), c.stage_count.as<int>(), mtiles, ST, e.hi.p, e.lo.p, dim,
                                   c.st_hi.p, c.st_lo.p, s));
    }
    {
        StageTimer tm(h, ST_SIM_FACT, s);
        HRAG_TRY(sim_tc_staged(h->q_hi.p, h->q_lo.p, Bq, c.st_hi.p, c.st_lo.p, ST, c.stage_count.as<int>(), dim,
                               c.st_S.as<float>(), n_ctas, s));
    }
    {
        StageTimer tm(h, ST_SEL_FACT, s);
        HRAG_TRY(screen_finish(c.st_S.as<float>(), Bq, ST, c.slot_ids.as<int>(), c.stage_count.as<int>(),
                               c.pos_of.as<int>(), F, c.cand_ids.as<int>(), c.cand_s1.as<float>(), c.cand_n.as<int>(),
                               c.err.as<float>(), k, h->mm_fact.as<float2>(), d_top_idx, d_top_score, d_nvalid, flag, s));
    }
    if (lo_host) return 0;
    // the exact path, run only when the flag is up (kernels that find it down return at once)
    {
        StageTimer tm(h, ST_SIM_FACT, s);
        HRAG_TRY(sim_tc(h->q_hi.p, h->q_lo.p, Bq, e.hi.p, e.lo.p, F, dim, 4, nullptr, 0, h->part_mm.as<float2>(),
                        h->part_keys.as<uint64_t>(), h->part_bound.as<uint64_t>(), n_ctas, s, flag));
    }
    StageTimer tm(h, ST_SEL_FACT, s);
    return merge_minmax_topk_gated(h->part_mm.as<float2>(), h->part_keys.as<uint64_t>(), Bq, nt, F, k,
                                   h->mm_fact.as<float2>(), d_top_idx, d_top_score, d_nvalid, flag,
                                   c.fallbacks.as<unsigned long long>(), s);
}

// Stage B's similarity part on stream s, Bq <= chunk_b: passage scores into S_buf [Bq, pad4(P)] and their per-row
// (min, max) into mm_buf.
int dev_stage_b_sim(hrag_t* h, int Bq, const float* d_qp, hrag::Buf& S_buf, hrag::Buf& mm_buf, cudaStream_t s,
                    int n_ctas) {
    const int P = h->t.n_passages;
    HRAG_CHECK(P > 0, "stage B: no passages loaded");
    const int64_t ld = pad4(P);
    HRAG_TRY(S_buf.ensure((size_t)Bq * ld * sizeof(float)));
    HRAG_TRY(mm_buf.ensure((size_t)Bq * sizeof(float2)));
    StageTimer tm(h, ST_SIM_PASS, s);
    HRAG_TRY(sim_scores(h, 1, d_qp, Bq, S_buf.as<float>(), ld, s, n_ctas));
    HRAG_TRY(row_minmax_topk(S_buf.as<float>(), Bq, P, ld, 0, mm_buf.as<float2>(), nullptr, nullptr, nullptr, s));
    h->last_pass_S = &S_buf;
    h->last_pass_rows = Bq;
    return 0;
}

// Stage B's solve part on `stream`: seeds -> PPR -> top-k over the scores S / mm_pass of dev_stage_b_sim (the PPR
// scores are gathered into S in place).
int dev_stage_b_solve(hrag_t* h, int Bq, float* S, float2* mm_pass, const int* d_kept_idx, const float* d_kept_score,
                      int k_facts, const uint8_t* d_dpr, float damping, float pnw, int link_top_k, int topk,
                      int iters_arg, float tol_arg, int* d_out_ids, float* d_out_scores) {
    const int P = h->t.n_passages;
    const int64_t ld = pad4(P);
    HRAG_TRY(h->mode.ensure((size_t)Bq * sizeof(int)));
    const SweepPlan plan = plan_sweeps(h, damping, iters_arg, tol_arg, h->ppr_precision == HRAG_PPR_MIXED && Bq > 16);
    const bool mixed = plan.mixed;
    const int Bp = mixed ? 32 : round_batch(std::min(h->ppr_batch, Bq));
    if (mixed) HRAG_TRY(ensure_stage_b_mixed(h, Bq, k_facts));
    else HRAG_TRY(ensure_state(h, Bp));
    HRAG_TRY(h->seed_vid.ensure((size_t)Bq * kSeedSlots * sizeof(int)));     // [Bq, kSeedSlots] seed slots
    HRAG_TRY(h->seed_w.ensure((size_t)Bq * kSeedSlots * sizeof(double)));
    {
        StageTimer tm(h, ST_SEED);
        HRAG_TRY(seed_entities(h->t, Bq, d_kept_idx, d_kept_score, k_facts, d_dpr, link_top_k, h->seed_vid.as<int>(),
                               h->seed_w.as<double>(), h->mode.as<int>(), h->stream));
    }
    if (k_facts == 0) {   // retrieve_dpr (HippoRAG.py:665-732): every query is a DPR query, no PPR at all
        StageTimer tm(h, ST_TOPK);
        HRAG_TRY(minmax_apply(S, Bq, P, ld, mm_pass, h->stream));
    }
    if (mixed && k_facts > 0) HRAG_TRY(stage_b_mixed(h, plan, Bq, S, ld, mm_pass, pnw, damping));
    for (int q0 = 0; q0 < Bq && k_facts > 0 && !mixed; q0 += Bp) {
        const int nb = std::min(Bp, Bq - q0);
        {
            StageTimer tm(h, ST_SEED);
            HRAG_CUDA(cudaMemsetAsync(h->V.p, 0, (size_t)h->g.n_global * Bp * sizeof(float), h->stream));
            HRAG_TRY(seed_passages(h->t, Bp, nb, S, ld, q0, mm_pass, pnw, h->V.as<float>(), h->stream));
            HRAG_TRY(seed_scatter(Bp, nb, q0, h->seed_vid.as<int>(), h->seed_w.as<double>(), h->V.as<float>(),
                                  h->stream));
        }
        float* Z = nullptr;
        HRAG_TRY(dev_ppr(h, Bp, plan.iters, damping, &Z));
        StageTimer tm(h, ST_TOPK);
        HRAG_TRY(gather_passage_scores(h->t, Bp, nb, q0, Z, h->sums.as<double>(), h->mode.as<int>(),
                                       mm_pass, S, ld, h->stream));
    }
    {
        StageTimer tm(h, ST_TOPK);
        HRAG_TRY(row_topk(S, Bq, P, ld, topk, d_out_ids, d_out_scores, h->stream));
    }
    return 0;
}

// Stage B at PRPACK accuracy on `stream`, Bq <= chunk_b: the same seeds, the reset in the reference's dtypes (float64
// node_weights from fp32 scores), float64 PPR by iterative refinement per sub-batch of <= 16 queries, the passage
// scores gathered in float64 into io64 [nb, pad4(P)] and their exact top-k.  S / mm_pass (dev_stage_b_sim) are only
// read.  *worst accumulates the residual and bound of the sub-batches solved; status 4 when one misses `target`.
int dev_stage_b_solve_f64(hrag_t* h, int Bq, const float* S, const float2* mm_pass, const int* d_kept_idx,
                          const float* d_kept_score, int k_facts, const uint8_t* d_dpr, double damping, float pnw,
                          int link_top_k, int topk, double target, int* d_out_ids, double* d_out_scores,
                          F64Refined* worst) {
    const int P = h->t.n_passages;
    const int N = h->g.n_global;
    const int64_t ld = pad4(P);
    const int Bp = round_batch(std::min(16, Bq));
    HRAG_TRY(h->mode.ensure((size_t)Bq * sizeof(int)));
    HRAG_TRY(ensure_state_f64(h, Bp, ld));
    HRAG_TRY(h->seed_vid.ensure((size_t)Bq * kSeedSlots * sizeof(int)));
    HRAG_TRY(h->seed_w.ensure((size_t)Bq * kSeedSlots * sizeof(double)));
    {
        StageTimer tm(h, ST_SEED);
        HRAG_TRY(seed_entities(h->t, Bq, d_kept_idx, d_kept_score, k_facts, d_dpr, link_top_k, h->seed_vid.as<int>(),
                               h->seed_w.as<double>(), h->mode.as<int>(), h->stream));
    }
    double* io = h->io64.as<double>();
    const double* xsum = h->sums64.as<double>() + 32;
    for (int q0 = 0; q0 < Bq; q0 += Bp) {
        const int nb = std::min(Bp, Bq - q0);
        if (k_facts > 0) {   // k_facts == 0 is retrieve_dpr (HippoRAG.py:665-732): every row is a DPR row, no PPR
            {
                StageTimer tm(h, ST_SEED);
                HRAG_TRY(seed_reset_f64(h->t, nb, N, q0, S, ld, mm_pass, pnw, h->seed_vid.as<int>(),
                                        h->seed_w.as<double>(), io, h->stream));
                HRAG_TRY(reset_f64(h, Bp, nb));
            }
            F64Refined r;
            HRAG_TRY(refine_f64(h, Bp, nb, damping, target, &r));
            if (r.active) return f64_missed(h, "hrag_stage_b_f64", r, target, worst->resid, worst->bound);
            worst->resid = std::max(worst->resid, r.resid);
            worst->bound = std::max(worst->bound, r.bound);
        }
        StageTimer tm(h, ST_TOPK);
        HRAG_TRY(gather_passage_scores_f64(h->t, Bp, nb, q0, h->X64.as<double>(), xsum, h->mode.as<int>(), mm_pass,
                                           S, ld, io, ld, h->stream));
        HRAG_TRY(row_topk(io, nb, P, ld, topk, d_out_ids + (size_t)q0 * topk, d_out_scores + (size_t)q0 * topk,
                          h->stream));
    }
    return 0;
}

// Persistent CTAs of the similarity GEMMs of chunk c + 1 while they share the GPU with chunk c's PPR sweeps in
// hrag_retrieve_resident: enough SMs that the GEMMs finish within the sweeps, the rest stay with the sweeps (which
// are bound by DRAM latency, not by SMs).  Work per chunk of Bq queries: GEMM 2 n_seg Bq (F + P) dim FLOP, sweeps
// (non-zeros x 32-column sweeps per sub-batch x sub-batches).  Rates measured at C3 inside the overlapped step, with
// paired sweeps and the bound-gated K2 epilogue, on an H100 SXM (132 SMs, 700 W) at G = 40: a paired sweep 0.381 ms
// per 32 columns (38.0 G non-zeros/s); K2 2.49 TFLOP/s per SM, 0.73 of its rate alone (3.43), as its TMA operand
// loads queue behind the sweeps' gathers.  The stage-A screen (one hi.hi product over the facts; its rescore counted
// as the split product over at most kScreenStageTiles staged tiles) reads twice the operand bytes per FLOP and
// suffers more next to the sweeps: 0.76 TFLOP/s per SM in the C3 step at G = 37, where the sweeps took 0.345 ms per 32
// columns (42 G non-zeros/s).  Its rate here is 0.66, 13 % below that: a G below the optimum costs far more than one
// above it (C3 scan: G = 28 +121 ms per step, G = 44 +5 ms).  DESIGN.md section 4 K2 has the scans of G.
int overlap_ctas(const hrag_t* h, int Bq, const SweepPlan& plan) {
    constexpr double kGemmFlopPerSmMs = 2.49e9, kScreenFlopPerSmMs = 0.66e9;
    const bool up_front = emb_planes(h, 0).streams();   // fact planes in host memory: stage A ran up front
    const bool screen = !up_front && screened(h);
    const double kSweepNnzPerMs = screen ? 4.20e7 : 3.80e7;
    const int n_seg = h->sim_mode == HRAG_SIM_BF16X3 ? 4 : 1;
    const int64_t fact_rows = up_front ? 0 : h->emb[0].rows;
    const double split_cols = (screen ? (double)kScreenStageTiles * 256 : (double)fact_rows) + (double)h->emb[1].rows;
    const double t_gemm = 2.0 * n_seg * Bq * split_cols * h->dim / kGemmFlopPerSmMs +
                          (screen ? 2.0 * Bq * (double)fact_rows * h->dim / kScreenFlopPerSmMs : 0.0);
    const int64_t sweeps = plan.mixed ? (int64_t)(plan.m1 + 1 + plan.m2) * ceil_div(Bq, 32)
                                      : (int64_t)plan.iters * ceil_div(Bq, round_batch(std::min(h->ppr_batch, Bq)));
    const double t_sweep = (double)sweeps * (double)h->g.nnz / kSweepNnzPerMs;
    const int g = (int)std::ceil(t_gemm / std::max(t_sweep, 1e-9));
    return std::min(std::max(g, 1), h->num_sms / 2);
}

// tables, graph and embeddings must describe the same index (a passage matrix with more rows than passage_vid
// would make the similarity kernel write past the score buffer)
static int check_loaded(hrag_t* h, const char* who, bool need_facts) {
    HRAG_CHECK(h->dim > 0 && h->g.n_global > 0 && h->t.passage_vid, std::string(who) + ": graph/tables/embeddings not loaded");
    HRAG_CHECK(h->emb[1].rows == h->t.n_passages,
               std::string(who) + ": passage embeddings have " + std::to_string(h->emb[1].rows) + " rows but passage_vid has " +
                   std::to_string(h->t.n_passages));
    HRAG_CHECK(!need_facts || h->n_facts_global == 0 || h->n_facts_global == h->t.n_facts,
               std::string(who) + ": fact embeddings have " + std::to_string(h->n_facts_global) + " rows but the fact tables have " +
                   std::to_string(h->t.n_facts));
    return 0;
}

// The host-buffer form of stage B: uploads the kept facts and flags, runs each chunk of chunk_b queries through the
// passage similarity (into S_pass / mm_pass) and solve(q0, nb, that chunk's kept facts, flags), which writes its ids
// and score_size-byte scores into d_out_ids / d_out_scores at row q0, and copies them back.
template <class Solve>
static int stage_b_host(hrag_t* h, const char* who, int B, const float* q_pass, const int32_t* kept_fact_idx,
                        const float* kept_fact_score, int k_facts, const uint8_t* dpr_only, int topk, size_t score_size,
                        int32_t* out_ids, void* out_scores, Solve solve) {
    HRAG_TRY(check_loaded(h, who, k_facts > 0));
    HRAG_CUDA(cudaSetDevice(h->device));
    const int64_t chunk = chunk_b(h);
    const int kf = std::max(k_facts, 1);
    HRAG_TRY(h->d_q2.ensure((size_t)std::min<int64_t>(chunk, std::max(B, 1)) * h->dim * sizeof(float)));
    HRAG_TRY(h->d_kept_idx.ensure((size_t)std::max(B, 1) * kf * sizeof(int)));
    HRAG_TRY(h->d_kept_score.ensure((size_t)std::max(B, 1) * kf * sizeof(float)));
    HRAG_TRY(h->d_dpr.ensure((size_t)std::max(B, 1)));
    HRAG_TRY(h->d_out_ids.ensure((size_t)std::max(B, 1) * topk * sizeof(int)));
    HRAG_TRY(h->d_out_scores.ensure((size_t)std::max(B, 1) * topk * score_size));
    if (B == 0) return resolve_spans(h);
    if (k_facts > 0) {
        HRAG_TRY(h2d(h, h->d_kept_idx.p, kept_fact_idx, (size_t)B * k_facts * sizeof(int)));
        HRAG_TRY(h2d(h, h->d_kept_score.p, kept_fact_score, (size_t)B * k_facts * sizeof(float)));
    }
    if (dpr_only) HRAG_TRY(h2d(h, h->d_dpr.p, dpr_only, (size_t)B));
    for (int64_t q0 = 0; q0 < B; q0 += chunk) {
        const int nb = (int)std::min<int64_t>(chunk, B - q0);
        HRAG_TRY(h2d(h, h->d_q2.p, q_pass + (size_t)q0 * h->dim, (size_t)nb * h->dim * sizeof(float)));
        HRAG_TRY(dev_stage_b_sim(h, nb, h->d_q2.as<float>(), h->S_pass, h->mm_pass, h->stream, h->num_sms));
        HRAG_TRY(solve(q0, nb, h->d_kept_idx.as<int>() + q0 * k_facts, h->d_kept_score.as<float>() + q0 * k_facts,
                       dpr_only ? h->d_dpr.as<uint8_t>() + q0 : nullptr));
    }
    HRAG_TRY(d2h(h, out_ids, h->d_out_ids.p, (size_t)B * topk * sizeof(int)));
    HRAG_TRY(d2h(h, out_scores, h->d_out_scores.p, (size_t)B * topk * score_size));
    return resolve_spans(h);
}

}  // namespace hrag

using namespace hrag;

// =================================================================================== C ABI
extern "C" {

const char* hrag_last_error(void) { return g_error.c_str(); }
const char* hrag_version(void) { return "hrag_b200 0.1 (sm_90a)"; }

int hrag_create(const int* device_ids, int n_devices, int shard_mode, hrag_t** out) {
    HRAG_CHECK(out != nullptr, "hrag_create: out is null");
    HRAG_CHECK(n_devices == 1 && device_ids != nullptr,
               "hrag_create: one handle drives one GPU (n_devices must be 1); use one process per GPU");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        set_error("hrag_create: no CUDA device visible -- this library has no CPU fallback");
        return 1;
    }
    HRAG_CHECK(device_ids[0] >= 0 && device_ids[0] < count, "hrag_create: bad device id");
    HRAG_CUDA(cudaSetDevice(device_ids[0]));
    cudaDeviceProp prop;
    HRAG_CUDA(cudaGetDeviceProperties(&prop, device_ids[0]));
    HRAG_CHECK(prop.major == 9 && prop.minor == 0, "hrag_create: this library is built for sm_90a (H100) only");
    std::unique_ptr<hrag_t, void (*)(hrag_t*)> h(new hrag_handle(), hrag_destroy);   // torn down if a step fails
    h->device = device_ids[0];
    h->shard_mode = shard_mode;
    h->num_sms = prop.multiProcessorCount;
    HRAG_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    HRAG_CUDA(cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking));
    // highest priority: the similarity GEMMs' persistent CTAs take their SMs as soon as a sweep grid drains, instead of
    // queueing behind the next sweep's grid
    int prio_least = 0, prio_greatest = 0;
    HRAG_CUDA(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
    HRAG_CUDA(cudaStreamCreateWithPriority(&h->stream_sim, cudaStreamNonBlocking, prio_greatest));
    for (int i = 0; i < 2; ++i) {
        HRAG_CUDA(cudaEventCreateWithFlags(&h->ev_ready[i], cudaEventDisableTiming));
        HRAG_CUDA(cudaEventCreateWithFlags(&h->ev_released[i], cudaEventDisableTiming));
        HRAG_CUDA(cudaEventCreateWithFlags(&h->ev_sim_ready[i], cudaEventDisableTiming));
        HRAG_CUDA(cudaEventCreateWithFlags(&h->ev_sim_consumed[i], cudaEventDisableTiming));
    }
    HRAG_CUDA(cudaEventCreateWithFlags(&h->ev_inputs, cudaEventDisableTiming));
    HRAG_CUDA(cudaEventCreateWithFlags(&h->ev_sim_start, cudaEventDisableTiming));
    *out = h.release();
    return 0;
}

void hrag_destroy(hrag_t* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    if (h->stream_sim) cudaStreamSynchronize(h->stream_sim);
    if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
    drop_captured_solves(h);
    index_share_destroy(h);
    for (auto e : h->pool) cudaEventDestroy(e);
    for (void* p : h->peer_slab) if (p) cudaIpcCloseMemHandle(p);
    for (cudaEvent_t e : {h->ev_ready[0], h->ev_ready[1], h->ev_released[0], h->ev_released[1], h->ev_inputs,
                          h->ev_sim_ready[0], h->ev_sim_ready[1], h->ev_sim_consumed[0], h->ev_sim_consumed[1],
                          h->ev_sim_start})
        if (e) cudaEventDestroy(e);
    for (cudaStream_t s : {h->stream_sim, h->stream2, h->stream}) if (s) cudaStreamDestroy(s);
    delete h;   // the buffers free themselves
}

int hrag_set_options(hrag_t* h, int ppr_method, int ppr_iters, int ppr_batch, int sim_mode) {
    HRAG_CHECK(h, "hrag_set_options: null handle");
    if (ppr_method >= 0) {
        HRAG_CHECK(ppr_method == HRAG_PPR_POWER || ppr_method == HRAG_PPR_CHEBYSHEV, "bad ppr_method");
        h->ppr_method = ppr_method;
    }
    if (ppr_iters > 0) h->ppr_iters = ppr_iters;
    if (ppr_batch > 0) {
        HRAG_CHECK(ppr_batch <= 64, "ppr_batch must be <= 64");
        h->ppr_batch = ppr_batch;
    }
    if (sim_mode >= 0) {
        HRAG_CHECK(sim_mode == HRAG_SIM_FP32 || sim_mode == HRAG_SIM_BF16X3 || sim_mode == HRAG_SIM_BF16,
                   "bad sim_mode");
        h->sim_mode = sim_mode;
    }
    return 0;
}

int hrag_set_ppr_precision(hrag_t* h, int precision, int sweeps1, int sweeps2) {
    HRAG_CHECK(h, "hrag_set_ppr_precision: null handle");
    if (precision >= 0) {
        HRAG_CHECK(precision == HRAG_PPR_FP32 || precision == HRAG_PPR_MIXED, "bad ppr precision");
        h->ppr_precision = precision;
    }
    if (sweeps1 > 0) h->mixed_m1 = sweeps1;
    if (sweeps2 > 0) h->mixed_m2 = sweeps2;
    return 0;
}

int hrag_stage_a(hrag_t* h, int32_t B, const float* q_fact, int32_t k, int32_t* top_idx, float* top_score,
                 int32_t* n_valid) {
    HRAG_CHECK(h && q_fact && top_idx && top_score && n_valid, "hrag_stage_a: null argument");
    HRAG_CHECK(B >= 0 && k >= 1 && k <= kMaxKeptFacts, "hrag_stage_a: k (linking_top_k) must be in [1, 32]");
    HRAG_CHECK(h->dim > 0, "hrag_stage_a: embeddings not loaded");
    HRAG_CUDA(cudaSetDevice(h->device));
    HRAG_TRY(h->d_top_idx.ensure((size_t)std::max(B, 1) * k * sizeof(int)));
    HRAG_TRY(h->d_top_score.ensure((size_t)std::max(B, 1) * k * sizeof(float)));
    HRAG_TRY(h->d_nvalid.ensure((size_t)std::max(B, 1) * sizeof(int)));
    HRAG_TRY(fact_stage_a(h, B, q_fact, false, k, h->d_top_idx.as<int>(), h->d_top_score.as<float>(),
                          h->d_nvalid.as<int>(), h->stream, h->debug_sim_ctas > 0 ? h->debug_sim_ctas : h->num_sms));
    if (B > 0) {
        HRAG_TRY(d2h(h, top_idx, h->d_top_idx.p, (size_t)B * k * sizeof(int)));
        HRAG_TRY(d2h(h, top_score, h->d_top_score.p, (size_t)B * k * sizeof(float)));
        HRAG_TRY(d2h(h, n_valid, h->d_nvalid.p, (size_t)B * sizeof(int)));
    }
    return resolve_spans(h);
}

int hrag_stage_b(hrag_t* h, int32_t B, const float* q_pass, const int32_t* kept_fact_idx,
                 const float* kept_fact_score, int32_t k_facts, const uint8_t* dpr_only, float damping,
                 float passage_node_weight, int32_t link_top_k, int32_t topk, int32_t iters, float tol,
                 int32_t* out_ids, float* out_scores) {
    HRAG_CHECK(h && q_pass && out_ids && out_scores, "hrag_stage_b: null argument");
    HRAG_CHECK(k_facts == 0 || (kept_fact_idx && kept_fact_score), "hrag_stage_b: kept facts missing");
    HRAG_CHECK(B >= 0 && k_facts >= 0 && k_facts <= kMaxKeptFacts && topk >= 1 && topk <= 2048,
               "hrag_stage_b: bad sizes (at most 32 kept facts per query, topk <= 2048)");
    HRAG_CHECK(damping > 0.f && damping < 1.f, "hrag_stage_b: damping must be in (0, 1)");
    HRAG_CHECK(iters >= 0 && tol >= 0.f, "hrag_stage_b: iters and tol must be >= 0 (0 = derive from damping)");
    return stage_b_host(h, "hrag_stage_b", B, q_pass, kept_fact_idx, kept_fact_score, k_facts, dpr_only, topk,
                        sizeof(float), out_ids, out_scores, [&](int64_t q0, int nb, const int* d_kept_idx,
                                                                const float* d_kept_score, const uint8_t* d_dpr) {
        return dev_stage_b_solve(h, nb, h->S_pass.as<float>(), h->mm_pass.as<float2>(), d_kept_idx, d_kept_score,
                                 k_facts, d_dpr, damping, passage_node_weight, link_top_k, topk, iters, tol,
                                 h->d_out_ids.as<int>() + q0 * topk, h->d_out_scores.as<float>() + q0 * topk);
    });
}

int hrag_stage_b_f64(hrag_t* h, int32_t B, const float* q_pass, const int32_t* kept_fact_idx,
                     const float* kept_fact_score, int32_t k_facts, const uint8_t* dpr_only, double damping,
                     float passage_node_weight, int32_t link_top_k, int32_t topk, double tol, int32_t* out_ids,
                     double* out_scores) {
    HRAG_CHECK(h && q_pass && out_ids && out_scores, "hrag_stage_b_f64: null argument");
    HRAG_CHECK(k_facts == 0 || (kept_fact_idx && kept_fact_score), "hrag_stage_b_f64: kept facts missing");
    HRAG_CHECK(B >= 0 && k_facts >= 0 && k_facts <= kMaxKeptFacts && topk >= 1 && topk <= 2048,
               "hrag_stage_b_f64: bad sizes (at most 32 kept facts per query, topk <= 2048)");
    HRAG_TRY(check_f64_call(h, "hrag_stage_b_f64", damping, tol));
    const double target = f64_target(tol);
    F64Refined worst;
    worst.resid = worst.bound = 0.0;
    HRAG_TRY(stage_b_host(h, "hrag_stage_b_f64", B, q_pass, kept_fact_idx, kept_fact_score, k_facts, dpr_only, topk,
                          sizeof(double), out_ids, out_scores, [&](int64_t q0, int nb, const int* d_kept_idx,
                                                                   const float* d_kept_score, const uint8_t* d_dpr) {
        return dev_stage_b_solve_f64(h, nb, h->S_pass.as<float>(), h->mm_pass.as<float2>(), d_kept_idx, d_kept_score,
                                     k_facts, d_dpr, damping, passage_node_weight, link_top_k, topk, target,
                                     h->d_out_ids.as<int>() + q0 * topk, h->d_out_scores.as<double>() + q0 * topk,
                                     &worst);
    }));
    h->last_rho = worst.resid;
    h->last_bound = worst.bound;
    return 0;
}

int hrag_retrieve_resident(hrag_t* h, int32_t B, const float* d_q_fact, const float* d_q_pass, float damping,
                           float passage_node_weight, int32_t link_top_k, int32_t topk, int32_t iters, float tol,
                           int32_t* d_out_ids, float* d_out_scores) {
    HRAG_CHECK(h && d_q_fact && d_q_pass && d_out_ids && d_out_scores, "hrag_retrieve_resident: null argument");
    HRAG_CHECK(B >= 0 && link_top_k >= 1 && link_top_k <= kMaxKeptFacts && topk >= 1 && topk <= 2048,
               "hrag_retrieve_resident: bad sizes (linking_top_k in [1, 32], topk <= 2048)");
    HRAG_CHECK(damping > 0.f && damping < 1.f, "hrag_retrieve_resident: damping must be in (0, 1)");
    HRAG_CHECK(iters >= 0 && tol >= 0.f, "hrag_retrieve_resident: iters and tol must be >= 0");
    HRAG_TRY(check_loaded(h, "hrag_retrieve_resident", true));
    HRAG_CUDA(cudaSetDevice(h->device));
    const int64_t chunk = std::min(chunk_a(h, link_top_k), chunk_b(h));
    const int64_t n_chunks = (B + chunk - 1) / chunk;
    const int k = link_top_k;
    // the per-chunk state the similarity part hands to the solve part: slot 0, and slot 1 when chunks overlap
    const bool overlap = h->world == 1 && n_chunks >= 2 && h->debug_sim_ctas >= 0;
    hrag::Buf* top_idx[2] = {&h->d_top_idx, &h->pipe.top_idx};
    hrag::Buf* top_score[2] = {&h->d_top_score, &h->pipe.top_score};
    hrag::Buf* nvalid[2] = {&h->d_nvalid, &h->pipe.nvalid};
    hrag::Buf* S_pass[2] = {&h->S_pass, &h->pipe.S_pass};
    hrag::Buf* mm_pass[2] = {&h->mm_pass, &h->pipe.mm_pass};
    for (int s = 0; s < (overlap ? 2 : 1); ++s) {
        HRAG_TRY(top_idx[s]->ensure((size_t)chunk * k * sizeof(int)));
        HRAG_TRY(top_score[s]->ensure((size_t)chunk * k * sizeof(float)));
        HRAG_TRY(nvalid[s]->ensure((size_t)chunk * sizeof(int)));
    }
    // stage A per chunk, or, when a fact plane streams, of the whole call first in one walk over the planes (per
    // pass of queries) into fs_top_* [B, k]; the chunks below then skip their stage A
    const bool up_front = emb_planes(h, 0).streams();
    if (up_front) {
        HRAG_TRY(h->fs_top_idx.ensure((size_t)std::max(B, 1) * k * sizeof(int)));
        HRAG_TRY(h->fs_top_score.ensure((size_t)std::max(B, 1) * k * sizeof(float)));
        HRAG_TRY(h->fs_nvalid.ensure((size_t)std::max(B, 1) * sizeof(int)));
        HRAG_TRY(fact_stage_a(h, B, d_q_fact, true, k, h->fs_top_idx.as<int>(), h->fs_top_score.as<float>(),
                              h->fs_nvalid.as<int>(), h->stream,
                              h->debug_sim_ctas > 0 ? h->debug_sim_ctas : h->num_sms));
    }
    // chunk c's similarity part on stream sim_s into slot c % 2 (stage A, then the passage GEMM + min/max)
    auto slot = [&](int64_t c) { return overlap ? (int)(c & 1) : 0; };
    auto similarity = [&](int64_t c, cudaStream_t sim_s, int n_ctas) -> int {
        const int64_t q0 = c * chunk;
        const int nb = (int)std::min<int64_t>(chunk, B - q0), s = slot(c);
        if (!up_front)
            HRAG_TRY(fact_stage_a(h, nb, d_q_fact + (size_t)q0 * h->dim, true, k, top_idx[s]->as<int>(),
                                  top_score[s]->as<float>(), nvalid[s]->as<int>(), sim_s, n_ctas));
        return dev_stage_b_sim(h, nb, d_q_pass + (size_t)q0 * h->dim, *S_pass[s], *mm_pass[s], sim_s, n_ctas);
    };
    // chunk c's solve part on `stream` (identity recognition-memory filter: the candidates are the kept facts)
    auto solve = [&](int64_t c) -> int {
        const int64_t q0 = c * chunk;
        const int nb = (int)std::min<int64_t>(chunk, B - q0), s = slot(c);
        const int* kept_idx = up_front ? h->fs_top_idx.as<int>() + q0 * k : top_idx[s]->as<int>();
        const float* kept_score = up_front ? h->fs_top_score.as<float>() + q0 * k : top_score[s]->as<float>();
        return dev_stage_b_solve(h, nb, S_pass[s]->as<float>(), mm_pass[s]->as<float2>(), kept_idx, kept_score, k,
                                 nullptr, damping, passage_node_weight, link_top_k, topk, iters, tol,
                                 d_out_ids + q0 * topk, d_out_scores + q0 * topk);
    };
    // one chunk, node-range sharding (its all-gathers and spin-waiting sweeps must not share SMs), or hrag_debug_sim_ctas
    if (!overlap) {
        for (int64_t c = 0; c < n_chunks; ++c) {
            HRAG_TRY(similarity(c, h->stream, h->num_sms));
            HRAG_TRY(solve(c));
        }
        return resolve_spans(h);
    }
    // Two streams: stream_sim runs chunk c + 1's similarity GEMMs on n_ctas SMs while `stream` runs chunk c's sweeps on
    // the others.  Every kernel computes what it computes on one stream, so the results are bit-identical.
    const SweepPlan plan = plan_sweeps(h, damping, iters, tol, h->ppr_precision == HRAG_PPR_MIXED && chunk > 16);
    const int n_ctas = h->debug_sim_ctas > 0 ? h->debug_sim_ctas : overlap_ctas(h, (int)chunk, plan);
    HRAG_CUDA(cudaEventRecord(h->ev_sim_start, h->stream));   // the caller's queries, ordered on `stream`
    HRAG_CUDA(cudaStreamWaitEvent(h->stream_sim, h->ev_sim_start, 0));
    HRAG_TRY(similarity(0, h->stream_sim, h->num_sms));        // nothing to overlap with yet: the whole GPU
    HRAG_CUDA(cudaEventRecord(h->ev_sim_ready[0], h->stream_sim));
    for (int64_t c = 0; c < n_chunks; ++c) {
        const int s = (int)(c & 1);
        if (c + 1 < n_chunks) {
            if (c + 1 >= 2) HRAG_CUDA(cudaStreamWaitEvent(h->stream_sim, h->ev_sim_consumed[s ^ 1], 0));   // chunk c - 1 is done
            HRAG_TRY(similarity(c + 1, h->stream_sim, n_ctas));
            HRAG_CUDA(cudaEventRecord(h->ev_sim_ready[s ^ 1], h->stream_sim));
        }
        HRAG_CUDA(cudaStreamWaitEvent(h->stream, h->ev_sim_ready[s], 0));
        HRAG_TRY(solve(c));
        HRAG_CUDA(cudaEventRecord(h->ev_sim_consumed[s], h->stream));
    }
    // (the last chunk's sim_ready was the last work on stream_sim, so `stream` has joined it: the caller's events on
    // `stream`, and resolve_spans' synchronise, cover all of the call)
    return resolve_spans(h);
}
int hrag_similarity(hrag_t* h, int which, int32_t B, const float* q, float* out) {
    HRAG_CHECK(h && q && out && (which == 0 || which == 1), "hrag_similarity: bad arguments");
    HRAG_CHECK(h->dim > 0 && h->emb[which].rows > 0, "hrag_similarity: embeddings not loaded");
    HRAG_CUDA(cudaSetDevice(h->device));
    const int64_t M = h->emb[which].rows, ld = pad4(M);
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>((int64_t)(2e9 / (4.0 * (double)ld)), kQueryChunk));
    hrag::Buf& Sb = which == 0 ? h->S_fact : h->S_pass;
    hrag::Buf& mm = which == 0 ? h->mm_fact : h->mm_pass;
    HRAG_TRY(Sb.ensure((size_t)std::min<int64_t>(chunk, std::max(B, 1)) * ld * sizeof(float)));
    HRAG_TRY(mm.ensure((size_t)std::min<int64_t>(chunk, std::max(B, 1)) * sizeof(float2)));
    HRAG_TRY(h->d_q.ensure((size_t)std::min<int64_t>(chunk, std::max(B, 1)) * h->dim * sizeof(float)));
    for (int64_t q0 = 0; q0 < B; q0 += chunk) {
        const int nb = (int)std::min<int64_t>(chunk, B - q0);
        HRAG_TRY(h2d(h, h->d_q.p, q + (size_t)q0 * h->dim, (size_t)nb * h->dim * sizeof(float)));
        HRAG_TRY(sim_scores(h, which, h->d_q.as<float>(), nb, Sb.as<float>(), ld, h->stream, h->num_sms));
        HRAG_TRY(row_minmax_topk(Sb.as<float>(), nb, M, ld, 0, mm.as<float2>(), nullptr, nullptr, nullptr, h->stream));
        HRAG_TRY(minmax_apply(Sb.as<float>(), nb, M, ld, mm.as<float2>(), h->stream));
        HRAG_CUDA(cudaMemcpy2DAsync(out + (size_t)q0 * M, (size_t)M * sizeof(float), Sb.p, (size_t)ld * sizeof(float),
                                    (size_t)M * sizeof(float), (size_t)nb, cudaMemcpyDeviceToHost, h->stream));
        h->stats.d2h_bytes += (int64_t)nb * M * 4;
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
    }
    (which == 0 ? h->last_fact_rows : h->last_pass_rows) = 0;
    return resolve_spans(h);
}

int hrag_topk_similarity(hrag_t* h, int which, int32_t B, const float* q, int32_t k, int32_t* out_ids,
                         float* out_scores) {
    HRAG_CHECK(h && q && out_ids && out_scores && (which == 0 || which == 1), "hrag_topk_similarity: bad arguments");
    HRAG_CHECK(k >= 1 && k <= 2048 && B >= 0, "hrag_topk_similarity: k must be in [1, 2048]");
    HRAG_CHECK(h->dim > 0 && h->emb[which].rows > 0, "hrag_topk_similarity: embeddings not loaded");
    HRAG_CUDA(cudaSetDevice(h->device));
    const int64_t M = h->emb[which].rows, ld = pad4(M);
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>((int64_t)(4e9 / (4.0 * (double)ld)), kQueryChunk));
    hrag::Buf& Sb = which == 0 ? h->S_fact : h->S_pass;
    const int64_t cb = std::min<int64_t>(chunk, std::max(B, 1));
    HRAG_TRY(Sb.ensure((size_t)cb * ld * sizeof(float)));
    HRAG_TRY(h->d_q.ensure((size_t)cb * h->dim * sizeof(float)));
    HRAG_TRY(h->d_out_ids.ensure((size_t)cb * k * sizeof(int)));
    HRAG_TRY(h->d_out_scores.ensure((size_t)cb * k * sizeof(float)));
    for (int64_t q0 = 0; q0 < B; q0 += chunk) {
        const int nb = (int)std::min<int64_t>(chunk, B - q0);
        HRAG_TRY(h2d(h, h->d_q.p, q + (size_t)q0 * h->dim, (size_t)nb * h->dim * sizeof(float)));
        {
            StageTimer tm(h, which == 0 ? ST_SIM_FACT : ST_SIM_PASS);
            HRAG_TRY(sim_scores(h, which, h->d_q.as<float>(), nb, Sb.as<float>(), ld, h->stream, h->num_sms));
        }
        {
            StageTimer tm(h, ST_TOPK);
            HRAG_TRY(row_topk(Sb.as<float>(), nb, M, ld, k, h->d_out_ids.as<int>(), h->d_out_scores.as<float>(), h->stream));
        }
        HRAG_TRY(d2h(h, out_ids + (size_t)q0 * k, h->d_out_ids.p, (size_t)nb * k * sizeof(int)));
        HRAG_TRY(d2h(h, out_scores + (size_t)q0 * k, h->d_out_scores.p, (size_t)nb * k * sizeof(float)));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
    }
    (which == 0 ? h->last_fact_rows : h->last_pass_rows) = 0;
    return resolve_spans(h);
}

int hrag_knn_threshold(hrag_t* h, int which, int32_t B, const float* q, float min_score, int32_t kmax,
                       int32_t* out_ids, float* out_scores, int32_t* n_found) {
    HRAG_CHECK(h && q && out_ids && out_scores && n_found && (which == 0 || which == 1), "hrag_knn_threshold: bad arguments");
    HRAG_CHECK(kmax >= 1 && kmax <= kCandidateCap && B >= 0, "hrag_knn_threshold: kmax must be in [1, 512]");
    HRAG_CHECK(!emb_planes(h, which).streams(),
               "hrag_knn_threshold: the fact planes are held in host memory (hrag_set_fact_memory); the threshold "
               "search runs on resident planes only");
    HRAG_CHECK(h->dim > 0 && h->emb[which].rows > 0 && h->emb[which].hi.p != nullptr,
               "hrag_knn_threshold: embeddings not loaded (needs the tensor-core layout: dim % 8 == 0)");
    HRAG_CHECK(h->sim_mode != HRAG_SIM_FP32, "hrag_knn_threshold: the threshold epilogue lives in the tensor-core kernel");
    HRAG_CUDA(cudaSetDevice(h->device));
    const int64_t M = h->emb[which].rows;
    const int64_t chunk = kQueryChunk;
    const int64_t cb = std::min<int64_t>(chunk, std::max(B, 1));
    HRAG_TRY(h->d_q.ensure((size_t)cb * h->dim * sizeof(float)));
    HRAG_TRY(h->part_keys.ensure((size_t)cb * kCandidateCap * sizeof(uint64_t)));
    HRAG_TRY(h->d_nvalid.ensure((size_t)cb * 2 * sizeof(int)));
    HRAG_TRY(h->d_out_ids.ensure((size_t)cb * kmax * sizeof(int)));
    HRAG_TRY(h->d_out_scores.ensure((size_t)cb * kmax * sizeof(float)));
    int* d_count = h->d_nvalid.as<int>();
    int* d_found = d_count + cb;
    for (int64_t q0 = 0; q0 < B; q0 += chunk) {
        const int nb = (int)std::min<int64_t>(chunk, B - q0);
        HRAG_TRY(h2d(h, h->d_q.p, q + (size_t)q0 * h->dim, (size_t)nb * h->dim * sizeof(float)));
        HRAG_CUDA(cudaMemsetAsync(d_count, 0, (size_t)nb * sizeof(int), h->stream));
        {
            StageTimer tm(h, which == 0 ? ST_SIM_FACT : ST_SIM_PASS);
            HRAG_TRY(split_queries(h, h->d_q.as<float>(), nb, h->stream));
            HRAG_TRY(sim_tc_threshold(h->q_hi.p, h->q_lo.p, nb, h->emb[which].hi.p, h->emb[which].lo.p, M, h->dim,
                                      h->sim_mode == HRAG_SIM_BF16X3 ? 4 : 1, min_score, h->part_keys.as<uint64_t>(),
                                      d_count, kCandidateCap, h->num_sms, h->stream));
        }
        {
            StageTimer tm(h, ST_TOPK);
            HRAG_TRY(sort_candidates(h->part_keys.as<uint64_t>(), d_count, nb, kCandidateCap, kmax, h->d_out_ids.as<int>(),
                                     h->d_out_scores.as<float>(), d_found, h->stream));
        }
        HRAG_TRY(d2h(h, out_ids + (size_t)q0 * kmax, h->d_out_ids.p, (size_t)nb * kmax * sizeof(int)));
        HRAG_TRY(d2h(h, out_scores + (size_t)q0 * kmax, h->d_out_scores.p, (size_t)nb * kmax * sizeof(float)));
        HRAG_TRY(d2h(h, n_found + q0, d_found, (size_t)nb * sizeof(int)));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
    }
    return resolve_spans(h);
}

void* hrag_stream(hrag_t* h) { return h ? (void*)h->stream : nullptr; }

int hrag_get_stats(hrag_t* h, hrag_stats_t* out) {
    HRAG_CHECK(h && out, "hrag_get_stats: null argument");
    h->stats.kernel_launches = launches_since_reset();
    h->stats.ppr_residual = h->last_rho;
    h->stats.ppr_error_bound = h->last_bound;
    *out = h->stats;
    return 0;
}

int hrag_reset_stats(hrag_t* h) {
    HRAG_CHECK(h, "hrag_reset_stats: null handle");
    h->stats = hrag_stats_t{};
    reset_launch_counter();
    return 0;
}

int hrag_debug_keep_scores(hrag_t* h, int keep) {
    HRAG_CHECK(h, "hrag_debug_keep_scores: null handle");
    h->keep_fact_scores = keep != 0;
    return 0;
}

int hrag_debug_sim_ctas(hrag_t* h, int n) {
    HRAG_CHECK(h, "hrag_debug_sim_ctas: null handle");
    h->debug_sim_ctas = n;
    return 0;
}

int hrag_debug_dense_first_sweep(hrag_t* h, int on) {
    HRAG_CHECK(h, "hrag_debug_dense_first_sweep: null handle");
    h->debug_dense_first_sweep = on != 0;
    return 0;
}

int hrag_debug_exact_stage_a(hrag_t* h, int on) {
    HRAG_CHECK(h, "hrag_debug_exact_stage_a: null handle");
    h->debug_exact_stage_a = on != 0;
    return 0;
}

int hrag_debug_fact_minmax(hrag_t* h, float* host_out, int64_t max_rows, int64_t* n_rows) {
    HRAG_CHECK(h && host_out && n_rows, "hrag_debug_fact_minmax: null argument");
    HRAG_CHECK(h->last_mm_rows <= max_rows, "hrag_debug_fact_minmax: host buffer too small");
    HRAG_CUDA(cudaSetDevice(h->device));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    if (h->last_mm_rows)
        HRAG_CUDA(cudaMemcpy(host_out, h->mm_fact.p, (size_t)h->last_mm_rows * sizeof(float2), cudaMemcpyDeviceToHost));
    *n_rows = h->last_mm_rows;
    return 0;
}

int hrag_debug_copy(hrag_t* h, int which, float* host_out, int64_t max_elems, int64_t* n_written) {
    HRAG_CHECK(h && host_out && n_written, "hrag_debug_copy: null argument");
    HRAG_CUDA(cudaSetDevice(h->device));
    const hrag::Buf& b = which == 0 ? h->S_fact : *h->last_pass_S;
    const int64_t rows = which == 0 ? h->last_fact_rows : h->last_pass_rows;
    const int64_t cols = which == 0 ? h->emb[0].rows : h->t.n_passages;
    const int64_t ld = pad4(cols);
    HRAG_CHECK(rows * cols <= max_elems, "hrag_debug_copy: host buffer too small");
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    if (rows && cols)
        HRAG_CUDA(cudaMemcpy2D(host_out, (size_t)cols * sizeof(float), b.p, (size_t)ld * sizeof(float),
                               (size_t)cols * sizeof(float), (size_t)rows, cudaMemcpyDeviceToHost));
    *n_written = rows * cols;
    return 0;
}

int hrag_debug_graph(hrag_t* h, int plane, void* host_out, int64_t max_bytes, int64_t* n_written) {
    HRAG_CHECK(h && n_written, "hrag_debug_graph: null argument");
    HRAG_CHECK(h->g.cv, "hrag_debug_graph: no graph loaded");
    HRAG_CHECK(plane >= 0 && plane <= 6, "hrag_debug_graph: plane must be in [0, 6]");
    const hrag::PprGraph& g = h->g;
    const void* src[7] = {g.row_ptr, g.cv, g.val_lo, g.row_order, g.long_rows, g.long_seg_ptr, g.segs};
    const int64_t bytes[7] = {4 * (int64_t)(g.n_rows + 1), 8 * g.nnz, g.val_lo ? 4 * g.nnz : 0, 4 * (int64_t)g.n_rows,
                              4 * (int64_t)g.n_long, g.n_long ? 4 * (int64_t)(g.n_long + 1) : 0, 16 * (int64_t)g.n_seg};
    *n_written = bytes[plane];
    if (!host_out) return 0;
    HRAG_CHECK(bytes[plane] <= max_bytes, "hrag_debug_graph: host buffer too small");
    HRAG_CUDA(cudaSetDevice(h->device));
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    if (bytes[plane]) HRAG_CUDA(cudaMemcpy(host_out, src[plane], (size_t)bytes[plane], cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"
