// The PPR solvers: sweep planning, the fp32 solver, the mixed-precision solver (fp16 state, one refinement round, a
// CUDA-graph cache of its solves) and float64 refinement; hrag_ppr, hrag_ppr_f64 and hrag_plan_sweeps.
#include <algorithm>
#include <cmath>

#include "handle.h"

namespace hrag {

int round_batch(int b) {  // PPR batch widths the sweep kernel is instantiated for
    if (b <= 4) return 4;
    if (b <= 8) return 8;
    if (b <= 16) return 16;
    if (b <= 32) return 32;
    return 64;
}

static size_t state_rows(hrag_t* h) {
    return (size_t)(h->world > 1 && h->row_bounds.empty() ? h->chunk_rows * h->world : h->g.n_global);
}

int ensure_state(hrag_t* h, int B) {
    const size_t bytes = state_rows(h) * B * sizeof(float);
    HRAG_TRY(h->V.ensure(bytes));
    HRAG_TRY(h->XA.ensure(bytes));
    HRAG_TRY(h->XC.ensure(bytes));
    HRAG_TRY(h->partials.ensure((size_t)ppr_sweep_partial_rows(h->g, B) * B * sizeof(float)));
    HRAG_TRY(h->sums.ensure(64 * sizeof(double)));
    return 0;
}

// [x0[0] | A | C | R | x0[1]] at base, rows `ld` halves apart
static StateLayout carve_layout(void* base, size_t rows, int ld) {
    StateLayout L;
    L.ld = ld;
    L.bytes = rows * ld * 2;
    void** bufs[5] = {&L.x0[0], &L.A, &L.C, &L.R, &L.x0[1]};
    for (int i = 0; i < 5; ++i) *bufs[i] = static_cast<char*>(base) + (size_t)i * L.bytes;
    return L;
}

unsigned long long* epoch_flags(const hrag_t* h, void* slab) {
    return reinterpret_cast<unsigned long long*>(static_cast<char*>(slab) + 5 * h->single.bytes);
}

static MixedSums* sub_batch_sums(hrag_t* h, int k) { return h->mixed_sums.as<MixedSums>() + k; }

int ensure_state_mixed(hrag_t* h) {
    const size_t rows = state_rows(h);
    if (h->slab.p == nullptr || h->single.bytes != rows * 32 * 2) {
        HRAG_CHECK(!h->p2p, "internal: the state slab cannot change after hrag_p2p_import");
        h->slab.reset();
        HRAG_TRY(h->slab.ensure(5 * rows * 32 * 2 + 256));
        h->single = carve_layout(h->slab.p, rows, 32);
        HRAG_CUDA(cudaMemset(epoch_flags(h, h->slab.p), 0, 256));
        if (!h->p2p_err.p) HRAG_TRY(h->p2p_err.zeros(sizeof(int)));
        if (!h->done_ctr.p) HRAG_TRY(h->done_ctr.zeros(sizeof(unsigned int)));
    }
    HRAG_TRY(h->mixed_part[0].ensure((size_t)std::max(mixed_partial_rows(h->g), 1024) * 32 * sizeof(float)));
    HRAG_TRY(h->mixed_sums.ensure(2 * sizeof(MixedSums)));
    HRAG_TRY(h->rhs[0].scale.ensure(32 * sizeof(float)));    // hrag_ppr's dense solves use set 0's scale and vsum
    HRAG_TRY(h->rhs[0].vsum.ensure(32 * sizeof(double)));
    if (h->rho.p == nullptr) HRAG_TRY(h->rho.zeros(sizeof(MixedRho)));
    return 0;
}

static int ensure_state_pair(hrag_t* h) {
    HRAG_CHECK(h->world == 1, "internal: paired solves run on a single GPU");
    const size_t rows = (size_t)h->g.n_global;
    HRAG_TRY(h->slab_pair.ensure(5 * rows * 64 * 2));
    h->pair = carve_layout(h->slab_pair.p, rows, 64);
    HRAG_TRY(h->mixed_part[1].ensure(h->mixed_part[0].cap));
    return 0;
}

// Compact right-hand-side sets 0 .. n_sets - 1 of stage B, their slot maps built.
static int ensure_compact_rhs(hrag_t* h, int n_sets) {
    const size_t n_slots = (size_t)h->t.n_passages + 32 * kSeedSlots;
    for (int s = 0; s < n_sets; ++s) {
        RhsSet& r = h->rhs[s];
        HRAG_TRY(r.slot_map.ensure((size_t)h->g.n_global * sizeof(int)));
        HRAG_TRY(r.slot_vid.ensure(n_slots * sizeof(int)));
        HRAG_TRY(r.Vc.ensure(n_slots * 32 * sizeof(float)));
        HRAG_TRY(r.R16.ensure(n_slots * 32 * 2));
        HRAG_TRY(r.scale.ensure(32 * sizeof(float)));
        HRAG_TRY(r.vsum.ensure(32 * sizeof(double)));
    }
    HRAG_TRY(h->prep_scratch.ensure((size_t)std::max(compact_rhs_partial_rows(h->t.n_passages), 1024) * 32 * sizeof(float)));
    for (; h->slot_maps_built < n_sets; ++h->slot_maps_built)
        HRAG_TRY(slot_map_build(h->g.n_global, h->t.n_passages, h->t.passage_vid,
                                h->rhs[h->slot_maps_built].slot_map.as<int>(), h->stream));
    return 0;
}

int drop_captured_solves(hrag_t* h) {
    const cudaError_t e = cudaStreamSynchronize(h->stream);   // none of them may still be executing
    for (auto& c : h->solve_graphs) cudaGraphExecDestroy(c.exec);
    h->solve_graphs.clear();
    HRAG_CUDA(e);
    return 0;
}

int invalidate_solves(hrag_t* h) {
    h->slot_maps_built = 0;
    return drop_captured_solves(h);
}

int resolve_spans(hrag_t* h) {
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    if (h->scr.fallbacks.p) {
        // the stage-A screen's fallbacks, counted on the device by work ordered before the end of `stream`
        unsigned long long n = 0;
        HRAG_CUDA(cudaMemcpyAsync(&n, h->scr.fallbacks.p, sizeof(n), cudaMemcpyDeviceToHost, h->stream));
        if (n) HRAG_CUDA(cudaMemsetAsync(h->scr.fallbacks.p, 0, sizeof(n), h->stream));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
        h->stats.stage_a_fallbacks += (int64_t)n;
    }
    if (h->p2p && h->p2p_err.p) {
        int err = 0;
        HRAG_CUDA(cudaMemcpy(&err, h->p2p_err.p, sizeof(int), cudaMemcpyDeviceToHost));
        if (err != 0) HRAG_CUDA(cudaMemset(h->p2p_err.p, 0, sizeof(int)));   // report once; this call's results are invalid
        HRAG_CHECK(err == 0, "node-range sharding: a peer GPU never published its rows (fused exchange timed out); "
                             "the results of this call are invalid");
    }
    if ((h->rho_dirty || h->check_tol > 0.0) && h->rho.p) {
        // every mixed solve of this call (a fresh capture or a replayed graph) raised rho_max, and overflow if an fp16
        // iterate left fp16's range.  Both are cleared here, checked call or not, so the next call is judged by its own
        // solves only.
        MixedRho rho;
        HRAG_CUDA(cudaMemcpy(&rho, h->rho.p, sizeof(rho), cudaMemcpyDeviceToHost));
        HRAG_CUDA(cudaMemset(h->rho.p, 0, sizeof(rho)));
        const double tol = h->check_tol, kappa = h->check_kappa;
        h->check_tol = h->check_kappa = 0.0;
        h->rho_dirty = false;
        if (rho.overflow) {
            set_error("PPR (mixed solver): an fp16 iterate reached 65520 in magnitude and would have been clamped, so "
                      "the result is invalid -- pass more sweeps (iters) or use HRAG_PPR_FP32");
            return 5;
        }
        if (tol > 0.0) {
            // a-posteriori check of the mixed solver: the refinement round contracts rho by kappa (plan_sweeps)
            h->last_rho = rho.rho_max;
            h->last_bound = (float)(rho.rho_max * kappa);
            if (!(rho.rho_max * kappa <= 10.0 * tol)) {
                set_error("PPR (mixed solver): measured relative residual " + std::to_string(rho.rho_max) +
                          " x predicted contraction " + std::to_string(kappa) + " misses tol " + std::to_string(tol) +
                          " -- pass more sweeps (iters) or use HRAG_PPR_FP32");
                return 4;
            }
        }
    }
    double* slots[ST_COUNT] = {&h->stats.ms_sim_fact, &h->stats.ms_select_fact, &h->stats.ms_sim_passage,
                               &h->stats.ms_seed, &h->stats.ms_ppr, &h->stats.ms_topk, &h->stats.ms_comm};
    for (auto& s : h->spans) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, s.a, s.b);
        *slots[s.stage] += ms;
        h->pool.push_back(s.a);
        h->pool.push_back(s.b);
    }
    h->spans.clear();
    h->stats.kernel_launches = launches_since_reset();
    return 0;
}

// Chebyshev semi-iteration on alpha P, whose spectrum lies in [-alpha, alpha]: sweep `it` (1-based) computes
// y = w (alpha P x + rhs) + (1 - w) prev, prev = the input of the sweep before.  Sweep 1 is a plain sweep (w = 1)
// into a, sweep 2 writes c, every later one overwrites prev in place.  Returns w, computed in double.
template <class T>
static float cheb_step(int it, float alpha, double* w, T* a, T* c, T* prev, T** y) {
    if (it == 1) { *y = a; return 1.f; }
    const double rho2 = (double)alpha * (double)alpha;
    *w = it == 2 ? 1.0 / (1.0 - rho2 / 2.0) : 1.0 / (1.0 - rho2 * *w / 4.0);
    *y = it == 2 ? c : prev;
    return (float)*w;
}

// One sweep of the n sub-batches of a solve in layout L (n = 2: one paired walk over the interleaved buffers x, prev,
// y).  in[k] holds sub-batch k's slot_map, rhs_h, v32 and col_scale; a dense rhs_h (slot_map null) is a buffer of L
// like x.  final: the column-sum partials of sub-batch k go to h->mixed_part[k].  x0c: MixedSweepIO::x0c (x or prev
// is then null).
static int mixed_sweep_n(hrag_t* h, const StateLayout& L, int n, int mode, const MixedSweepIO* in, const void* x,
                         const void* prev, void* y, float alpha, float w, float t, bool final, int* n_part,
                         int x0c = 0) {
    MixedSweepIO io[2];
    for (int k = 0; k < n; ++k) {
        io[k] = in[k];
        io[k].x0c = x0c;
        if (!io[k].slot_map) io[k].rhs_h = L.part(io[k].rhs_h, k);
        io[k].xh = L.part(x, k);
        io[k].prevh = L.part(prev, k);
        io[k].yh = L.part(y, k);
        io[k].partials = final ? h->mixed_part[k].as<float>() : nullptr;
    }
    int* overflow = h->rho.p ? &h->rho.as<MixedRho>()->overflow : nullptr;
    // the exchange (sharded, n = 1): fused peer stores when the peers are mapped, an NCCL all-gather otherwise
    HRAG_TRY(mixed_sweep(h->g, mode, io, n, alpha, w, t, n_part, overflow, peers_for(h, io[0].yh), sync_for_sweep(h),
                         h->stream));
    if (!h->p2p) HRAG_TRY(exchange_rows_bytes(h, io[0].yh, 32 * 2));
    return 0;
}

// Column sums of sub-batch k of the last final sweep -> its MixedSums' `which`
static int mixed_sums(hrag_t* h, int n, int n_part, double (MixedSums::*which)[32]) {
    for (int k = 0; k < n; ++k)
        HRAG_TRY(colsum_reduce(h->mixed_part[k].as<float>(), n_part, 32, sub_batch_sums(h, k)->*which, h->stream));
    return 0;
}

// m Chebyshev sweeps of the fp16 solver on (I - aP) x = rhs for n sub-batches in layout L, first iterate x_first (= rhs
// as a dense buffer of L; null: the compact rhs itself, read through its slot map by sweeps 1 and 2); rhs[k] holds
// sub-batch k's rhs_h and its slot_map (null = dense).  Iterates alternate between bufA and bufC; *result = the last
// one, its column sums land in the sub-batches' MixedSums' `which`.
static int mixed_cheb(hrag_t* h, const StateLayout& L, int n, const MixedSweepIO* rhs, void* x_first, void* bufA,
                      void* bufC, int m, float alpha, void** result, double (MixedSums::*which)[32]) {
    HRAG_CHECK(m >= 1, "mixed solver: sweep count must be >= 1");
    double w = 1.0;
    void *x = x_first, *prev = nullptr, *y = nullptr;
    int n_part = 0;
    for (int it = 1; it <= m; ++it) {
        const float wf = cheb_step(it, alpha, &w, bufA, bufC, prev, &y);
        const int x0c = x_first || it > 2 ? 0 : it;      // 1: x is the compact rhs, 2: prev is
        HRAG_TRY(mixed_sweep_n(h, L, n, 0, rhs, x, prev, y, alpha, wf, 1.f, it == m, &n_part, x0c));
        prev = x;
        x = y;
        h->stats.ppr_sweeps += n;
        h->stats.ppr_columns += 32 * n;
    }
    HRAG_TRY(mixed_sums(h, n, n_part, which));   // local rows only: see dev_ppr_mixed_body
    *result = y;
    return 0;
}

// ---- sweep counts from (damping, tol) --------------------------------------------------------
// P is similar to a symmetric stochastic matrix, so the spectrum of aP is real in [-a, a]: Chebyshev
// semi-iteration contracts by sigma = a / (1 + sqrt(1 - a^2)) per sweep (0.268 at a = 0.5), the plain power
// sweep by a.  fp16 storage of the iterate leaves a relative L1 error of about kHalfNoise / (1 - a) in a
// converged fp16 solve (5e-4 at a = 0.5 against the float64 oracle); one refinement round
// multiplies the error by kappa = that + 2 sigma^m2.
constexpr double kHalfNoise = 2.5e-4;
// pure function of its arguments (exported as hrag_plan_sweeps so the rule is testable without a GPU); method:
// HRAG_PPR_CHEBYSHEV / HRAG_PPR_POWER for the fp32 solver; the *_override values are the handle's pins (0 = none)
static SweepPlan plan_sweeps_raw(int method, int fp32_override, int m1_override, int m2_override, float alpha,
                                 int iters_arg, float tol_arg, bool want_mixed) {
    SweepPlan p;
    const double a = alpha;
    const double sigma = method == HRAG_PPR_CHEBYSHEV ? a / (1.0 + std::sqrt(1.0 - a * a)) : a;
    p.tol = tol_arg > 0.f ? (double)tol_arg : kDefaultTol;
    // fp32 solver: truncation two decades under the target (1e-8 by default: the fp32 floor is ~1e-7)
    const double trunc = std::max(p.tol * 1e-2, 1e-10);
    p.iters = (int)std::ceil(std::log(trunc) / std::log(sigma) - 1e-9);
    if (fp32_override > 0) p.iters = fp32_override;
    if (iters_arg > 0) p.iters = iters_arg;
    p.iters = std::max(p.iters, 1);
    // mixed solver
    const double noise = kHalfNoise / (1.0 - a);
    const double sig_c = a / (1.0 + std::sqrt(1.0 - a * a));            // the fp16 solves are always Chebyshev
    p.m1 = (int)std::ceil(std::log(0.055 * noise) / std::log(sig_c) - 1e-9);
    p.m2 = (int)std::ceil(std::log(0.2 * noise) / std::log(sig_c) - 1e-9);
    if (m1_override > 0) p.m1 = m1_override;
    if (m2_override > 0) p.m2 = m2_override;
    if (iters_arg > 0) { p.m1 = iters_arg; p.m2 = std::max(1, iters_arg - 1); }
    p.m1 = std::max(p.m1, 1);
    p.m2 = std::max(p.m2, 1);
    p.kappa = noise + 2.0 * std::pow(sig_c, p.m2);
    const double e1 = noise + 2.0 * std::pow(sig_c, p.m1);
    const bool overridden = iters_arg > 0 || m1_override > 0 || m2_override > 0;
    // one refinement round must reach the target, otherwise the fp32 solver (which converges to its floor) runs
    p.mixed = want_mixed && (overridden || e1 * p.kappa <= p.tol);
    p.check = p.mixed && (!overridden || tol_arg > 0.f);
    return p;
}
SweepPlan plan_sweeps(const hrag_t* h, float alpha, int iters_arg, float tol_arg, bool want_mixed) {
    return plan_sweeps_raw(h->ppr_method, h->ppr_iters, h->mixed_m1, h->mixed_m2, alpha, iters_arg, tol_arg, want_mixed);
}

static int dev_ppr_mixed_body(hrag_t* h, const SweepPlan& plan, float alpha, int n, const MixedRhs* in, void** X0,
                              void** D) {
    const StateLayout& L = n == 2 ? h->pair : h->single;
    // the right-hand sides of the first solve (the compact or dense rhs), the residual (exact v) and the correction (r)
    MixedSweepIO first[2], resid[2], corr[2];
    for (int k = 0; k < n; ++k) {
        first[k].slot_map = resid[k].slot_map = in[k].slot_map;
        first[k].rhs_h = in[k].rhs16;
        resid[k].v32 = in[k].Vexact;
        resid[k].col_scale = in[k].scale;
        corr[k].rhs_h = L.R;
    }
    // x0_dense is also the correction's first work buffer, which its first sweep overwrites in full
    void* x0_dense = in[0].x0_dense;
    void* x0 = nullptr;
    void* d = nullptr;
    HRAG_TRY(mixed_cheb(h, L, n, first, in[0].x0_compact ? nullptr : x0_dense, L.A, L.C, plan.m1, alpha, &x0,
                        &MixedSums::x0));
    void* other = (x0 == L.A) ? L.C : L.A;
    int n_part = 0;
    HRAG_TRY(mixed_sweep_n(h, L, n, 1, resid, x0, nullptr, L.R, alpha, 1.f, kMixedT, true, &n_part));
    h->stats.ppr_sweeps += n;
    h->stats.ppr_columns += 32 * n;
    HRAG_TRY(mixed_sums(h, n, n_part, &MixedSums::r));
    HRAG_TRY(mixed_cheb(h, L, n, corr, L.R, x0_dense, other, plan.m2, alpha, &d, &MixedSums::d));
    if (h->world > 1) {      // node-range sharding: every rank summed its own rows -- ONE all-reduce for the three sums
        static_assert(sizeof(MixedSums) == 96 * sizeof(double), "x0, d and r sums are contiguous");
        StageTimer tc(h, ST_COMM);
        double* sums = sub_batch_sums(h, 0)->x0;
        HRAG_NCCL(g_nccl.AllReduce(sums, sums, 96, ncclDouble, ncclSum, h->comm, h->stream));
    }
    for (int k = 0; k < n; ++k) {
        HRAG_TRY(residual_check(sub_batch_sums(h, k)->r, in[k].vsum, in[k].scale, 1.f / kMixedT,
                                &h->rho.as<MixedRho>()->rho_max, h->stream));
        X0[k] = L.part(x0, k);
        D[k] = L.part(d, k);
    }
    return 0;
}

// The solve of one sub-batch is ~20 launches whose arguments depend only on the buffer set and the sweep plan, so on a
// single GPU it is captured once per (set, plan) into a CUDA graph and replayed (one launch per sub-batch instead of ~20:
// what bounds small real graphs like MuSiQue-1k, where a sweep is a few microseconds of work).  Multi-GPU runs (epoch
// values change per sweep) take the plain path.  n = 2 solves a pair of sub-batches in one paired walk per sweep
// (single GPU; in[0].x0_dense is then the pair's [N, 2, 32] buffer).  X0[k] / D[k] = sub-batch k's iterate and
// correction (rows L.ld halves apart), their column sums in sub_batch_sums(h, k).
static int dev_ppr_mixed(hrag_t* h, const SweepPlan& plan, float alpha, int n, const MixedRhs* in, void** X0,
                         void** D) {
    HRAG_CHECK(n == 1 || (n == 2 && h->world == 1), "internal: paired mixed solves run on a single GPU");
    StageTimer tm(h, ST_PPR);
    h->rho_dirty = true;     // set here, not in the body: the body runs on the host only while a graph is captured
    if (h->world > 1) {
        HRAG_TRY(dev_ppr_mixed_body(h, plan, alpha, n, in, X0, D));
        return p2p_wait(h);     // the consumers of X0 / D (gather kernels) need every peer's last rows
    }
    hrag_handle::SolveGraph* sg = nullptr;
    for (auto& c : h->solve_graphs)
        if (c.n == n && c.in[0] == in[0] && (n == 1 || c.in[1] == in[1]) && c.m1 == plan.m1 && c.m2 == plan.m2 &&
            c.alpha == alpha && c.generation == g_buf_generation) sg = &c;
    if (sg == nullptr) {
        if (h->solve_graphs.size() >= 8) HRAG_TRY(drop_captured_solves(h));   // bounded cache: drop everything stale
        hrag_handle::SolveGraph c;
        c.n = n;
        for (int k = 0; k < n; ++k) c.in[k] = in[k];
        c.m1 = plan.m1; c.m2 = plan.m2; c.alpha = alpha; c.generation = g_buf_generation;
        const int64_t sw0 = h->stats.ppr_sweeps, col0 = h->stats.ppr_columns, l0 = launches_since_reset();
        HRAG_CUDA(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
        const int rc = dev_ppr_mixed_body(h, plan, alpha, n, in, c.X0, c.D);
        cudaGraph_t graph = nullptr;
        const cudaError_t ce = cudaStreamEndCapture(h->stream, &graph);
        HRAG_TRY(rc);
        HRAG_CUDA(ce);
        HRAG_CUDA(cudaGraphInstantiate(&c.exec, graph, 0));
        cudaGraphDestroy(graph);
        c.sweeps = h->stats.ppr_sweeps - sw0; c.columns = h->stats.ppr_columns - col0; c.launches = launches_since_reset() - l0;
        h->stats.ppr_sweeps = sw0; h->stats.ppr_columns = col0;   // nothing ran yet: counted at launch below
        count_launch((int)-c.launches);
        h->solve_graphs.push_back(c);
        sg = &h->solve_graphs.back();
    }
    HRAG_CUDA(cudaGraphLaunch(sg->exec, h->stream));
    h->stats.ppr_sweeps += sg->sweeps;
    h->stats.ppr_columns += sg->columns;
    count_launch((int)sg->launches);
    for (int k = 0; k < n; ++k) {
        X0[k] = sg->X0[k];
        D[k] = sg->D[k];
    }
    return 0;
}

// single GPU: consecutive sub-batches of stage B are solved in pairs, one walk of the CSR per sweep for both (an odd
// last one alone); node-range sharding solves them one by one (its exchange is fused into the single-state sweep)
static bool solve_in_pairs(const hrag_t* h, int Bq) { return h->world == 1 && Bq > 32; }

int ensure_stage_b_mixed(hrag_t* h, int Bq, int k_facts) {
    const bool pairs = k_facts > 0 && solve_in_pairs(h, Bq);
    HRAG_TRY(ensure_state_mixed(h));
    if (pairs) HRAG_TRY(ensure_state_pair(h));
    return ensure_compact_rhs(h, pairs ? 4 : 2);
}

// Two streams: stream2 builds solve i+1's compact right-hand sides (passage weights + phrase seeds on P + 2048 slots,
// column scales and the fp16 copy) while `stream` runs the sweeps of solve i.  Solve i (one sub-batch, or a pair) uses
// the sets of parity i & 1: set p, and p + 2 for the second sub-batch of a pair, and the buffer x0[p] of its layout.
// On one GPU the first solve reads its first iterate compactly (MixedRhs::x0_compact); node-range sharding, whose
// peers exchange the rows of every sweep's input, and hrag_debug_dense_first_sweep scatter it into x0[p] first.
int stage_b_mixed(hrag_t* h, const SweepPlan& plan, int Bq, float* S, int64_t ldS, const float2* mm_pass, float pnw,
                  float damping) {
    const bool pairs = solve_in_pairs(h, Bq);
    const bool x0_compact = h->world == 1 && !h->debug_dense_first_sweep;
    if (plan.check) h->check_tol = std::max(h->check_tol, plan.tol), h->check_kappa = plan.kappa;
    HRAG_CUDA(cudaEventRecord(h->ev_inputs, h->stream));            // S, min/max, seed lists are ready
    HRAG_CUDA(cudaStreamWaitEvent(h->stream2, h->ev_inputs, 0));
    int it = 0;
    for (int q0 = 0; q0 < Bq; ++it) {
        const int n = pairs && Bq - q0 > 32 ? 2 : 1;
        const int par = it & 1;
        const StateLayout& L = n == 2 ? h->pair : h->single;
        if (it >= 2) HRAG_CUDA(cudaStreamWaitEvent(h->stream2, h->ev_released[par], 0));   // sets are free again
        MixedRhs in[2];
        int nb[2] = {0, 0};
        for (int k = 0; k < n; ++k) {
            RhsSet& set = h->rhs[par + 2 * k];
            const int qk = q0 + 32 * k;
            nb[k] = std::min(32, Bq - qk);
            in[k].x0_dense = L.x0[par];
            in[k].x0_compact = x0_compact;
            in[k].slot_map = set.slot_map.as<int>();
            in[k].Vexact = set.Vc.as<float>();
            in[k].rhs16 = set.R16.p;
            in[k].scale = set.scale.as<float>();
            in[k].vsum = set.vsum.as<double>();
            HRAG_TRY(compact_prepare_rhs(h->t, nb[k], qk, S, ldS, mm_pass, pnw, kSeedSlots, h->seed_vid.as<int>(),
                                         h->seed_w.as<double>(), damping, set.slot_map.as<int>(),
                                         set.slot_vid.as<int>(), set.Vc.as<float>(), set.R16.p,
                                         x0_compact ? nullptr : L.part(L.x0[par], k),
                                         L.ld, (int64_t)h->g.n_global, h->prep_scratch.as<float>(),
                                         set.vsum.as<double>(), set.scale.as<float>(), h->stream2));
        }
        HRAG_CUDA(cudaEventRecord(h->ev_ready[par], h->stream2));
        HRAG_CUDA(cudaStreamWaitEvent(h->stream, h->ev_ready[par], 0));
        void *X0[2] = {nullptr, nullptr}, *D[2] = {nullptr, nullptr};
        HRAG_TRY(dev_ppr_mixed(h, plan, damping, n, in, X0, D));
        {
            StageTimer tm(h, ST_TOPK);
            for (int k = 0; k < n; ++k) {
                const MixedSums* sums = sub_batch_sums(h, k);
                HRAG_TRY(gather_passage_scores_mixed(h->t, nb[k], q0 + 32 * k, X0[k], D[k], L.ld, 1.f / kMixedT,
                                                     sums->x0, sums->d, h->mode.as<int>(), mm_pass, S, ldS,
                                                     h->stream));
                HRAG_TRY(compact_release_slots(h->t.n_passages, nb[k], q0 + 32 * k, kSeedSlots, h->seed_vid.as<int>(),
                                               h->rhs[par + 2 * k].slot_map.as<int>(), h->stream));
            }
        }
        HRAG_TRY(p2p_signal(h));   // peers may overwrite this rank's state buffers from here on
        HRAG_CUDA(cudaEventRecord(h->ev_released[par], h->stream));
        q0 += 32 * n;
    }
    // (every prepare was consumed by a solve on `stream`, so stream2 is drained in stream order)
    return 0;
}

// Solves the PPR fixed point for the B columns of V; *result points at the final iterate
// (one of XA / XC), sums[b] = its column sums.
int dev_ppr(hrag_t* h, int B, int iters, float alpha, float** result) {
    HRAG_CHECK(iters >= 1, "ppr_iters must be >= 1");
    StageTimer tm(h, ST_PPR);
    float* V = h->V.as<float>();
    float* A = h->XA.as<float>();
    float* C = h->XC.as<float>();
    const bool cheb = h->ppr_method == HRAG_PPR_CHEBYSHEV;
    int n_part = 0;
    float *x = V, *prev = nullptr, *y = nullptr;
    double w = 1.0;
    for (int it = 1; it <= iters; ++it) {
        float* part = it == iters ? h->partials.as<float>() : nullptr;
        y = (it & 1) ? A : C;
        const float wf = cheb ? cheb_step(it, alpha, &w, A, C, prev, &y) : 1.f;
        HRAG_TRY(ppr_sweep(h->g, B, x, V, cheb ? prev : nullptr, y, alpha, wf, part, &n_part, h->stream));
        HRAG_TRY(exchange_rows(h, y, B));
        prev = x;
        x = y;
        h->stats.ppr_sweeps += 1;
        h->stats.ppr_columns += B;
    }
    HRAG_TRY(colsum_reduce(h->partials.as<float>(), n_part, B, h->sums.as<double>(), h->stream));
    if (h->world > 1) {
        StageTimer tc(h, ST_COMM);
        HRAG_NCCL(g_nccl.AllReduce(h->sums.p, h->sums.p, B, ncclDouble, ncclSum, h->comm, h->stream));
    }
    *result = y;
    return 0;
}

// Float64 PPR by iterative refinement (DESIGN.md section 2): per sub-batch of <= 16 columns, x = 0, r = v; every
// round solves (I - aP32) d = fp32(r) with the fp32 solver, x += d in fp64, and recomputes r = v - x + a(hi + lo)x
// in fp64.  P is column-substochastic, so ||(I - aP)^-1||_1 <= 1 / (1 - a), and ||x||_1 >= ||v||_1; normalising at
// most doubles the error, hence the rigorous bound ||pi - pi_hat||_1 <= 2 ||r||_1 / ((1 - a) ||v||_1) per column.
constexpr double kF64DefaultTol = 1e-10;   // PRPACK's target (HippoRAG.py:1736-1743)
constexpr double kF64MinTol = 1e-13;       // above the fp64 floor of the bound (~1e-14 at damping 0.5)
constexpr int kF64MaxRounds = 4;

int check_f64_call(hrag_t* h, const char* who, double damping, double tol) {
    const std::string w(who);
    HRAG_CHECK(damping > 0.0 && damping < 1.0, w + ": damping must be in (0, 1)");
    HRAG_CHECK(tol == 0.0 || tol >= kF64MinTol,
               w + ": tol must be 0 (= 1e-10) or >= 1e-13; a smaller bound is below what the fp64 residual can certify");
    HRAG_CHECK(h->g.n_global > 0, w + ": graph not loaded");
    HRAG_CHECK(h->world == 1, w + ": not available on a node-range-sharded handle (world > 1); solve on a handle that "
                                  "holds the whole graph");
    HRAG_CHECK(h->g.val_lo != nullptr, w + ": the graph was loaded from fp32 values and has no fp64 operator; load it "
                                           "with hrag_load_graph_csr_f64 or hrag_load_graph_coo");
    return 0;
}

double f64_target(double tol) { return tol > 0.0 ? tol : kF64DefaultTol; }

int ensure_state_f64(hrag_t* h, int Bp, int64_t io_cols) {
    const size_t cells = (size_t)h->g.n_global * Bp;
    HRAG_TRY(ensure_state(h, Bp));
    HRAG_TRY(h->X64.ensure(cells * sizeof(double)));
    HRAG_TRY(h->V64.ensure(cells * sizeof(double)));
    HRAG_TRY(h->io64.ensure((size_t)std::max<int64_t>(io_cols, h->g.n_global) * Bp * sizeof(double)));
    const int64_t rows_resid = resid_f64_partial_rows(h->g, Bp);
    const int64_t part_rows = std::max<int64_t>(2 * rows_resid, ceil_div((int64_t)cells, 256));
    HRAG_TRY(h->part64.ensure((size_t)part_rows * Bp * sizeof(double)));
    HRAG_TRY(h->sums64.ensure(48 * sizeof(double)));
    return 0;
}

int reset_f64(hrag_t* h, int Bp, int nb) {
    int n_part = 0;
    double* part_v = h->part64.as<double>();
    HRAG_TRY(reset_to_state_f64(h->io64.as<double>(), nb, h->g.n_global, Bp, h->V64.as<double>(), h->V.as<float>(),
                                h->X64.as<double>(), part_v, &n_part, h->stream));
    return colsum_reduce_f64(part_v, n_part, Bp, h->sums64.as<double>(), h->stream);
}

int refine_f64(hrag_t* h, int Bp, int nb, double damping, double target, F64Refined* out) {
    const int N = h->g.n_global;
    const size_t cells = (size_t)N * Bp;
    // the fp32 solves run at fp32(damping); the fp64 residual uses damping itself, so the refinement converges to
    // the solution at the damping asked (float32(0.85) alone moves pi by ~1e-7)
    const float damping32 = (float)damping;
    const SweepPlan plan = plan_sweeps(h, damping32, 0, (float)kDefaultTol, false);   // fp32 solver at its own tol
    const int64_t rows_resid = resid_f64_partial_rows(h->g, Bp);
    double* X = h->X64.as<double>();
    double* V = h->V64.as<double>();
    double* part_r = h->part64.as<double>();
    double* part_x = part_r + (size_t)rows_resid * Bp;
    double* vsum = h->sums64.as<double>();
    double* rsum = vsum + 16;
    double* xsum = vsum + 32;
    const double a = damping;
    // every column refines until its own bound meets the target and then keeps its iterate: a query's result does
    // not depend on the queries it shares the sub-batch with
    unsigned active = (1u << nb) - 1u;
    double resid = 0.0;
    for (int round = 0; round < kF64MaxRounds && active; ++round) {
        float* D = nullptr;
        int n_part = 0;
        HRAG_TRY(dev_ppr(h, Bp, plan.iters, damping32, &D));    // (I - aP32) d = fp32(r), r = h->V
        {
            StageTimer tm(h, ST_PPR);
            HRAG_TRY(add_correction_f64(X, D, (int64_t)cells, Bp, active, h->stream));
            HRAG_TRY(resid_sweep_f64(h->g, Bp, X, V, h->V.as<float>(), a, part_r, part_x, &n_part, h->stream));
            HRAG_TRY(colsum_reduce_f64(part_r, n_part, Bp, rsum, h->stream));
            HRAG_TRY(colsum_reduce_f64(part_x, n_part, Bp, xsum, h->stream));
        }
        h->stats.ppr_sweeps += 1;
        h->stats.ppr_columns += Bp;
        double s[32];
        HRAG_CUDA(cudaMemcpyAsync(s, vsum, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
        resid = 0.0;
        for (int b = 0; b < nb; ++b) {
            const double rel = s[b] > 0.0 ? s[16 + b] / s[b] : 0.0;   // a reset without mass has nothing to bound
            resid = std::max(resid, rel);
            if (2.0 * rel / (1.0 - a) <= target) active &= ~(1u << b);
        }
    }
    out->resid = resid;
    out->bound = 2.0 * resid / (1.0 - a);
    out->active = active;
    return 0;
}

// A call's end when a sub-batch missed the target: the stats report the call so far, status 4
int f64_missed(hrag_t* h, const char* who, const F64Refined& r, double target, double call_resid, double call_bound) {
    HRAG_TRY(resolve_spans(h));
    h->last_rho = std::max(call_resid, r.resid);
    h->last_bound = std::max(call_bound, r.bound);
    char msg[200];
    snprintf(msg, sizeof(msg), "%s: after %d refinement rounds the error bound is %.3e, above tol %.3e", who,
             kF64MaxRounds, r.bound, target);
    set_error(msg);
    return 4;
}

}  // namespace hrag

using namespace hrag;

extern "C" {

int hrag_ppr(hrag_t* h, int32_t B, const float* reset, float damping, int32_t iters, float tol, float* out) {
    HRAG_CHECK(h && reset && out, "hrag_ppr: null argument");
    HRAG_CHECK(B >= 0 && damping > 0.f && damping < 1.f, "hrag_ppr: bad arguments");
    HRAG_CHECK(iters >= 0 && tol >= 0.f, "hrag_ppr: iters and tol must be >= 0 (0 = derive from damping)");
    HRAG_CHECK(h->g.n_global > 0, "hrag_ppr: graph not loaded");
    HRAG_CUDA(cudaSetDevice(h->device));
    const int N = h->g.n_global;
    // same gate as stage B: batches of <= 16 reset vectors run the fp32 solver at their own width
    const SweepPlan plan = plan_sweeps(h, damping, iters, tol, h->ppr_precision == HRAG_PPR_MIXED && B > 16);
    const bool mixed = plan.mixed;
    const int Bp = mixed ? 32 : round_batch(std::min(h->ppr_batch, std::max(B, 1)));
    if (mixed) { HRAG_TRY(ensure_state_mixed(h)); HRAG_TRY(h->V.ensure(state_rows(h) * 32 * sizeof(float))); }
    else HRAG_TRY(ensure_state(h, Bp));
    if (mixed && plan.check) { h->check_tol = plan.tol; h->check_kappa = plan.kappa; }
    HRAG_TRY(h->d_reset.ensure((size_t)Bp * N * sizeof(float)));
    HRAG_TRY(h->d_scores.ensure((size_t)Bp * N * sizeof(float)));
    for (int q0 = 0; q0 < B; q0 += Bp) {
        const int nb = std::min(Bp, B - q0);
        HRAG_TRY(h2d(h, h->d_reset.p, reset + (size_t)q0 * N, (size_t)nb * N * sizeof(float)));
        HRAG_TRY(reset_to_state(h->d_reset.as<float>(), nb, N, Bp, h->V.as<float>(), h->stream));
        if (mixed) {
            void *X0 = nullptr, *D = nullptr;
            MixedRhs in;
            in.Vexact = h->V.as<float>();
            in.rhs16 = in.x0_dense = h->single.x0[0];
            in.scale = h->rhs[0].scale.as<float>();
            in.vsum = h->rhs[0].vsum.as<double>();
            HRAG_TRY(mixed_prepare_rhs(in.Vexact, (int64_t)N, damping, h->mixed_part[0].as<float>(),
                                       h->rhs[0].vsum.as<double>(), h->rhs[0].scale.as<float>(), in.x0_dense,
                                       h->stream));
            HRAG_TRY(dev_ppr_mixed(h, plan, damping, 1, &in, &X0, &D));
            const MixedSums* sums = sub_batch_sums(h, 0);
            HRAG_TRY(state_to_scores_mixed(X0, D, 1.f / kMixedT, nb, N, sums->x0, sums->d, h->d_scores.as<float>(),
                                           h->stream));
            HRAG_TRY(p2p_signal(h));
        } else {
            float* Z = nullptr;
            HRAG_TRY(dev_ppr(h, Bp, plan.iters, damping, &Z));
            HRAG_TRY(state_to_scores(Z, nb, N, Bp, h->sums.as<double>(), h->d_scores.as<float>(), h->stream));
        }
        HRAG_TRY(d2h(h, out + (size_t)q0 * N, h->d_scores.p, (size_t)nb * N * sizeof(float)));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
    }
    return resolve_spans(h);
}

int hrag_bench_sweep(hrag_t* h, int32_t B, int32_t sweeps, int32_t method, float* ms_per_sweep) {
    HRAG_CHECK(h && ms_per_sweep && sweeps >= 1, "hrag_bench_sweep: bad arguments");
    HRAG_CHECK(B == 4 || B == 8 || B == 16 || B == 32 || B == 64, "hrag_bench_sweep: B in {4,8,16,32,64}");
    HRAG_CHECK(h->g.n_global > 0, "hrag_bench_sweep: graph not loaded");
    HRAG_CUDA(cudaSetDevice(h->device));
    // fp16-state sweep (Chebyshev form), B = 32: 2 = dense rhs, 3 = compact rhs, 4 = the paired sweep of two
    // compact-rhs sub-batches ([N, 2, 32] state), timed per paired sweep (64 columns); 5 / 6 = the paired first sweep
    // of a solve (plain), gathering the dense first iterate x0 (5) or the compact rhs through the slot maps (6)
    const bool first = method == 5 || method == 6;
    const bool paired = method == 4 || first;
    const bool mixed = method == 2 || method == 3 || paired;
    HRAG_CHECK(!paired || h->world == 1, "hrag_bench_sweep: the paired sweep runs on a single-GPU handle");
    const bool cheb = method == HRAG_PPR_CHEBYSHEV;
    MixedSweepIO rhs[2];     // the fp16 sweeps' right-hand sides
    void *A = nullptr, *C = nullptr;
    if (mixed) {
        HRAG_CHECK(B == 32, "hrag_bench_sweep: the mixed solver runs at B = 32");
        HRAG_TRY(ensure_state_mixed(h));
        const StateLayout& L = h->single;
        rhs[0].rhs_h = L.x0[0];
        if (method >= 3) {
            HRAG_CHECK(h->t.passage_vid != nullptr, "hrag_bench_sweep: the compact-rhs sweep needs hrag_load_tables");
            HRAG_TRY(ensure_compact_rhs(h, 2));
            for (int s = 0; s < 2; ++s) {
                rhs[s].slot_map = h->rhs[s].slot_map.as<int>();
                rhs[s].rhs_h = h->rhs[s].R16.p;
                HRAG_CUDA(cudaMemsetAsync(h->rhs[s].R16.p, 0x2c, h->rhs[s].R16.cap, h->stream));
            }
        }
        const size_t hb = (size_t)h->g.n_global * 32 * 2;
        for (void* p : {L.x0[0], L.A, L.C}) HRAG_CUDA(cudaMemsetAsync(p, 0x2c, hb, h->stream));   // 0x2c2c = 0.065
        A = L.A, C = L.C;
        if (paired) {
            HRAG_TRY(ensure_state_pair(h));
            for (void* p : {h->pair.x0[0], h->pair.A, h->pair.C}) HRAG_CUDA(cudaMemsetAsync(p, 0x2c, 2 * hb, h->stream));
            A = h->pair.A, C = h->pair.C;
        }
    } else {
        HRAG_TRY(ensure_state(h, B));
        const size_t bytes = (size_t)h->g.n_global * B * sizeof(float);
        HRAG_CUDA(cudaMemsetAsync(h->V.p, 0x3c, bytes, h->stream));     // 0x3c3c3c3c = 0.0115f
        HRAG_CUDA(cudaMemsetAsync(h->XA.p, 0x3c, bytes, h->stream));
        HRAG_CUDA(cudaMemsetAsync(h->XC.p, 0x3c, bytes, h->stream));
        A = h->XA.p, C = h->XC.p;
    }
    cudaEvent_t e0, e1;
    HRAG_CUDA(cudaEventCreate(&e0));
    HRAG_CUDA(cudaEventCreate(&e1));
    for (int pass = 0; pass < 2; ++pass) {   // pass 0 = warm-up (3 sweeps), pass 1 = timed
        const int n = pass == 0 ? 3 : sweeps;
        if (pass == 1) HRAG_CUDA(cudaEventRecord(e0, h->stream));
        for (int i = 0; i < n; ++i) {
            void* x = (i & 1) ? C : A;
            void* y = (i & 1) ? A : C;
            float* yf = static_cast<float*>(y);
            if (first) {
                const bool dense = method == 5;
                HRAG_TRY(mixed_sweep_n(h, h->pair, 2, 0, rhs, dense ? h->pair.x0[0] : nullptr, nullptr, y, 0.5f, 1.f,
                                       1.f, false, nullptr, dense ? 0 : 1));
            } else if (mixed) {
                HRAG_TRY(mixed_sweep_n(h, paired ? h->pair : h->single, paired ? 2 : 1, 0, rhs, x, y, y, 0.5f, 1.07f,
                                       1.f, false, nullptr));
            } else {
                HRAG_TRY(ppr_sweep(h->g, B, static_cast<float*>(x), h->V.as<float>(), cheb ? yf : nullptr, yf, 0.5f,
                                   cheb ? 1.07f : 1.f, nullptr, nullptr, h->stream));
                HRAG_TRY(exchange_rows(h, yf, B));
            }
        }
        if (pass == 1) HRAG_CUDA(cudaEventRecord(e1, h->stream));
    }
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    float ms = 0.f;
    HRAG_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    *ms_per_sweep = ms / sweeps;
    for (auto& s : h->spans) { h->pool.push_back(s.a); h->pool.push_back(s.b); }
    h->spans.clear();
    return 0;
}

int hrag_ppr_f64(hrag_t* h, int32_t B, const double* reset, double damping, double tol, double* out) {
    HRAG_CHECK(h && reset && out, "hrag_ppr_f64: null argument");
    HRAG_CHECK(B >= 0, "hrag_ppr_f64: bad arguments");
    HRAG_TRY(check_f64_call(h, "hrag_ppr_f64", damping, tol));
    HRAG_CUDA(cudaSetDevice(h->device));
    const double target = f64_target(tol);
    const int N = h->g.n_global;
    const int Bp = round_batch(std::min(16, std::max(B, 1)));
    HRAG_TRY(ensure_state_f64(h, Bp, N));
    double* xsum = h->sums64.as<double>() + 32;
    double call_resid = 0.0, call_bound = 0.0;
    for (int q0 = 0; q0 < B; q0 += Bp) {
        const int nb = std::min(Bp, B - q0);
        HRAG_TRY(h2d(h, h->io64.p, reset + (size_t)q0 * N, (size_t)nb * N * sizeof(double)));
        HRAG_TRY(reset_f64(h, Bp, nb));
        F64Refined r;
        HRAG_TRY(refine_f64(h, Bp, nb, damping, target, &r));
        if (r.active) return f64_missed(h, "hrag_ppr_f64", r, target, call_resid, call_bound);
        call_resid = std::max(call_resid, r.resid);
        call_bound = std::max(call_bound, r.bound);
        HRAG_TRY(state_to_scores_f64(h->X64.as<double>(), nb, N, Bp, xsum, h->io64.as<double>(), h->stream));
        HRAG_TRY(d2h(h, out + (size_t)q0 * N, h->io64.p, (size_t)nb * N * sizeof(double)));
        HRAG_CUDA(cudaStreamSynchronize(h->stream));
    }
    HRAG_TRY(resolve_spans(h));
    h->last_rho = call_resid;
    h->last_bound = call_bound;
    return 0;
}

int hrag_plan_sweeps(float damping, float tol, int32_t iters, int32_t batch, int32_t* use_mixed, int32_t* fp32_sweeps,
                     int32_t* mixed_sweeps1, int32_t* mixed_sweeps2, double* predicted_error) {
    HRAG_CHECK(use_mixed && fp32_sweeps && mixed_sweeps1 && mixed_sweeps2 && predicted_error, "hrag_plan_sweeps: null argument");
    HRAG_CHECK(damping > 0.f && damping < 1.f && tol >= 0.f && iters >= 0, "hrag_plan_sweeps: bad arguments");
    const SweepPlan p = plan_sweeps_raw(HRAG_PPR_CHEBYSHEV, 0, 0, 0, damping, iters, tol, batch > 16);
    const double a = damping, sig = a / (1.0 + std::sqrt(1.0 - a * a)), noise = kHalfNoise / (1.0 - a);
    *use_mixed = p.mixed ? 1 : 0;
    *fp32_sweeps = p.iters;
    *mixed_sweeps1 = p.m1;
    *mixed_sweeps2 = p.m2;
    *predicted_error = p.mixed ? (noise + 2.0 * std::pow(sig, p.m1)) * p.kappa : 2.0 * std::pow(sig, p.iters);
    return 0;
}

}  // extern "C"
